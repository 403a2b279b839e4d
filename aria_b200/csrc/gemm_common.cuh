// Shared pieces of the wgmma GEMM kernels (gemm.cu: dense / grouped GEMMs, gemm_wgrad.cu: weight gradients): parameters,
// the device-side tile scheduler and the fused epilogues.
//
// Persistent, warp-specialised wgmma GEMM for sm_90a (bf16 x bf16 -> fp32 in registers -> bf16):
//   * warpgroup 0 : TMA producer (one elected thread: cp.async.bulk.tensor, SWIZZLE_128B tiles, mbarrier complete_tx)
//   * warpgroups 1-2 : consumers; each issues wgmma m64 x BN x k16 for its 64 rows of the 128-row tile, then stages its fp32
//     accumulator in shared memory and runs the fused epilogue row by row (two threads per row, 16-byte global stores).
//     The producer keeps streaming the next tile's k-blocks into the ring meanwhile.
//
// One kernel template serves (a) nn.Linear-layout dense GEMMs (B = [N,K], K-major), (b) the reference's
// grouped expert GEMM (aria/model/moe_lm.py:398-428,467-484: B = [E,K,N], consumed N-contiguous through an
// MN-major wgmma descriptor — the HF weight layout is used as is, no repack) with a device-side tile
// scheduler over the expert row offsets (no host sync, cf. moe_lm.py:478), and (c) the fused epilogues:
// bias/activation/residual, SwiGLU (moe_lm.py:505-507), and RoPE + head-major scatter for q/k/v.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int GEMM_THREADS = 384;  // warpgroup 0 TMA producer, warpgroups 1-2 MMA + epilogue (64 rows each)
constexpr int CONSUMER_WARPS = 8;
constexpr int acc_ld(int BN) { return BN + 4; }  // staging row stride (floats): 16-byte aligned rows, spread over the banks

struct GemmParams {
  int M, N, K;  // N = output columns per segment
  int num_groups;
  const int32_t* group_offsets;
  const int32_t* group_counts;     // non-NULL: group g = rows [group_offsets[g], + group_counts[g]) (fixed-capacity regions)
  const uint64_t* out_group_base;  // non-NULL (LINEAR): rows of group g are stored at out_group_base[g] + (out_group_row0[g] + r)*ldo
  const int32_t* out_group_row0;   //   — e.g. straight into the source rank's combine buffer over NVLink (expert parallelism)
  int b_group_rows;  // K-major grouped weights [G, N, K]: B row of (group g, column c) is g*b_group_rows + c (0: dense)
  int group_mod;  // weight block of group g: g % group_mod (> 0: expert-parallel (source rank, expert) groups), g / -group_mod (< 0:
                  // (expert, source rank) groups - the groups of one expert are neighbours and share its weights in L2), g (0)
  int n_seg;
  int act;
  const __nv_bfloat16* bias[3];
  const __nv_bfloat16* residual;
  int64_t ldr;
  __nv_bfloat16* out[3];
  int64_t ldo;
  int head_dim, head_ld, rows_per_batch, pos0;
  int64_t stride_b, stride_h;
  int rope_mask;
  const __nv_bfloat16* rope_cos;
  const __nv_bfloat16* rope_sin;
  const int32_t* position_ids;
  const float* b_scale;  // fp8 B (gemm_kernel<.., B_FP8 = true>, gemm_w8a8_kernel): [G, B columns] fp32 scale of each weight column
};

ARIA_DEVICE int weight_block(const GemmParams& p, int grp) {
  return p.group_mod > 0 ? grp % p.group_mod : (p.group_mod < 0 ? grp / (-p.group_mod) : grp);
}

// The dynamic shared memory from its first 1024-byte boundary: the SW128 swizzle pattern repeats every 1024 bytes
ARIA_DEVICE uint8_t* smem_1024() {
  extern __shared__ uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

// full / empty mbarrier pairs of a STAGES-slot ring at `at`: full[i] completes when slot i holds its data, empty[i] when its
// readers have released it.  init() runs on one thread before the block's first barrier.
template <int STAGES>
struct BarrierRing {
  uint64_t* full;
  uint64_t* empty;
  ARIA_DEVICE explicit BarrierRing(void* at) : full(static_cast<uint64_t*>(at)), empty(full + STAGES) {}
  ARIA_DEVICE void init(uint32_t full_arrivals, uint32_t empty_arrivals) const {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], full_arrivals);
      mbar_init(&empty[i], empty_arrivals);
    }
  }
};

// A reader's or writer's position in a STAGES-slot ring: the slot, and the barrier phase it waits for there
template <int STAGES>
struct RingPos {
  uint32_t stage = 0, phase = 0;
  ARIA_DEVICE void next() {
    const bool wrap = ++stage == STAGES;
    stage = wrap ? 0 : stage;
    phase ^= wrap;
  }
};

// Column of B that column x of tile n_idx multiplies: BN consecutive columns, or for SwiGLU the gate columns
// [n_idx BN/2, +BN/2), then the matching up columns, N further on
template <int BN, int EPI>
ARIA_DEVICE int tile_b_col(int x, int n_idx, int N) {
  constexpr int OUT_BN = BN / 2;
  if constexpr (EPI == ARIA_EPI_SWIGLU) return x < OUT_BN ? n_idx * OUT_BN + x : N + n_idx * OUT_BN + x - OUT_BN;
  else return n_idx * BN + x;
}

// Grouped launches (group_offsets != NULL) pack the groups' rows back to back, so a BM-row A box of a group's last m-tile would
// mostly fetch other groups' rows: at 72 rows per expert 56 of 128, at batch-32 decode 125 of 128, again for every n-tile of
// the group.  Their producer loads only the rows the group owns, rounded up to the smaller box of a second tensor map.
constexpr int A_BOX_MIN = 16;
ARIA_DEVICE int tile_a_rows(int rows, int m_idx) { return min(BM, (rows - m_idx * BM + A_BOX_MIN - 1) & ~(A_BOX_MIN - 1)); }

// Loads the first n_rows (a multiple of A_BOX_MIN: tile_a_rows, or BM for a dense launch) rows of the A tile at row `row`
// into the stage at `sa`, n_rows * 128 bytes on the mbarrier: a whole tile as the one box of `full`, a shorter one as boxes of
// `small` (A_BOX_MIN rows).  SW128 swizzles by shared-memory address and a small box is two whole 1 KB swizzle atoms, so the
// boxes compose to the bytes the BM-row box would have put there.  (A 64-row box in front of the small ones measured the same
// as small boxes alone, DESIGN §6.)
// INVARIANT: the stage's rows past n_rows keep whatever an earlier tile left there, and the consumers still multiply them.
// That is safe only because row r of the accumulator depends on row r of A alone, and every epilogue a grouped launch
// reaches (LINEAR, SWIGLU: one thread per row, stores under row_ok) neither stores a row at or past the group's end nor
// reads another row's values for a row it stores.
ARIA_DEVICE void tma_load_a_rows(uint32_t sa, const CUtensorMap* full, const CUtensorMap* small, uint32_t bar_addr, int c0,
                                 int row, int n_rows) {
  if (n_rows == BM) return tma_load_2d_addr(sa, full, bar_addr, c0, row);
  for (int r = 0; r < n_rows; r += A_BOX_MIN) tma_load_2d_addr(sa + r * 128, small, bar_addr, c0, row + r);
}

// Whether a consumer warp skips a tile.  The condition is the same in every lane, which the compiler cannot see; taken from
// lane 0 it is uniform to it as well.  Otherwise it treats the skip as a divergent branch and puts a warp re-convergence in
// front of every k-block's first wgmma, which cost the compute-bound fp8 launches 2-4 % (H100 SXM, 700 W).
ARIA_DEVICE bool sits_out(bool cond) { return __shfl_sync(0xffffffffu, cond ? 1 : 0, 0) != 0; }

// A consumer thread: its place in the wgmma accumulator fragment of its warpgroup's 64 rows (cw: warpgroup 1 or 2 -> 0 / 1),
// and the row it finishes in the epilogue with its `half` of the columns
struct ConsumerThread {
  int cw, frag_row, frag_col, epi_row, half;
};
ARIA_DEVICE ConsumerThread consumer_thread(int cw, int lane) {
  const int tid = threadIdx.x & 127;
  return {cw, cw * 64 + (tid >> 5) * 16 + (lane >> 2), 2 * (lane & 3), cw * 64 + (tid & 63), tid >> 6};
}

// The scales of this thread's accumulator columns (8 j + frag_col, +1) in tile n_idx of group grp, fetched while the k-loop
// runs; columns past the weight's end get 0
template <int BN, int EPI>
ARIA_DEVICE void load_col_scales(const GemmParams& p, int grp, int n_idx, int frag_col, float2 (&bsc)[BN / 8]) {
  const int ncols = EPI == ARIA_EPI_SWIGLU ? 2 * p.N : p.N;
  const float* srow = p.b_scale + static_cast<int64_t>(weight_block(p, grp)) * ncols;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = tile_b_col<BN, EPI>(8 * j, n_idx, p.N) + frag_col;
    bsc[j] = col < ncols ? __ldg(reinterpret_cast<const float2*>(srow + col)) : make_float2(0.f, 0.f);
  }
}

// Monotonic decoder of the persistent tile index -> (group, m-tile, n-tile).  Tiles are ordered group-major,
// then n-tile, with the m-tile innermost so that CTAs running concurrently share the same weight tile.
struct TileSched {
  const int32_t* offs;
  const int32_t* cnts;
  int G, n_tiles, M;
  int g, mt_prefix, g_row0, g_rows, g_mt, bm;
  __device__ void init(const GemmParams& p, int n_tiles_, int bm_ = BM) {
    bm = bm_;
    offs = p.group_offsets;
    cnts = p.group_counts;
    G = p.num_groups;
    n_tiles = n_tiles_;
    M = p.M;
    g = -1;
    mt_prefix = 0;
    g_mt = 0;
    g_row0 = 0;
    g_rows = 0;
  }
  __device__ bool load_group(int gi) {
    if (gi >= G) return false;
    if (offs) {
      g_row0 = offs[gi];
      g_rows = cnts ? cnts[gi] : offs[gi + 1] - g_row0;
    } else {
      g_row0 = 0;
      g_rows = M;
    }
    g_mt = (g_rows + bm - 1) / bm;
    return true;
  }
  __device__ bool decode(int t, int& grp, int& m_idx, int& n_idx, int& row0, int& rows) {
    if (g < 0) {
      g = 0;
      if (!load_group(0)) return false;
    }
    while (t >= (mt_prefix + g_mt) * n_tiles) {
      mt_prefix += g_mt;
      ++g;
      if (!load_group(g)) return false;
    }
    int r = t - mt_prefix * n_tiles;
    n_idx = r / g_mt;
    m_idx = r - n_idx * g_mt;
    grp = g;
    row0 = g_row0;
    rows = g_rows;
    return true;
  }
};

ARIA_DEVICE float act_apply(float x, int act) {
  if (act == ARIA_ACT_GELU_TANH) {
    // torch gelu(approximate="tanh"): one fp32 evaluation, rounded once by the caller
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    float inner = k0 * (x + k1 * x * x * x);
    return 0.5f * x * (1.f + fast_tanh(inner));
  }
  if (act == ARIA_ACT_GELU_NEW) {
    // transformers NewGELUActivation evaluated op by op on bf16 tensors (aria/model/projector.py:40-45):
    // 0.5 * x * (1.0 + tanh(sqrt(2/pi) * (x + 0.044715 * pow(x, 3))))
    float p3 = bf16r(x * x * x);
    float t = bf16r(0.044715f * p3);
    t = bf16r(x + t);
    t = bf16r(0.7978845608028654f * t);
    t = bf16r(fast_tanh(t));
    t = bf16r(1.0f + t);
    float h = bf16r(0.5f * x);
    return h * t;
  }
  return x;
}

// 32 consecutive fp32 accumulator values of one row of the shared-memory staging tile (16-byte aligned)
ARIA_DEVICE void ld_acc32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + 4 * i);
    r[4 * i] = v.x;
    r[4 * i + 1] = v.y;
    r[4 * i + 2] = v.z;
    r[4 * i + 3] = v.w;
  }
}

// Fused epilogue of one accumulator tile: this thread owns one output row and walks the tile's columns in 32-column
// chunks.  `acc` points at the row in the shared-memory staging tile (fp32, BN columns).
//   LINEAR / HEADS : the tile covers output columns [n_idx*BN, +BN)
//   SWIGLU         : accumulator columns [0,BN/2) hold the gate, [BN/2,BN) the up projection; output columns
//                    [n_idx*BN/2, +BN/2)
// `half` (0/1) selects which half of the tile's column chunks this thread handles: two threads share each row.
template <int BN, int EPI>
ARIA_DEVICE void epilogue_tile(const GemmParams& p, const float* acc, const int n_out_total, const int n_idx,
                               const int64_t grow, const bool row_ok, const int half, const int grp = 0, const int r_in_grp = 0) {
  constexpr int OUT_BN = (EPI == ARIA_EPI_SWIGLU) ? BN / 2 : BN;
  if constexpr (EPI == ARIA_EPI_SWIGLU) {
    // out[:, n] = bf16( bf16(silu(bf16(gate))) * bf16(up) )  — rounding points of moe_lm.py:505-507
    __nv_bfloat16* orow = p.out[0] + grow * p.ldo + n_idx * OUT_BN;
    constexpr int NCH = OUT_BN / 32;
    const int cb = (half * NCH / 2) * 32, ce = half ? OUT_BN : (NCH / 2) * 32;
#pragma unroll 1
    for (int c = cb; c < ce; c += 32) {
      uint32_t g[32], u[32];
      ld_acc32(acc + c, g);
      ld_acc32(acc + OUT_BN + c, u);
      uint32_t o[16];
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        float g0 = __uint_as_float(g[j]), g1 = __uint_as_float(g[j + 1]);
        float u0 = __uint_as_float(u[j]), u1 = __uint_as_float(u[j + 1]);
        bf16r2(g0, g1);
        bf16r2(u0, u1);
        float s0 = fast_silu(g0), s1 = fast_silu(g1);
        bf16r2(s0, s1);
        o[j >> 1] = pack_bf16(s0 * u0, s1 * u1);
      }
      if (row_ok) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int col = n_idx * OUT_BN + c + q * 8;
          if (col + 8 <= p.N)
            *reinterpret_cast<uint4*>(orow + c + q * 8) = make_uint4(o[q * 4], o[q * 4 + 1], o[q * 4 + 2], o[q * 4 + 3]);
        }
      }
    }
  } else if constexpr (EPI == ARIA_EPI_LINEAR) {
    const int col0 = n_idx * BN;
    const int seg = col0 / p.N;  // bias is per segment; out is [m, n_seg*n]
    const __nv_bfloat16* bias = p.bias[seg];
    __nv_bfloat16* orow = p.out[0] + grow * p.ldo + col0;
    if (p.out_group_base)  // per-group destination (possibly a peer GPU's memory: the stores then travel over NVLink)
      orow = reinterpret_cast<__nv_bfloat16*>(p.out_group_base[grp]) + static_cast<int64_t>(p.out_group_row0[grp] + r_in_grp) * p.ldo + col0;
    const __nv_bfloat16* rrow = (p.residual && row_ok) ? p.residual + grow * p.ldr + col0 : nullptr;
    // Two-deep software pipeline over the 32-column chunks of this thread's half: the accumulator chunk, the bias vectors and
    // the residual row pieces of chunk i + 1 are all in flight while chunk i is converted and stored, so the global-load
    // latencies overlap instead of adding up once per 8 columns.
    constexpr int NCH = BN / 32, NCHH = NCH - NCH / 2;  // chunks of the tile / of the larger half (BN = 32: all in half 1)
    const int cb = half ? (NCH / 2) * 32 : 0;
    const int n_my = half ? NCH - NCH / 2 : NCH / 2;
    if (n_my == 0) return;
    uint32_t v[2][32];
    uint4 bv[2][4], rv[2][4];
    auto issue = [&](int c, int set) {
      ld_acc32(acc + c, v[set]);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int col = col0 + c + q * 8;
        const bool ok = col + 8 <= n_out_total;
        bv[set][q] = (bias && ok) ? __ldg(reinterpret_cast<const uint4*>(bias + (col - seg * p.N))) : make_uint4(0, 0, 0, 0);
        rv[set][q] = (rrow && ok) ? *reinterpret_cast<const uint4*>(rrow + c + q * 8) : make_uint4(0, 0, 0, 0);
      }
    };
    issue(cb, 0);
#pragma unroll
    for (int i = 0; i < NCHH; ++i) {
      if (i >= n_my) break;
      const int c = cb + i * 32;
      const int set = i & 1;
      if (i + 1 < n_my) issue(c + 32, set ^ 1);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int col = col0 + c + q * 8;
        if (col + 8 > n_out_total) continue;
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = __uint_as_float(v[set][q * 8 + j]);
        if (bias) {
          const uint32_t bw[4] = {bv[set][q].x, bv[set][q].y, bv[set][q].z, bv[set][q].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            x[2 * j] += bf16_lo(bw[j]);
            x[2 * j + 1] += bf16_hi(bw[j]);
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = bf16r(x[j]);
        if (p.act != ARIA_ACT_NONE) {
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = bf16r(act_apply(x[j], p.act));
        }
        if (row_ok) {
          if (rrow) {
            const uint32_t rw[4] = {rv[set][q].x, rv[set][q].y, rv[set][q].z, rv[set][q].w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              x[2 * j] += bf16_lo(rw[j]);
              x[2 * j + 1] += bf16_hi(rw[j]);
            }
          }
          *reinterpret_cast<uint4*>(orow + c + q * 8) =
              make_uint4(pack_bf16(x[0], x[1]), pack_bf16(x[2], x[3]), pack_bf16(x[4], x[5]), pack_bf16(x[6], x[7]));
        }
      }
    }
  } else {  // ARIA_EPI_HEADS, a RoPE segment (the others go through heads_store_tile)
    const int col0 = n_idx * BN;
    const int seg = col0 / p.N;
    const int cseg0 = col0 - seg * p.N;
    const int b = static_cast<int>(grow / p.rows_per_batch);
    const int tok = static_cast<int>(grow - static_cast<int64_t>(b) * p.rows_per_batch);
    __nv_bfloat16* obase = p.out[seg] + b * p.stride_b + static_cast<int64_t>(p.pos0 + tok) * p.head_ld;
    // head_dim == 128 and BN a multiple of it: the tile holds BN/128 whole heads. rotate-half RoPE with op-by-op
    // bf16 rounding:  out = bf16(bf16(x*cos) + bf16(rotate_half(x)*sin))
    const int pos = row_ok ? (p.position_ids ? p.position_ids[grow] : p.pos0 + tok) : 0;
    const __nv_bfloat16* cs = p.rope_cos + static_cast<int64_t>(pos) * p.head_dim;
    const __nv_bfloat16* sn = p.rope_sin + static_cast<int64_t>(pos) * p.head_dim;
    constexpr int NHC = BN / 64;
#pragma unroll 1
    for (int hc = half * NHC / 2; hc < (half ? NHC : NHC / 2); hc += 1) {
      // hc enumerates (head-in-tile, 32-column chunk of the low half): hh = hc / 2, c = (hc & 1) * 32
      const int hh = hc >> 1, c = (hc & 1) * 32;
      __nv_bfloat16* orow = obase + (cseg0 / p.head_dim + hh) * p.stride_h;
      const float* th = acc + hh * 128;
      uint32_t lo[32], hi[32];
      ld_acc32(th + c, lo);
      ld_acc32(th + 64 + c, hi);
      // all 16 table vectors of this chunk are requested before anything waits (they were loaded one group at a time
      // inside the loop below, each followed by its use)
      uint4 tc_lo[4], ts_lo[4], tc_hi[4], ts_hi[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        tc_lo[q] = __ldg(reinterpret_cast<const uint4*>(cs + c + q * 8));
        ts_lo[q] = __ldg(reinterpret_cast<const uint4*>(sn + c + q * 8));
        tc_hi[q] = __ldg(reinterpret_cast<const uint4*>(cs + 64 + c + q * 8));
        ts_hi[q] = __ldg(reinterpret_cast<const uint4*>(sn + 64 + c + q * 8));
      }
      if (row_ok) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint4 c_lo = tc_lo[q], s_lo = ts_lo[q], c_hi = tc_hi[q], s_hi = ts_hi[q];
          const uint32_t cl[4] = {c_lo.x, c_lo.y, c_lo.z, c_lo.w}, sl[4] = {s_lo.x, s_lo.y, s_lo.z, s_lo.w};
          const uint32_t ch[4] = {c_hi.x, c_hi.y, c_hi.z, c_hi.w}, sh[4] = {s_hi.x, s_hi.y, s_hi.z, s_hi.w};
          float ol[8], oh[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float xl = __uint_as_float(lo[q * 8 + j]);
            float xh = __uint_as_float(hi[q * 8 + j]);
            bf16r2(xl, xh);
            float cosl = (j & 1) ? bf16_hi(cl[j >> 1]) : bf16_lo(cl[j >> 1]);
            float sinl = (j & 1) ? bf16_hi(sl[j >> 1]) : bf16_lo(sl[j >> 1]);
            float cosh_ = (j & 1) ? bf16_hi(ch[j >> 1]) : bf16_lo(ch[j >> 1]);
            float sinh_ = (j & 1) ? bf16_hi(sh[j >> 1]) : bf16_lo(sh[j >> 1]);
            float a0 = xl * cosl, a1 = -xh * sinl, b0 = xh * cosh_, b1 = xl * sinh_;
            bf16r2(a0, a1);
            bf16r2(b0, b1);
            ol[j] = a0 + a1;
            oh[j] = b0 + b1;
          }
          *reinterpret_cast<uint4*>(orow + c + q * 8) =
              make_uint4(pack_bf16(ol[0], ol[1]), pack_bf16(ol[2], ol[3]), pack_bf16(ol[4], ol[5]), pack_bf16(ol[6], ol[7]));
          *reinterpret_cast<uint4*>(orow + 64 + c + q * 8) =
              make_uint4(pack_bf16(oh[0], oh[1]), pack_bf16(oh[2], oh[3]), pack_bf16(oh[4], oh[5]), pack_bf16(oh[6], oh[7]));
        }
      }
    }
  }
}

// A HEADS tile without RoPE: the warpgroup's 64 staged rows (warpgroup cw), bias added, stored into the head-major buffers
// 16 bytes per thread, with consecutive threads on consecutive 8-column chunks of a row.  Each warp store then covers whole
// runs of two rows' heads; with one row per thread, every store hit 32 rows head_ld apart (a power-of-two stride), and the ViT
// q/k/v projection took twice as long as a plain linear of the same shape.  Arithmetic and rounding are unchanged.
template <int BN>
ARIA_DEVICE void heads_store_tile(const GemmParams& p, const float* stg, int cw, int m_idx, int n_idx, int row0, int rows) {
  constexpr int ACC_LD = acc_ld(BN), CH = BN / 8;
  const int col0 = n_idx * BN;
  const int seg = col0 / p.N;
  const int cseg0 = col0 - seg * p.N;
  const __nv_bfloat16* bias = p.bias[seg];
  __nv_bfloat16* out = p.out[seg];
#pragma unroll 1
  for (int i = threadIdx.x & 127; i < 64 * CH; i += 128) {
    const int r = cw * 64 + i / CH, c = (i % CH) * 8;
    const int r_in_grp = m_idx * BM + r;
    const int cs = cseg0 + c;  // column inside the segment
    if (r_in_grp >= rows || cs + 8 > p.N) continue;
    const float4 lo = *reinterpret_cast<const float4*>(stg + r * ACC_LD + c);
    const float4 hi = *reinterpret_cast<const float4*>(stg + r * ACC_LD + c + 4);
    float x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    if (bias) {
      const uint4 bv = __ldg(reinterpret_cast<const uint4*>(bias + cs));
      const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        x[2 * j] += bf16_lo(bw[j]);
        x[2 * j + 1] += bf16_hi(bw[j]);
      }
    }
    const int grow = row0 + r_in_grp;
    const int b = grow / p.rows_per_batch, tok = grow - b * p.rows_per_batch;
    const int head = cs / p.head_dim, d = cs - head * p.head_dim;
    *reinterpret_cast<uint4*>(out + b * p.stride_b + static_cast<int64_t>(p.pos0 + tok) * p.head_ld + head * p.stride_h + d) =
        make_uint4(pack_bf16(x[0], x[1]), pack_bf16(x[2], x[3]), pack_bf16(x[4], x[5]), pack_bf16(x[6], x[7]));
  }
}

// Scales applied to the fp32 accumulator as it is staged, before any rounding of the epilogue: none, per B column, or per A
// row and then per B column
enum class AccScale { NONE, COL, ROW_COL };

// The end of a consumer warpgroup's tile: stage its fp32 accumulator rows in `stg` ([BM][acc_ld(BN)]), scaled by the column
// scales `bsc` (load_col_scales) and the row scales of the fragment's two rows `as0` / `as1` as SCALE says, then run the
// epilogue on this thread's row (HEADS segments without RoPE: on the warpgroup's rows, heads_store_tile).
template <int BN, int EPI, AccScale SCALE>
ARIA_DEVICE void stage_and_epilogue(const GemmParams& p, float* stg, const ConsumerThread& ct, const float (&acc)[BN / 2],
                                    const float2 (&bsc)[BN / 8], float as0, float as1, int n_out_total, int grp, int m_idx,
                                    int n_idx, int row0, int rows) {
  constexpr int ACC_LD = acc_ld(BN);
  auto scaled = [](float a, float as, float bs) {
    if constexpr (SCALE == AccScale::ROW_COL) return a * as * bs;
    else if constexpr (SCALE == AccScale::COL) return a * bs;
    else return a;
  };
  named_bar_sync(1 + ct.cw, 128);  // the previous tile's epilogue has finished reading this warpgroup's staging rows
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    float* d0 = stg + ct.frag_row * ACC_LD + 8 * j + ct.frag_col;
    *reinterpret_cast<float2*>(d0) = make_float2(scaled(acc[4 * j], as0, bsc[j].x), scaled(acc[4 * j + 1], as0, bsc[j].y));
    *reinterpret_cast<float2*>(d0 + 8 * ACC_LD) =
        make_float2(scaled(acc[4 * j + 2], as1, bsc[j].x), scaled(acc[4 * j + 3], as1, bsc[j].y));
  }
  named_bar_sync(1 + ct.cw, 128);
  if constexpr (EPI == ARIA_EPI_HEADS) {
    if (!((p.rope_mask >> (n_idx * BN / p.N)) & 1)) {
      heads_store_tile<BN>(p, stg, ct.cw, m_idx, n_idx, row0, rows);
      return;
    }
  }
  const int r_in_grp = m_idx * BM + ct.epi_row;
  const bool row_ok = r_in_grp < rows;
  const int64_t grow = static_cast<int64_t>(row0) + r_in_grp;
  epilogue_tile<BN, EPI>(p, stg + ct.epi_row * ACC_LD, n_out_total, n_idx, grow, row_ok, ct.half, grp, r_in_grp);
}

}  // namespace aria
