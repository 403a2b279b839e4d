// Attention for sm_90a.
//
// aria_attention_fwd: flash-style forward with both contractions on wgmma tensor cores:
//     S = Q K^T   (A = Q tile, B = K tile, both K-major SW128 in shared memory, S accumulates in registers)
//     O += P V    (A = P, bf16, straight from the registers that held S; B = V tile consumed MN-major — V is [keys, d] with d
//                  contiguous, exactly the HF cache layout — O accumulates in registers)
//   warpgroup 0: TMA producer (Q once, K/V through a ring of separately released K and V slots); warpgroups 1-2: 64 query
//   rows each, fp32 online softmax on the fragments (four threads share a row: max / sum over two shuffles) and the final
//   normalise + store.  The two consumer warpgroups take turns issuing their wgmmas (ping-pong on named barriers), so one
//   runs its softmax while the other's products run; at HD = 80 each also issues S_{j+1} with PV_j before its softmax.
//   One CTA per (batch, head, 128 queries); causal launches visit the heaviest query tiles first.
// Replaces flash_attn_func / SDPA behind LLAMA_ATTENTION_CLASSES (aria/model/moe_lm.py:594) and the
// Idefics2 / nn.MultiheadAttention attention of the ViT + projector (vision_encoder.py:120, projector.py:93), whose
// 72-wide heads live in 128-wide rows: at HD = 80 only columns 0-79 of K and V are loaded (a 64-column SW128 box plus a
// 16-column SW32 box), QK contracts 80 columns (5 k-steps) and PV produces 80 (m64n64 + m64n16); out_hd of them are stored.
// Scores and softmax statistics stay fp32.  The running row max is raised lazily, only when it grows by more than 2^8: P then
// lies in [0, 256] and is rounded to bf16 at that scale, which measured closer to transformers' eager attention (the reference
// of the ViT path) than rounding P relative to the exact running max, and it skips most rescales of O.
//
// aria_attention_fwd_varlen: causal attention over sequences packed along one row (padding-free fine-tuning), on the
//   shared-prefix prefill's pipeline with no prefix; each sequence bit-identical to aria_attention_fwd_lse on it alone.
// aria_attention_prefill_paged_varlen: packed prompt segments, each after a paged prefix of its own (batched admission in the
//   serving engine); each segment bit-identical to aria_attention_prefill_paged_prefix on it alone.
//
// aria_attention_decode: single-query attention against the KV cache; HBM-bound, CUDA cores, split-KV.
// aria_attention_decode_devlen: the same kernels with the key count of each row read from device memory (graph replays).
// aria_attention_decode_paged: the devlen kernels over a paged KV cache (page pools and a block table, continuous batching).
// aria_attention_decode_fp8 / _devlen_fp8: the same split-KV kernels over an e4m3 KV cache with per-token scales.
// aria_attention_decode_paged_fp8: the fp8 kernels over e4m3 page pools with per-token scale pools (fp8 KV pages).
// aria_attention_decode_shared_prefix: n rows per prompt decode against one shared prompt cache plus their own tail caches.
// aria_attention_decode_multi: Q consecutive queries per row against its cache (prompt-lookup verification), each query
//   bit-identical to the devlen kernels.
#include <type_traits>

#include "common.cuh"
#include "fp8.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int AT_BM = 128;   // queries per CTA
constexpr int AT_BN = 128;   // keys per step
constexpr int AT_D = 128;    // head dim (row width of q / k / v)
constexpr int AT_TILE = AT_BM * AT_D * 2;  // 32 KB: the Q tile, and one K or V ring slot at HD = 128
constexpr int AT_HALF = AT_TILE / 2;       // one SW128 column chunk: [128 rows][64 bf16]
constexpr int AT_THREADS = 384;            // producer warpgroup + two consumer warpgroups
constexpr uint32_t AT_BAR_TURN = 1;        // named barriers 1, 2: consumer warpgroup 0 / 1 may issue its wgmmas

// Per head-dim layout.  HD = 128: a K (or V) ring slot is two SW128 column chunks.  HD = 80: the SW128 chunk of columns
// 0-63 plus a [128 keys][16] SW32 tile of columns 64-79, 20 KB instead of 32, which leaves room for a four-stage ring.
template <int HD>
struct AttnCfg {
  static constexpr int KV_TILE = HD == 80 ? AT_HALF + AT_BN * 32 : AT_TILE;
  static constexpr int STAGES = HD == 80 ? 4 : 2;
  static constexpr int NO = HD == 80 ? 80 : 128;  // output columns PV produces
  // S_{j+1} in flight during the softmax of block j needs a second score fragment; at HD = 128 it does not fit beside the
  // 64-register O without spills, so that path runs the ping-pong alone
  static constexpr bool INTRA = HD == 80;
  static constexpr int SMEM = 1024 + AT_TILE /*Q*/ + STAGES * 2 * KV_TILE /*K, V*/ + 256;
};

struct AttnParams {
  int B, H, Tq, Tk;
  int out_hd;
  float scale_log2;
  const uint8_t* key_mask;  // [B, Tk] 1 = masked out
  __nv_bfloat16* out;       // [B, Tq, H*out_hd]
  float* lse;               // [B, H, Tq] natural-log logsumexp of scale * q.k (LSE instantiations only)
  int n_q_tiles;
};

// Suffix prefill over a shared prefix (aria_attention_prefill_shared_prefix): the queries and the suffix keys are B segments
// packed along one sequence, segment b = rows [cu[b], cu[b + 1]); every query also sees the P keys of one prefix cache.
struct SharedPrefixParams {
  const int32_t* cu;  // [n_seg + 1] device segment starts
  int n_seg;
  int P;
};

// The key tiles of one 128-query tile [q0, q_end) of the shared-prefix prefill, in order: the prefix tiles at rows 128 j, then,
// for each segment present in the query tile, 128-key tiles aligned at the segment's start up to its last query in the tile.
// The producer and every consumer thread walk the same sequence, one tile per step.
struct SharedTileWalk {
  const int32_t* cu;
  int n_seg, n_pre, q_end;
  int b, c, e, t;   // current segment, its start / end, tile index inside it
  int k0, seg_c;    // the current tile: first key row (prefix or packed) and segment start (-1 for a prefix tile)

  __device__ __forceinline__ static int seg_tiles(int c, int e, int q_end) {
    return e > c ? (min(e, q_end) - 1 - c) / AT_BN + 1 : 0;
  }
  __device__ __forceinline__ void init(const SharedPrefixParams& sp, int q0, int q_end_) {
    cu = sp.cu;
    n_seg = sp.n_seg;
    n_pre = (sp.P + AT_BN - 1) / AT_BN;
    q_end = q_end_;
    b = packed_segment(cu, n_seg, q0);
    c = cu[b];
    e = cu[b + 1];
    t = -1;
  }
  // total tiles (prefix + suffix); reads the segment starts without moving the walk
  __device__ __forceinline__ int count() const {
    int n = n_pre, cc = c, ee = e, bb = b;
    while (bb < n_seg && cc < q_end) {
      n += seg_tiles(cc, ee, q_end);
      ++bb;
      cc = max(ee, cc);
      ee = bb < n_seg ? cu[bb + 1] : cc;
    }
    return n;
  }
  // move to tile j (called for j = 0, 1, 2, ... in order)
  __device__ __forceinline__ void step(int j) {
    if (j < n_pre) {
      k0 = j * AT_BN;
      seg_c = -1;
      return;
    }
    ++t;
    while (t >= seg_tiles(c, e, q_end) && b < n_seg) {
      ++b;
      c = max(e, c);
      e = b < n_seg ? cu[b + 1] : c;
      t = 0;
    }
    k0 = c + t * AT_BN;
    seg_c = c;
  }
};

// Prefill over a paged prefix (aria_attention_prefill_paged_prefix): the shared-prefix prefill whose prefix is P keys
// (a multiple of 256) held in pool pages, key 256 i + r at row r of page pages[i].
struct PagedPrefixParams {
  const int32_t* cu;     // [n_seg + 1] device segment starts of the packed suffixes
  int n_seg;
  int P;
  const int32_t* pages;  // [>= P / 256] device page list of the prefix
};

// Prefill of packed segments over paged prefixes of their own (aria_attention_prefill_paged_varlen): segment b is packed rows
// [cu[b], cu[b + 1]) and attends to its prefix_lens[b] keys (a multiple of 256) in pages page_table[b * table_stride + i].
struct PagedVarlenParams {
  const int32_t* cu;           // [n_seg + 1] device segment starts
  const int32_t* prefix_lens;  // [n_seg] device
  const int32_t* page_table;   // [n_seg, table_stride] device
  int64_t table_stride;
  int n_seg;
};

// HD = head dim contracted by QK^T (80 for the 72-wide ViT heads, 128 for the LM); LSE: also store the row logsumexp
// (what the backward needs to recompute P).  tmK16 / tmV16: 16-column SW32 boxes of columns 64-79 (HD = 80 only).
// SHARED (HD = 128): the shared-prefix suffix prefill; the keys walk the prefix (tmPK / tmPV, rows [0, sp.P)) and then the
// query tile's segments of the packed suffix (tmK / tmV), SharedTileWalk; a query sees the prefix and its own segment up to
// itself.  A key masked for a row adds exact zeros to that row, so each row's arithmetic is: the prefix tiles, then its own
// segment's tiles, whatever else shares its query tile.
// PAGED (with SHARED): tmPK / tmPV map a page pool [n_pages, H, 256, 128] and prefix tile j (keys 128 j ..) is rows
// 128 (j & 1) .. of page pages[j >> 1]; only the producer reads the page list.  The tiles, and so every row's arithmetic, are
// those of the contiguous prefix.
// SEGS (with PAGED): every segment has a prefix of its own (PagedVarlenParams).  Query tiles do not cross segments: the
// 128-query tiles of segment b are aligned at its start, and tile index q_tile counts the tiles of the segments before it, so
// a CTA is the CTA of the same tile in aria_attention_prefill_paged_prefix run on segment b alone (n_seg = 1, its P and page
// list) and computes the same arithmetic; the rows of its tile past the segment's end are not stored.  Tile indices past the
// last tile (the grid is sized for an upper bound) exit at once.
template <int HD, bool CAUSAL, bool LSE, bool SHARED, bool PAGED = false, bool SEGS = false>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                              const CUtensorMap& tmK16, const CUtensorMap& tmV16, const CUtensorMap& tmPK,
                                              const CUtensorMap& tmPV, const AttnParams& p, const SharedPrefixParams& sp,
                                              const int32_t* pages = nullptr, const PagedVarlenParams* vl = nullptr) {
  static_assert(!SHARED || (HD == 128 && !CAUSAL), "the shared-prefix prefill runs at head dim 128 with its own mask");
  static_assert(!PAGED || SHARED, "a paged prefix is a shared-prefix prefill");
  static_assert(!SEGS || (PAGED && !LSE), "per-segment prefixes are paged");
  constexpr int S = AttnCfg<HD>::STAGES, KVT = AttnCfg<HD>::KV_TILE, NO = AttnCfg<HD>::NO;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                            // [2 chunks][128 rows][64]
  uint8_t* sK = sQ + AT_TILE;                    // [STAGES][KV_TILE]
  uint8_t* sV = sK + S * KVT;                    // [STAGES][KV_TILE]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + S * KVT);
  uint64_t* q_full = bars;                       // [1]
  uint64_t* k_full = bars + 1;                   // [STAGES]
  uint64_t* v_full = k_full + S;                 // [STAGES]
  uint64_t* k_empty = v_full + S;                // [STAGES], one arrival per consumer warp
  uint64_t* v_empty = k_empty + S;               // [STAGES], one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int BH = p.B * p.H;
  const int bh = blockIdx.x % BH;
  const int q_tile = p.n_q_tiles - 1 - blockIdx.x / BH;  // heaviest (latest rows) first
  const int b = bh / p.H, h = bh % p.H;
  int q0 = q_tile * AT_BM;
  int q_stop = p.Tq;  // rows at or past q_stop are not stored
  [[maybe_unused]] SharedPrefixParams seg_sp{};
  [[maybe_unused]] const int32_t* seg_pages = pages;
  if constexpr (SEGS) {
    int sg = 0, t = q_tile, c = vl->cu[0], e = vl->cu[1];
    while (t >= (e - c + AT_BM - 1) / AT_BM) {
      t -= (e - c + AT_BM - 1) / AT_BM;
      if (++sg == vl->n_seg) return;  // past the last tile: the whole CTA leaves before any barrier
      c = e;
      e = vl->cu[sg + 1];
    }
    q0 = c + t * AT_BM;
    q_stop = min(q0 + AT_BM, e);
    seg_sp = SharedPrefixParams{vl->cu + sg, 1, vl->prefix_lens[sg]};
    seg_pages = vl->page_table + sg * vl->table_stride;
  }
  const SharedPrefixParams& spx = SEGS ? seg_sp : sp;
  const int pos_off = p.Tk - p.Tq;
  int n_kv = (p.Tk + AT_BN - 1) / AT_BN;
  if (CAUSAL) n_kv = min(n_kv, (pos_off + min(q0 + AT_BM, p.Tq) - 1) / AT_BN + 1);
  SharedTileWalk walk;
  if constexpr (SHARED) {
    walk.init(spx, q0, min(q0 + AT_BM, q_stop));
    n_kv = walk.count();
  }

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    if (HD == 80) {
      prefetch_tmap(&tmK16);
      prefetch_tmap(&tmV16);
    }
    mbar_init(q_full, 1);
    for (int i = 0; i < S; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 8);
      mbar_init(&v_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<24>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_full, AT_TILE);
      tma_load_4d(sQ, &tmQ, q_full, 0, q0, h, b);
      tma_load_4d(sQ + AT_HALF, &tmQ, q_full, 64, q0, h, b);
      // K slots are freed once both warpgroups hold S_j, V slots after PV_j: the K loads run ahead of the V loads
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % S;
        const uint32_t ph = ((j / S) & 1) ^ 1;
        if constexpr (SHARED) {
          walk.step(j);
          const CUtensorMap* mk = walk.seg_c < 0 ? &tmPK : &tmK;
          const CUtensorMap* mv = walk.seg_c < 0 ? &tmPV : &tmV;
          int row = walk.k0, page = 0;
          if constexpr (PAGED) {
            // an entry outside the pool is an out-of-bounds box: TMA fills it with zeros
            if (walk.seg_c < 0) {
              row = (j & 1) * AT_BN;
              page = seg_pages[j >> 1];
            }
          }
          mbar_wait(&k_empty[s], ph);
          mbar_arrive_expect_tx(&k_full[s], KVT);
          tma_load_4d(sK + s * KVT, mk, &k_full[s], 0, row, h, page);
          tma_load_4d(sK + s * KVT + AT_HALF, mk, &k_full[s], 64, row, h, page);
          mbar_wait(&v_empty[s], ph);
          mbar_arrive_expect_tx(&v_full[s], KVT);
          tma_load_4d(sV + s * KVT, mv, &v_full[s], 0, row, h, page);
          tma_load_4d(sV + s * KVT + AT_HALF, mv, &v_full[s], 64, row, h, page);
          continue;
        }
        mbar_wait(&k_empty[s], ph);
        mbar_arrive_expect_tx(&k_full[s], KVT);
        tma_load_4d(sK + s * KVT, &tmK, &k_full[s], 0, j * AT_BN, h, b);
        tma_load_4d(sK + s * KVT + AT_HALF, HD == 80 ? &tmK16 : &tmK, &k_full[s], 64, j * AT_BN, h, b);
        mbar_wait(&v_empty[s], ph);
        mbar_arrive_expect_tx(&v_full[s], KVT);
        tma_load_4d(sV + s * KVT, &tmV, &v_full[s], 0, j * AT_BN, h, b);
        tma_load_4d(sV + s * KVT + AT_HALF, HD == 80 ? &tmV16 : &tmV, &v_full[s], 64, j * AT_BN, h, b);
      }
    }
    return;
  }

  // =========================== consumer warpgroup cw: query rows [q0 + 64 cw, +64) ===========================
  // FlashAttention-3 schedule.  Inside a warpgroup, S_j = Q K_j^T is issued together with PV_{j-1}, and the softmax of block
  // j runs while PV_{j-1} is in flight.  Across the two warpgroups, named barriers hand the right to issue back and forth
  // (ping-pong), so one warpgroup's products run while the other does its softmax.
  setmaxnreg_inc<240>();
  const int cw = wg - 1;
  const int r_lo = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's two rows: r_lo and r_lo + 8
  const int qpos_lo = pos_off + r_lo, qpos_hi = qpos_lo + 8;
  const int kq = 2 * (lane & 3);                                  // key / column offset of this thread in an 8-wide block
  const uint8_t* km = p.key_mask ? p.key_mask + static_cast<int64_t>(b) * p.Tk : nullptr;
  int c_lo = 0, c_hi = 0;  // SHARED: segment starts of this thread's two rows
  if constexpr (SHARED) {
    c_lo = spx.cu[packed_segment(spx.cu, spx.n_seg, r_lo)];
    c_hi = spx.cu[packed_segment(spx.cu, spx.n_seg, r_lo + 8)];
  }
  const uint32_t sQa = smem_u32(sQ) + cw * 64 * 128, sKa = smem_u32(sK), sVa = smem_u32(sV);
  const uint32_t my_turn = AT_BAR_TURN + cw, other_turn = AT_BAR_TURN + (cw ^ 1);
  // K-major k-step kk (16 columns of the head): chunk kk / 4, +32 B per step inside the chunk
  auto kmaj_off = [](int kk) { return static_cast<uint32_t>((kk >> 2) * AT_HALF + (kk & 3) * 32); };

  float o[NO / 2];
#pragma unroll
  for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  float sc[64];       // scores of the newest block, then its P (fp32)
  uint32_t pa[8][4];  // P of the previous block as the A operand of PV: k-step kk = {row lo keys +0/+1, row hi, lo +8/+9, hi}
  float f_lo = 1.f, f_hi = 1.f;

  // S = Q K^T over the K tile in ring slot s.  HD = 80: k-steps 0-3 on the SW128 chunk, k-step 4 (columns 64-79) with K
  // from its SW32 tile; Q keeps both SW128 chunks.
  auto issue_qk = [&](int s) {
    const uint32_t kt = sKa + s * KVT;
    constexpr int KS = HD == 80 ? 4 : HD / 16;
#pragma unroll
    for (int kk = 0; kk < KS; ++kk)
      wgmma_m64n128_ss<0, 0>(sc, make_smem_desc(sQa + kmaj_off(kk), 16, 1024), make_smem_desc(kt + kmaj_off(kk), 16, 1024),
                             kk ? 1u : 0u);
    if constexpr (HD == 80)
      wgmma_m64n128_ss<0, 0>(sc, make_smem_desc(sQa + kmaj_off(4), 16, 1024), make_smem_desc_sw32(kt + AT_HALF, 256), 1u);
  };
  // O += P V over the V tile in ring slot s, V consumed MN-major.  HD = 128: m64n128 over both SW128 chunks (LBO = 16 KB
  // between them, SBO = 1024 per 8 keys, +2048 B per 16 keys).  HD = 80: m64n64 on the SW128 chunk (o[0..31]) and
  // m64n16 on the SW32 tile (o[32..39]; SBO = 256 per 8 keys, +512 B per 16 keys).
  auto issue_pv = [&](int s) {
    const uint32_t vt = sVa + s * KVT;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      if constexpr (HD == 80) {
        wgmma_m64n64_rs<1>(*reinterpret_cast<float(*)[32]>(&o[0]), pa[kk], make_smem_desc(vt + kk * 2048, AT_HALF, 1024));
        wgmma_m64n16_rs<1>(*reinterpret_cast<float(*)[8]>(&o[32]), pa[kk], make_smem_desc_sw32(vt + AT_HALF + kk * 512, 256));
      } else {
        wgmma_m64n128_rs<1>(o, pa[kk], make_smem_desc(vt + kk * 2048, AT_HALF, 1024));
      }
    }
  };
  auto release = [&](uint64_t* bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
  };
  // Online softmax of block j on sc, in place (sc becomes P in fp32).  Returns whether the row max was raised; O must then
  // be scaled by f_lo / f_hi before PV_j, which is done once PV_{j-1} has landed.
  auto softmax = [&](int j) -> bool {
    if constexpr (SHARED) {
      // prefix tile: -inf on rows at or past P; suffix tile: -inf unless the key is in the row's segment, at or before it
      const int k0 = walk.k0, sc_ = walk.seg_c;
      if (sc_ >= 0 || k0 + AT_BN > spx.P) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kc = k0 + 8 * jj + kq + e;
            if (sc_ < 0 ? kc >= spx.P : (sc_ != c_lo || kc > r_lo)) sc[4 * jj + e] = -INFINITY;
            if (sc_ < 0 ? kc >= spx.P : (sc_ != c_hi || kc > r_lo + 8)) sc[4 * jj + 2 + e] = -INFINITY;
          }
        }
      }
    } else {
      const int k0 = j * AT_BN;
      const bool need_mask = (k0 + AT_BN > p.Tk) || (CAUSAL && (k0 + AT_BN - 1 > pos_off + q0 + cw * 64)) || km != nullptr;
      if (need_mask) {  // rare path (diagonal / tail / padded keys): -inf on dead keys
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kc = k0 + 8 * jj + kq + e;
            const bool gone = kc >= p.Tk || (km && km[kc]);
            if (gone || (CAUSAL && kc > qpos_lo)) sc[4 * jj + e] = -INFINITY;
            if (gone || (CAUSAL && kc > qpos_hi)) sc[4 * jj + 2 + e] = -INFINITY;
          }
        }
      }
    }
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      mx_lo = fmaxf(mx_lo, fmaxf(sc[4 * jj], sc[4 * jj + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(sc[4 * jj + 2], sc[4 * jj + 3]));
    }
#pragma unroll
    for (int o_ = 1; o_ <= 2; o_ <<= 1) {
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, o_));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, o_));
    }
    // lazy max (see the header); the four threads of a row hold the same m and mx, so they take the same decision
    const float mc_lo = fmaxf(m_lo, mx_lo * p.scale_log2), mc_hi = fmaxf(m_hi, mx_hi * p.scale_log2);
    const bool up_lo = (mc_lo - m_lo > 8.0f) || (m_lo == -INFINITY && mc_lo > -INFINITY);
    const bool up_hi = (mc_hi - m_hi > 8.0f) || (m_hi == -INFINITY && mc_hi > -INFINITY);
    const bool rescale = __any_sync(0xffffffffu, up_lo || up_hi);
    if (rescale) {
      f_lo = !up_lo ? 1.f : (m_lo == -INFINITY ? 0.f : fast_ex2(m_lo - mc_lo));
      f_hi = !up_hi ? 1.f : (m_hi == -INFINITY ? 0.f : fast_ex2(m_hi - mc_hi));
      if (up_lo) m_lo = mc_lo;
      if (up_hi) m_hi = mc_hi;
      l_lo *= f_lo;
      l_hi *= f_hi;
    }
    const float neg_lo = (m_lo == -INFINITY) ? 0.f : -m_lo, neg_hi = (m_hi == -INFINITY) ? 0.f : -m_hi;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const bool hi = r & 1;
        const float x0 = fast_ex2(fmaf(sc[8 * kk + 2 * r], p.scale_log2, hi ? neg_hi : neg_lo));
        const float x1 = fast_ex2(fmaf(sc[8 * kk + 2 * r + 1], p.scale_log2, hi ? neg_hi : neg_lo));
        if (hi) l_hi += x0 + x1; else l_lo += x0 + x1;
        sc[8 * kk + 2 * r] = x0;
        sc[8 * kk + 2 * r + 1] = x1;
      }
    }
    return rescale;
  };
  auto rescale_o = [&]() {
#pragma unroll
    for (int jj = 0; jj < NO / 8; ++jj) {
      o[4 * jj] *= f_lo;
      o[4 * jj + 1] *= f_lo;
      o[4 * jj + 2] *= f_hi;
      o[4 * jj + 3] *= f_hi;
    }
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_bf16(sc[8 * kk + 2 * r], sc[8 * kk + 2 * r + 1]);
    }
  };

  mbar_wait(q_full, 0);
  if (cw == 1) named_bar_arrive(other_turn, 256);  // warpgroup 0 issues first

  if constexpr (!AttnCfg<HD>::INTRA) {
    // HD = 128: ping-pong only.  S_j and PV_j are issued in turns of their own and each is waited for before the next step.
    for (int j = 0; j < n_kv; ++j) {
      const int s = j % S;
      const uint32_t ph = (j / S) & 1;
      if constexpr (SHARED) walk.step(j);
      mbar_wait(&k_full[s], ph);
      named_bar_sync(my_turn, 256);
      wgmma_fence();
      issue_qk(s);
      wgmma_commit();
      named_bar_arrive(other_turn, 256);
      wgmma_wait<0>();
      fence_regs(sc);
      release(&k_empty[s]);
      if (softmax(j)) rescale_o();
      pack_p();
      mbar_wait(&v_full[s], ph);
      named_bar_sync(my_turn, 256);
      wgmma_fence();
      issue_pv(s);
      wgmma_commit();
      if (cw == 0 || j + 1 < n_kv) named_bar_arrive(other_turn, 256);  // warpgroup 1 issues last: no turn to hand back
      wgmma_wait<0>();
      fence_regs(o);
      release(&v_empty[s]);
    }
  } else {
    // block 0: S_0 alone (O is still zero, nothing to rescale)
    mbar_wait(&k_full[0], 0);
    named_bar_sync(my_turn, 256);
    wgmma_fence();
    issue_qk(0);
    wgmma_commit();
    named_bar_arrive(other_turn, 256);
    wgmma_wait<0>();
    fence_regs(sc);
    release(&k_empty[0]);
    softmax(0);
    pack_p();

    for (int j = 1; j < n_kv; ++j) {
      const int s = j % S, sp = (j - 1) % S;
      mbar_wait(&k_full[s], (j / S) & 1);
      mbar_wait(&v_full[sp], ((j - 1) / S) & 1);
      named_bar_sync(my_turn, 256);
      wgmma_fence();
      issue_qk(s);
      wgmma_commit();
      issue_pv(sp);
      wgmma_commit();
      named_bar_arrive(other_turn, 256);
      wgmma_wait<1>();  // S_j has landed, PV_{j-1} may still run
      fence_regs(sc);
      release(&k_empty[s]);
      const bool rescale = softmax(j);
      wgmma_wait<0>();
      fence_regs(o);
      fence_regs(sc);  // P_j is packed into pa only after PV_{j-1} has read the old pa
      release(&v_empty[sp]);
      if (rescale) rescale_o();
      pack_p();
    }

    // last block: PV alone
    {
      const int sp = (n_kv - 1) % S;
      mbar_wait(&v_full[sp], ((n_kv - 1) / S) & 1);
      named_bar_sync(my_turn, 256);
      wgmma_fence();
      issue_pv(sp);
      wgmma_commit();
      if (cw == 0) named_bar_arrive(other_turn, 256);  // warpgroup 1 issues last: there is no turn left to hand back
      wgmma_wait<0>();
      fence_regs(o);
      release(&v_empty[sp]);
    }
  }

#pragma unroll
  for (int o_ = 1; o_ <= 2; o_ <<= 1) {
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, o_);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, o_);
  }
  if constexpr (LSE) {
    // sum_k 2^(s_k - m) = l for ANY m (the lazy max included), so log2-sum-exp2 = m + log2 l; -inf for a row that sees no key
    if ((lane & 3) == 0) {
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int q = r_lo + 8 * hrow;
        const float l = hrow ? l_hi : l_lo, m = hrow ? m_hi : m_lo;
        if (q < p.Tq) p.lse[static_cast<int64_t>(bh) * p.Tq + q] = l > 0.f ? (m + log2f(l)) * 0.6931471805599453f : -INFINITY;
      }
    }
  }
  const int64_t ld = static_cast<int64_t>(p.H) * p.out_hd;
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int q = r_lo + 8 * hrow;
    if (q >= q_stop) continue;
    const float l = hrow ? l_hi : l_lo;
    const float inv_l = l > 0.f ? 1.0f / l : 0.f;
    __nv_bfloat16* orow = p.out + (static_cast<int64_t>(b) * p.Tq + q) * ld + h * p.out_hd;
#pragma unroll
    for (int jj = 0; jj < NO / 8; ++jj) {
      if (8 * jj < p.out_hd)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + kq) = pack_bf16(o[4 * jj + 2 * hrow] * inv_l, o[4 * jj + 2 * hrow + 1] * inv_l);
    }
  }
}

template <int HD, bool CAUSAL, bool LSE>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmK16,
                const __grid_constant__ CUtensorMap tmV16, const AttnParams p) {
  attn_fwd_body<HD, CAUSAL, LSE, false>(tmQ, tmK, tmV, tmK16, tmV16, tmK, tmV, p, SharedPrefixParams{});
}

// One CTA per (head, 128 packed queries): tmQ / tmK / tmV map the packed suffix [1, H, S_tot, 128], tmPK / tmPV the prefix
// cache [1, H, P, 128] (rows past P are outside the map: never read).  With P = 0 this is the varlen causal forward
// (aria_attention_fwd_varlen): every key tile is aligned at its segment's start; LSE adds the logsumexp store [H, S_tot].
template <bool LSE>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_prefill_shared_prefix_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                  const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmPK,
                                  const __grid_constant__ CUtensorMap tmPV, const AttnParams p, const SharedPrefixParams sp) {
  attn_fwd_body<128, false, LSE, true>(tmQ, tmK, tmV, tmK, tmV, tmPK, tmPV, p, sp);
}

// One CTA per (head, 128 packed queries): tmQ / tmK / tmV map the packed suffix [1, H, S_tot, 128] as above, tmPK / tmPV the
// layer's page pools [n_pages, H, 256, 128].
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_prefill_paged_prefix_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmPK,
                                 const __grid_constant__ CUtensorMap tmPV, const AttnParams p, const PagedPrefixParams pp) {
  attn_fwd_body<128, false, false, true, true>(tmQ, tmK, tmV, tmK, tmV, tmPK, tmPV, p, SharedPrefixParams{pp.cu, pp.n_seg, pp.P},
                                               pp.pages);
}

// One CTA per (head, query tile of one segment): tmQ / tmK / tmV map the packed rows [1, H, S_tot, 128], tmPK / tmPV the
// layer's page pools [n_pages, H, 256, 128]; p.n_q_tiles bounds the segments' tile count.
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_prefill_paged_varlen_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmPK,
                                 const __grid_constant__ CUtensorMap tmPV, const AttnParams p, const PagedVarlenParams vl) {
  attn_fwd_body<128, false, false, true, true, true>(tmQ, tmK, tmV, tmK, tmV, tmPK, tmPV, p, SharedPrefixParams{}, nullptr, &vl);
}

// ------------------------------------------------------------------------------------------------
// Decode: one query per (b,h); block = 4 warps over a contiguous chunk of keys; each lane owns 4 dims.
// Partial (m, l, acc[128]) per (b,h,split) -> workspace; a second kernel merges the splits.
// DEVLEN: the key count of row b is the device value lens[b] (at most Tk = T_max, the cache rows the grid is sized for) and
// the key mask has the row stride mask_stride.  A split that starts past lens[b] sees no key and writes (m = -inf, l = 0,
// acc = 0); the merge reads the first ceil(lens[b] / DEC_SPLIT_KEYS) splits only, so row b is bit-identical to the host-length
// launch with Tk = lens[b].
// KV_FP8: k / v are e4m3 codes [B, H, T_max, 128] with one fp32 scale per (row, head, token) at k_scale / v_scale (strides
// sc_stride_b / sc_stride_h).  A lane widens its 4 codes per key exactly; the key scale multiplies the reduced dot product and
// the value weight is pw * v_scale.  Split size, warp -> key assignment and update order are the bf16 kernel's, so with
// power-of-two scales (both products exact) the result is bit-identical to the bf16 kernel run on the tensors code * scale.
// PAGED (with DEVLEN): kc / vc are page pools [n_pages, H, DEC_SPLIT_KEYS, 128] (kv_stride_b is the page stride) and
// split s of row b reads page block_table[b * bt_stride + s], which holds the row's keys [256 s, 256 s + 256).  A page is one
// split, so every key is read by the warp, and updated in the order, of the contiguous kernel: row b is bit-identical to
// the DEVLEN kernel on a cache that holds the same keys.  A live split whose entry is not a page of the pool reads no key.
// With KV_FP8 the scales are pools [n_pages, H, DEC_SPLIT_KEYS] too (sc_stride_b is their page stride), read from the same page.
constexpr int DEC_SPLIT_KEYS = 256;

template <bool DEVLEN, bool KV_FP8, bool PAGED = false, typename KV = std::conditional_t<KV_FP8, uint8_t, __nv_bfloat16>>
__device__ __forceinline__ void decode_partial(const __nv_bfloat16* __restrict__ q, const KV* __restrict__ kc,
                                               const KV* __restrict__ vc, const float* __restrict__ k_scale,
                                               const float* __restrict__ v_scale, const uint8_t* __restrict__ key_mask,
                                               float* __restrict__ ws, int H, int Tk, int64_t q_stride_b, int64_t q_stride_h,
                                               int64_t kv_stride_b, int64_t kv_stride_h, int64_t sc_stride_b, int64_t sc_stride_h,
                                               float scale_log2, int splits, const int32_t* __restrict__ lens, int mask_stride,
                                               const int32_t* __restrict__ block_table = nullptr, int64_t bt_stride = 0,
                                               int n_pages = 0) {
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / H, h = bh % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int len = DEVLEN ? min(lens[b], Tk) : Tk;
  const int k_begin = split * DEC_SPLIT_KEYS;
  int k_end = min(len, k_begin + DEC_SPLIT_KEYS);
  const KV* kbase;
  const KV* vbase;
  [[maybe_unused]] int page = 0;
  if constexpr (PAGED) {
    page = k_begin < k_end ? block_table[b * bt_stride + split] : 0;
    if (page < 0 || page >= n_pages) k_end = k_begin;
    // key kk of the split is row kk - k_begin of its page
    const int64_t off = static_cast<int64_t>(page) * kv_stride_b + h * kv_stride_h - static_cast<int64_t>(k_begin) * AT_D;
    kbase = kc + off;
    vbase = vc + off;
  } else {
    kbase = kc + b * kv_stride_b + h * kv_stride_h;
    vbase = vc + b * kv_stride_b + h * kv_stride_h;
  }
  const uint8_t* km = key_mask ? key_mask + static_cast<int64_t>(b) * (DEVLEN ? mask_stride : Tk) : nullptr;
  const uint2 qv = *reinterpret_cast<const uint2*>(q + b * q_stride_b + h * q_stride_h + lane * 4);
  const float q0 = bf16_lo(qv.x) * scale_log2, q1 = bf16_hi(qv.x) * scale_log2, q2 = bf16_lo(qv.y) * scale_log2,
              q3 = bf16_hi(qv.y) * scale_log2;
  float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if constexpr (!KV_FP8) {
    for (int k0 = k_begin + warp * 4; k0 < k_end; k0 += 16) {
      float s[4];
      uint2 vv[4];
      bool live[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k0 + u;
        live[u] = kk < k_end && !(km && km[kk]);
        if (live[u]) {
          const uint2 kv = __ldg(reinterpret_cast<const uint2*>(kbase + static_cast<int64_t>(kk) * AT_D + lane * 4));
          vv[u] = __ldg(reinterpret_cast<const uint2*>(vbase + static_cast<int64_t>(kk) * AT_D + lane * 4));
          s[u] = q0 * bf16_lo(kv.x) + q1 * bf16_hi(kv.x) + q2 * bf16_lo(kv.y) + q3 * bf16_hi(kv.y);
        } else {
          s[u] = 0.f;
          vv[u] = make_uint2(0, 0);
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (live[u]) {
          const float m_new = fmaxf(m, s[u]);
          const float f = exp2f(m - m_new), pw = exp2f(s[u] - m_new);
          l = l * f + pw;
          a0 = a0 * f + pw * bf16_lo(vv[u].x);
          a1 = a1 * f + pw * bf16_hi(vv[u].x);
          a2 = a2 * f + pw * bf16_lo(vv[u].y);
          a3 = a3 * f + pw * bf16_hi(vv[u].y);
          m = m_new;
        }
      }
    }
  } else {
    const float* ksb;
    const float* vsb;
    if constexpr (PAGED) {  // the scale of key kk is entry kk - k_begin of its page's scale rows
      const int64_t off = static_cast<int64_t>(page) * sc_stride_b + h * sc_stride_h - k_begin;
      ksb = k_scale + off;
      vsb = v_scale + off;
    } else {
      ksb = k_scale + b * sc_stride_b + h * sc_stride_h;
      vsb = v_scale + b * sc_stride_b + h * sc_stride_h;
    }
    // A lane reads 4 + 4 bytes per key, half of what the bf16 loop reads, so the loads of step k0 + 16 are issued before the
    // arithmetic of step k0 to keep as many bytes in flight per warp.
    uint32_t kn[4], vn[4];
    float ksn[4], vsn[4];
    bool ln[4];
    auto load = [&](int k0) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k0 + u;
        ln[u] = kk < k_end && !(km && km[kk]);
        if (ln[u]) {
          kn[u] = __ldg(reinterpret_cast<const uint32_t*>(kbase + static_cast<int64_t>(kk) * AT_D + lane * 4));
          vn[u] = __ldg(reinterpret_cast<const uint32_t*>(vbase + static_cast<int64_t>(kk) * AT_D + lane * 4));
          ksn[u] = __ldg(ksb + kk);
          vsn[u] = __ldg(vsb + kk);
        } else {
          kn[u] = vn[u] = 0u;
          ksn[u] = vsn[u] = 0.f;
        }
      }
    };
    load(k_begin + warp * 4);
    for (int k0 = k_begin + warp * 4; k0 < k_end; k0 += 16) {
      uint32_t kq[4], vq[4];
      float ks[4], vs[4], s[4];
      bool live[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        kq[u] = kn[u];
        vq[u] = vn[u];
        ks[u] = ksn[u];
        vs[u] = vsn[u];
        live[u] = ln[u];
      }
      load(k0 + 16);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (live[u]) {
          const float4 c = e4m3x4_to_float4(kq[u]);
          s[u] = q0 * c.x + q1 * c.y + q2 * c.z + q3 * c.w;
        } else {
          s[u] = 0.f;
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (live[u]) {
          const float su = s[u] * ks[u];
          const float m_new = fmaxf(m, su);
          const float f = exp2f(m - m_new), pw = exp2f(su - m_new);
          const float pv = pw * vs[u];
          const float4 c = e4m3x4_to_float4(vq[u]);
          l = l * f + pw;
          a0 = a0 * f + pv * c.x;
          a1 = a1 * f + pv * c.y;
          a2 = a2 * f + pv * c.z;
          a3 = a3 * f + pv * c.w;
          m = m_new;
        }
      }
    }
  }
  // merge the 4 warps through shared memory
  __shared__ float sm_m[4], sm_l[4], sm_a[4][AT_D];
  if (lane == 0) {
    sm_m[warp] = m;
    sm_l[warp] = l;
  }
  sm_a[warp][lane * 4 + 0] = a0;
  sm_a[warp][lane * 4 + 1] = a1;
  sm_a[warp][lane * 4 + 2] = a2;
  sm_a[warp][lane * 4 + 3] = a3;
  __syncthreads();
  const int d = threadIdx.x;  // 128 threads = 128 dims
  float M = fmaxf(fmaxf(sm_m[0], sm_m[1]), fmaxf(sm_m[2], sm_m[3]));
  float L = 0.f, A = 0.f;
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const float f = (sm_m[w] == -INFINITY) ? 0.f : exp2f(sm_m[w] - M);
    L += sm_l[w] * f;
    A += sm_a[w][d] * f;
  }
  float* o = ws + (static_cast<int64_t>(bh) * splits + split) * (AT_D + 2);
  o[d] = A;
  if (d == 0) {
    o[AT_D] = M;
    o[AT_D + 1] = L;
  }
}

template <bool DEVLEN>
__global__ void __launch_bounds__(128) attn_decode_partial(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                                                           const __nv_bfloat16* __restrict__ vc, const uint8_t* __restrict__ key_mask,
                                                           float* __restrict__ ws, int H, int Tk,
                                                           int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b,
                                                           int64_t kv_stride_h, float scale_log2, int splits,
                                                           const int32_t* __restrict__ lens, int mask_stride) {
  decode_partial<DEVLEN, false>(q, kc, vc, nullptr, nullptr, key_mask, ws, H, Tk, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, 0,
                                0, scale_log2, splits, lens, mask_stride);
}

template <bool DEVLEN>
__global__ void __launch_bounds__(128) attn_decode_partial_fp8(const __nv_bfloat16* __restrict__ q, const uint8_t* __restrict__ kc,
                                                               const uint8_t* __restrict__ vc, const float* __restrict__ k_scale,
                                                               const float* __restrict__ v_scale, const uint8_t* __restrict__ key_mask,
                                                               float* __restrict__ ws, int H, int Tk, int64_t q_stride_b,
                                                               int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h,
                                                               int64_t sc_stride_b, int64_t sc_stride_h, float scale_log2, int splits,
                                                               const int32_t* __restrict__ lens, int mask_stride) {
  decode_partial<DEVLEN, true>(q, kc, vc, k_scale, v_scale, key_mask, ws, H, Tk, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h,
                               sc_stride_b, sc_stride_h, scale_log2, splits, lens, mask_stride);
}

__global__ void __launch_bounds__(128) attn_decode_partial_paged(const __nv_bfloat16* __restrict__ q,
                                                                 const __nv_bfloat16* __restrict__ k_pool,
                                                                 const __nv_bfloat16* __restrict__ v_pool, float* __restrict__ ws,
                                                                 int H, int Tk, int64_t q_stride_b, int64_t q_stride_h,
                                                                 int64_t page_stride, int64_t pool_stride_h, float scale_log2,
                                                                 int splits, const int32_t* __restrict__ lens,
                                                                 const int32_t* __restrict__ block_table, int64_t bt_stride,
                                                                 int n_pages) {
  decode_partial<true, false, true>(q, k_pool, v_pool, nullptr, nullptr, nullptr, ws, H, Tk, q_stride_b, q_stride_h, page_stride,
                                    pool_stride_h, 0, 0, scale_log2, splits, lens, 0, block_table, bt_stride, n_pages);
}

__global__ void __launch_bounds__(128) attn_decode_partial_paged_fp8(
    const __nv_bfloat16* __restrict__ q, const uint8_t* __restrict__ k_pool, const uint8_t* __restrict__ v_pool,
    const float* __restrict__ k_scale, const float* __restrict__ v_scale, float* __restrict__ ws, int H, int Tk, int64_t q_stride_b,
    int64_t q_stride_h, int64_t page_stride, int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h,
    float scale_log2, int splits, const int32_t* __restrict__ lens, const int32_t* __restrict__ block_table, int64_t bt_stride,
    int n_pages) {
  decode_partial<true, true, true>(q, k_pool, v_pool, k_scale, v_scale, nullptr, ws, H, Tk, q_stride_b, q_stride_h, page_stride,
                                   pool_stride_h, scale_page_stride, scale_stride_h, scale_log2, splits, lens, 0, block_table,
                                   bt_stride, n_pages);
}

template <bool DEVLEN>
__global__ void __launch_bounds__(128) attn_decode_merge(const float* __restrict__ ws, __nv_bfloat16* __restrict__ out, int splits,
                                                         const int32_t* __restrict__ lens, int H) {
  const int bh = blockIdx.x, d = threadIdx.x;
  const float* base = ws + static_cast<int64_t>(bh) * splits * (AT_D + 2);
  const int n = DEVLEN ? min(splits, (lens[bh / H] + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS) : splits;
  float M = -INFINITY;
  for (int s = 0; s < n; ++s) M = fmaxf(M, base[s * (AT_D + 2) + AT_D]);
  float L = 0.f, A = 0.f;
  for (int s = 0; s < n; ++s) {
    const float ms = base[s * (AT_D + 2) + AT_D];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
    L += base[s * (AT_D + 2) + AT_D + 1] * f;
    A += base[s * (AT_D + 2) + d] * f;
  }
  out[static_cast<int64_t>(bh) * AT_D + d] = __float2bfloat16_rn(L > 0.f ? A / L : 0.f);
}

// ------------------------------------------------------------------------------------------------
// Shared-prefix decode: R = G * n rows, row r = g * n + j, attend to the prompt cache of group g (prefix, [G, H, P_max, 128])
// and then to their own generated rows (tail, [R, H, N_max, 128]).  Row r is bit-identical to the DEVLEN kernels run on the
// expanded layout: a cache of row r holding the prefix at [0, P_g), masked rows up to S_g = 256 * ceil(P_g / 256) and the tail
// at [S_g, S_g + tail_len).  That is because every 256-key split of the expanded row is computed here with the same keys, key
// order and arithmetic:
//   - prefix splits by attn_decode_prefix_partial, one CTA per (group, head, split), which stages the split's K and V in shared
//     memory once and runs decode_partial's loop for each of the group's n queries (warp -> key k_begin + 4 warp + 16 i + u, the
//     same per-key update and the same 4-warp merge), one 4-warp team per query;
//   - tail splits by the unchanged attn_decode_partial<true> on the tail cache, with lens = tail_lens;
//   - attn_decode_merge_shared reads the live prefix splits, then the live tail splits, in the order attn_decode_merge reads
//     the expanded row's splits.
// Each prompt key and value is read from HBM once per (group, head) and step instead of n times.
constexpr int SP_TEAMS = 8;                                 // 4-warp teams per prefix CTA
constexpr int SP_SMEM = 2 * DEC_SPLIT_KEYS * AT_D * 2;      // K and V of one split: 128 KB

// decode_partial<DEVLEN, bf16>'s loop and 4-warp merge for one query over keys [k_begin, k_end), run by one 4-warp team with
// the split's K and V staged in shared memory (rows from k_begin); the partial (acc[128], m, l) goes to o.  Named barrier
// 1 + team holds the team's 128 threads.  This is attn_decode_prefix_partial's per-query body; that kernel keeps its own copy
// so that its code stays as it was compiled before.
__device__ __forceinline__ void decode_team_split(const __nv_bfloat16* __restrict__ qp, const __nv_bfloat16* sKb,
                                                  const __nv_bfloat16* sVb, const uint8_t* __restrict__ km, int k_begin, int k_end,
                                                  float scale_log2, int team, float (*sm_m)[4], float (*sm_l)[4],
                                                  float (*sm_a)[4][AT_D], float* __restrict__ o) {
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const uint2 qv = *reinterpret_cast<const uint2*>(qp + lane * 4);
  const float q0 = bf16_lo(qv.x) * scale_log2, q1 = bf16_hi(qv.x) * scale_log2, q2 = bf16_lo(qv.y) * scale_log2,
              q3 = bf16_hi(qv.y) * scale_log2;
  float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int k0 = k_begin + warp * 4; k0 < k_end; k0 += 16) {
    float s[4];
    uint2 vv[4];
    bool live[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int kk = k0 + u;
      live[u] = kk < k_end && !(km && km[kk]);
      if (live[u]) {
        const uint2 kv = *reinterpret_cast<const uint2*>(sKb + (kk - k_begin) * AT_D + lane * 4);
        vv[u] = *reinterpret_cast<const uint2*>(sVb + (kk - k_begin) * AT_D + lane * 4);
        s[u] = q0 * bf16_lo(kv.x) + q1 * bf16_hi(kv.x) + q2 * bf16_lo(kv.y) + q3 * bf16_hi(kv.y);
      } else {
        s[u] = 0.f;
        vv[u] = make_uint2(0, 0);
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
#pragma unroll
      for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (live[u]) {
        const float m_new = fmaxf(m, s[u]);
        const float f = exp2f(m - m_new), pw = exp2f(s[u] - m_new);
        l = l * f + pw;
        a0 = a0 * f + pw * bf16_lo(vv[u].x);
        a1 = a1 * f + pw * bf16_hi(vv[u].x);
        a2 = a2 * f + pw * bf16_lo(vv[u].y);
        a3 = a3 * f + pw * bf16_hi(vv[u].y);
        m = m_new;
      }
    }
  }
  // the team's 4-warp merge, as decode_partial's
  if (lane == 0) {
    sm_m[team][warp] = m;
    sm_l[team][warp] = l;
  }
  sm_a[team][warp][lane * 4 + 0] = a0;
  sm_a[team][warp][lane * 4 + 1] = a1;
  sm_a[team][warp][lane * 4 + 2] = a2;
  sm_a[team][warp][lane * 4 + 3] = a3;
  named_bar_sync(1 + team, 128);
  const int d = threadIdx.x & 127;
  float M = fmaxf(fmaxf(sm_m[team][0], sm_m[team][1]), fmaxf(sm_m[team][2], sm_m[team][3]));
  float L = 0.f, A = 0.f;
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const float f = (sm_m[team][w] == -INFINITY) ? 0.f : exp2f(sm_m[team][w] - M);
    L += sm_l[team][w] * f;
    A += sm_a[team][w][d] * f;
  }
  o[d] = A;
  if (d == 0) {
    o[AT_D] = M;
    o[AT_D + 1] = L;
  }
  named_bar_sync(1 + team, 128);  // the team's next query overwrites sm_*
}

__global__ void __launch_bounds__(128 * SP_TEAMS, 1)
attn_decode_prefix_partial(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                           const __nv_bfloat16* __restrict__ vc, const int32_t* __restrict__ prefix_lens,
                           const uint8_t* __restrict__ key_mask, int mask_stride, float* __restrict__ ws, int n, int H, int P_max,
                           int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, float scale_log2,
                           int splits) {
  extern __shared__ uint4 sp_smem[];
  uint4* sK = sp_smem;                                      // [256 keys][16 x 16 B]
  uint4* sV = sp_smem + DEC_SPLIT_KEYS * (AT_D / 8);
  __shared__ float sm_m[SP_TEAMS][4], sm_l[SP_TEAMS][4], sm_a[SP_TEAMS][4][AT_D];
  const int gh = blockIdx.x, split = blockIdx.y;
  const int g = gh / H, h = gh % H;
  const int len = min(prefix_lens[g], P_max);
  const int k_begin = split * DEC_SPLIT_KEYS, k_end = min(len, k_begin + DEC_SPLIT_KEYS);
  const __nv_bfloat16* kbase = kc + g * kv_stride_b + h * kv_stride_h;
  const __nv_bfloat16* vbase = vc + g * kv_stride_b + h * kv_stride_h;
  const uint8_t* km = key_mask ? key_mask + static_cast<int64_t>(g) * mask_stride : nullptr;
  // stage the live keys of the split; masked keys and rows at or past the prefix length are never read
  for (int i = threadIdx.x; i < (k_end - k_begin) * (AT_D / 8); i += blockDim.x) {
    const int kk = k_begin + i / (AT_D / 8), c = i % (AT_D / 8);
    if (km && km[kk]) continue;
    sK[i] = __ldg(reinterpret_cast<const uint4*>(kbase + static_cast<int64_t>(kk) * AT_D) + c);
    sV[i] = __ldg(reinterpret_cast<const uint4*>(vbase + static_cast<int64_t>(kk) * AT_D) + c);
  }
  __syncthreads();
  const int team = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const __nv_bfloat16* sKb = reinterpret_cast<const __nv_bfloat16*>(sK);
  const __nv_bfloat16* sVb = reinterpret_cast<const __nv_bfloat16*>(sV);
  for (int j = team; j < n; j += SP_TEAMS) {
    const int r = g * n + j;
    // decode_partial<DEVLEN, bf16> for row r over keys [k_begin, k_end), with K and V from shared memory
    const uint2 qv = *reinterpret_cast<const uint2*>(q + r * q_stride_b + h * q_stride_h + lane * 4);
    const float q0 = bf16_lo(qv.x) * scale_log2, q1 = bf16_hi(qv.x) * scale_log2, q2 = bf16_lo(qv.y) * scale_log2,
                q3 = bf16_hi(qv.y) * scale_log2;
    float m = -INFINITY, l = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int k0 = k_begin + warp * 4; k0 < k_end; k0 += 16) {
      float s[4];
      uint2 vv[4];
      bool live[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k0 + u;
        live[u] = kk < k_end && !(km && km[kk]);
        if (live[u]) {
          const uint2 kv = *reinterpret_cast<const uint2*>(sKb + (kk - k_begin) * AT_D + lane * 4);
          vv[u] = *reinterpret_cast<const uint2*>(sVb + (kk - k_begin) * AT_D + lane * 4);
          s[u] = q0 * bf16_lo(kv.x) + q1 * bf16_hi(kv.x) + q2 * bf16_lo(kv.y) + q3 * bf16_hi(kv.y);
        } else {
          s[u] = 0.f;
          vv[u] = make_uint2(0, 0);
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (live[u]) {
          const float m_new = fmaxf(m, s[u]);
          const float f = exp2f(m - m_new), pw = exp2f(s[u] - m_new);
          l = l * f + pw;
          a0 = a0 * f + pw * bf16_lo(vv[u].x);
          a1 = a1 * f + pw * bf16_hi(vv[u].x);
          a2 = a2 * f + pw * bf16_lo(vv[u].y);
          a3 = a3 * f + pw * bf16_hi(vv[u].y);
          m = m_new;
        }
      }
    }
    // the team's 4-warp merge, as decode_partial's; named barrier 1 + team holds the team's 128 threads
    if (lane == 0) {
      sm_m[team][warp] = m;
      sm_l[team][warp] = l;
    }
    sm_a[team][warp][lane * 4 + 0] = a0;
    sm_a[team][warp][lane * 4 + 1] = a1;
    sm_a[team][warp][lane * 4 + 2] = a2;
    sm_a[team][warp][lane * 4 + 3] = a3;
    named_bar_sync(1 + team, 128);
    const int d = threadIdx.x & 127;
    float M = fmaxf(fmaxf(sm_m[team][0], sm_m[team][1]), fmaxf(sm_m[team][2], sm_m[team][3]));
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float f = (sm_m[team][w] == -INFINITY) ? 0.f : exp2f(sm_m[team][w] - M);
      L += sm_l[team][w] * f;
      A += sm_a[team][w][d] * f;
    }
    float* o = ws + ((static_cast<int64_t>(r) * H + h) * splits + split) * (AT_D + 2);
    o[d] = A;
    if (d == 0) {
      o[AT_D] = M;
      o[AT_D + 1] = L;
    }
    named_bar_sync(1 + team, 128);  // the team's next query overwrites sm_*
  }
}

// Multi-query decode (prompt-lookup verification): Q queries per (row, head), query i of row b at device key count
// lens[b * Q + i] (the row's queries are consecutive tokens, so their counts are consecutive).  One CTA per (row, head, 256-key
// split) stages the live keys of the split once for all Q queries, and min(Q, SP_TEAMS) 4-warp teams run decode_team_split per
// query: the key assignment, per-key update and 4-warp merge of decode_partial<DEVLEN>.  attn_decode_merge<true> then merges
// each query's live splits with lens, so query i of row b is bit-identical to aria_attention_decode_devlen at lens[b * Q + i].
__global__ void __launch_bounds__(128 * SP_TEAMS, 1)
attn_decode_multi_partial(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                          const __nv_bfloat16* __restrict__ vc, const int32_t* __restrict__ lens,
                          const uint8_t* __restrict__ key_mask, int mask_stride, float* __restrict__ ws, int Q, int H, int T_max,
                          int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_q, int64_t kv_stride_b, int64_t kv_stride_h,
                          float scale_log2, int splits) {
  extern __shared__ uint4 sp_smem[];
  uint4* sK = sp_smem;
  uint4* sV = sp_smem + DEC_SPLIT_KEYS * (AT_D / 8);
  __shared__ float sm_m[SP_TEAMS][4], sm_l[SP_TEAMS][4], sm_a[SP_TEAMS][4][AT_D];
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / H, h = bh % H;
  int len_max = 0;
  for (int i = 0; i < Q; ++i) len_max = max(len_max, min(lens[b * Q + i], T_max));
  const int k_begin = split * DEC_SPLIT_KEYS, k_stage = min(len_max, k_begin + DEC_SPLIT_KEYS);
  const __nv_bfloat16* kbase = kc + b * kv_stride_b + h * kv_stride_h;
  const __nv_bfloat16* vbase = vc + b * kv_stride_b + h * kv_stride_h;
  const uint8_t* km = key_mask ? key_mask + static_cast<int64_t>(b) * mask_stride : nullptr;
  for (int i = threadIdx.x; i < (k_stage - k_begin) * (AT_D / 8); i += blockDim.x) {
    const int kk = k_begin + i / (AT_D / 8), c = i % (AT_D / 8);
    if (km && km[kk]) continue;
    sK[i] = __ldg(reinterpret_cast<const uint4*>(kbase + static_cast<int64_t>(kk) * AT_D) + c);
    sV[i] = __ldg(reinterpret_cast<const uint4*>(vbase + static_cast<int64_t>(kk) * AT_D) + c);
  }
  __syncthreads();
  const int team = threadIdx.x >> 7, n_teams = blockDim.x >> 7;
  for (int i = team; i < Q; i += n_teams) {
    const int k_end = min(min(lens[b * Q + i], T_max), k_begin + DEC_SPLIT_KEYS);
    decode_team_split(q + b * q_stride_b + h * q_stride_h + i * q_stride_q, reinterpret_cast<const __nv_bfloat16*>(sK),
                      reinterpret_cast<const __nv_bfloat16*>(sV), km, k_begin, k_end, scale_log2, team, sm_m, sm_l, sm_a,
                      ws + ((static_cast<int64_t>(b * Q + i) * H + h) * splits + split) * (AT_D + 2));
  }
}

// attn_decode_merge over the prefix splits, then the tail splits, of row r = blockIdx.x / H
__global__ void __launch_bounds__(128) attn_decode_merge_shared(const float* __restrict__ ws_prefix, const float* __restrict__ ws_tail,
                                                                __nv_bfloat16* __restrict__ out, int prefix_splits, int tail_splits,
                                                                const int32_t* __restrict__ prefix_lens,
                                                                const int32_t* __restrict__ tail_lens, int n, int H) {
  const int rh = blockIdx.x, d = threadIdx.x;
  const int r = rh / H;
  const float* bp = ws_prefix + static_cast<int64_t>(rh) * prefix_splits * (AT_D + 2);
  const float* bt = ws_tail + static_cast<int64_t>(rh) * tail_splits * (AT_D + 2);
  const int np = min(prefix_splits, (prefix_lens[r / n] + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS);
  const int nt = min(tail_splits, (tail_lens[r] + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS);
  float M = -INFINITY;
  for (int s = 0; s < np; ++s) M = fmaxf(M, bp[s * (AT_D + 2) + AT_D]);
  for (int s = 0; s < nt; ++s) M = fmaxf(M, bt[s * (AT_D + 2) + AT_D]);
  float L = 0.f, A = 0.f;
  for (int s = 0; s < np; ++s) {
    const float ms = bp[s * (AT_D + 2) + AT_D];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
    L += bp[s * (AT_D + 2) + AT_D + 1] * f;
    A += bp[s * (AT_D + 2) + d] * f;
  }
  for (int s = 0; s < nt; ++s) {
    const float ms = bt[s * (AT_D + 2) + AT_D];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
    L += bt[s * (AT_D + 2) + AT_D + 1] * f;
    A += bt[s * (AT_D + 2) + d] * f;
  }
  out[static_cast<int64_t>(rh) * AT_D + d] = __float2bfloat16_rn(L > 0.f ? A / L : 0.f);
}

// box of [128 rows][cols] per (head, batch): 64 columns with SW128, or the 16-column SW32 box of the HD = 80 path
static int make_tmap_heads(CUtensorMap* tm, const void* ptr, int T, int H, int B, int64_t stride_b, int64_t stride_h,
                           uint32_t cols = 64, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  uint64_t dims[4] = {static_cast<uint64_t>(AT_D), static_cast<uint64_t>(T), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
  uint64_t str[3] = {static_cast<uint64_t>(AT_D) * 2, static_cast<uint64_t>(stride_h) * 2, static_cast<uint64_t>(stride_b) * 2};
  uint32_t box[4] = {cols, 128, 1, 1};
  return make_tmap_bf16_swz(tm, ptr, 4, dims, str, box, swizzle);
}

template <int HD, bool CAUSAL, bool LSE>
static int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const CUtensorMap& tmK16,
                       const CUtensorMap& tmV16, const AttnParams& p, int64_t grid, cudaStream_t stream) {
  auto kern = attn_fwd_kernel<HD, CAUSAL, LSE>;
  constexpr int smem = AttnCfg<HD>::SMEM;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, kern, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  kern<<<static_cast<int>(grid), AT_THREADS, smem, stream>>>(tmQ, tmK, tmV, tmK16, tmV16, p);
  return check_launch("attn_fwd_kernel");
}

// aria_attention_fwd and aria_attention_fwd_lse: one launcher, the logsumexp store is a compile-time flag of the same kernel
static int attention_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const uint8_t* key_mask, int32_t B,
                         int32_t H, int32_t Tq, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b,
                         int64_t kv_stride_h, int32_t out_hd, float scale, int32_t causal, cudaStream_t stream) {
  ARIA_CHECK_ARG(q && k && v && out);
  ARIA_CHECK_ARG(B > 0 && H > 0 && Tq > 0 && Tk > 0 && Tk >= (causal ? Tq : 0));
  ARIA_CHECK_ARG(out_hd > 0 && out_hd <= AT_D && out_hd % 8 == 0);
  ARIA_CHECK_ARG(q_stride_b % 8 == 0 && q_stride_h % 8 == 0 && kv_stride_b % 8 == 0 && kv_stride_h % 8 == 0);
  CUtensorMap tmQ, tmK, tmV, tmK16, tmV16;
  int rc = make_tmap_heads(&tmQ, q, Tq, H, B, q_stride_b, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, Tk, H, B, kv_stride_b, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, Tk, H, B, kv_stride_b, kv_stride_h);
  if (rc) return rc;
  if (out_hd <= 80) {  // columns 64-79 of K and V
    rc = make_tmap_heads(&tmK16, k, Tk, H, B, kv_stride_b, kv_stride_h, 16, CU_TENSOR_MAP_SWIZZLE_32B);
    if (rc) return rc;
    rc = make_tmap_heads(&tmV16, v, Tk, H, B, kv_stride_b, kv_stride_h, 16, CU_TENSOR_MAP_SWIZZLE_32B);
    if (rc) return rc;
  } else {  // unused at HD = 128
    tmK16 = tmK;
    tmV16 = tmV;
  }
  AttnParams p{};
  p.B = B;
  p.H = H;
  p.Tq = Tq;
  p.Tk = Tk;
  p.out_hd = out_hd;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.key_mask = key_mask;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.lse = lse;
  p.n_q_tiles = (Tq + AT_BM - 1) / AT_BM;
  const int64_t grid = static_cast<int64_t>(B) * H * p.n_q_tiles;
  ARIA_CHECK_ARG(grid < (1ll << 31));
#define ARIA_ATTN_LAUNCH(HD, C, L) launch_attn<HD, C, L>(tmQ, tmK, tmV, tmK16, tmV16, p, grid, stream)
  if (lse) {
    if (out_hd <= 80) return causal ? ARIA_ATTN_LAUNCH(80, true, true) : ARIA_ATTN_LAUNCH(80, false, true);
    return causal ? ARIA_ATTN_LAUNCH(128, true, true) : ARIA_ATTN_LAUNCH(128, false, true);
  }
  if (out_hd <= 80) return causal ? ARIA_ATTN_LAUNCH(80, true, false) : ARIA_ATTN_LAUNCH(80, false, false);
  return causal ? ARIA_ATTN_LAUNCH(128, true, false) : ARIA_ATTN_LAUNCH(128, false, false);
#undef ARIA_ATTN_LAUNCH
}

}  // namespace aria

using namespace aria;

extern "C" int64_t aria_attention_fwd_workspace_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk, int32_t out_hd, int32_t causal) {
  (void)B; (void)H; (void)Tq; (void)Tk; (void)out_hd; (void)causal;
  return 0;  // one CTA per (batch, head, 128 queries): no partial results to merge
}

extern "C" int aria_attention_fwd(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask, int32_t B,
                                  int32_t H, int32_t Tq, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h,
                                  int64_t kv_stride_b, int64_t kv_stride_h, int32_t out_hd, float scale, int32_t causal,
                                  void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  (void)workspace; (void)workspace_bytes;
  return attention_fwd(q, k, v, out, nullptr, key_mask, B, H, Tq, Tk, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, out_hd,
                       scale, causal, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int aria_attention_fwd_lse(const void* q, const void* k, const void* v, void* out, float* lse, const uint8_t* key_mask,
                                      int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h,
                                      int64_t kv_stride_b, int64_t kv_stride_h, int32_t out_hd, float scale, int32_t causal,
                                      void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  (void)workspace; (void)workspace_bytes;
  ARIA_CHECK_ARG(lse);
  return attention_fwd(q, k, v, out, lse, key_mask, B, H, Tq, Tk, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, out_hd,
                       scale, causal, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int aria_attention_prefill_shared_prefix(const void* q, const void* k, const void* v, const void* prefix_k,
                                                    const void* prefix_v, const int32_t* cu_seqlens, void* out, int32_t B, int32_t H,
                                                    int32_t S_tot, int32_t P, int32_t P_max, int64_t q_stride_h, int64_t kv_stride_h,
                                                    int64_t prefix_stride_h, float scale, aria_stream_t stream_) {
  ARIA_CHECK_ARG(q && k && v && prefix_k && prefix_v && cu_seqlens && out);
  ARIA_CHECK_ARG(B > 0 && H > 0 && S_tot >= B && P > 0 && P <= P_max);
  ARIA_CHECK_ARG(q_stride_h >= static_cast<int64_t>(S_tot) * AT_D && kv_stride_h >= static_cast<int64_t>(S_tot) * AT_D &&
                 prefix_stride_h >= static_cast<int64_t>(P_max) * AT_D);
  ARIA_CHECK_ARG(q_stride_h % 8 == 0 && kv_stride_h % 8 == 0 && prefix_stride_h % 8 == 0);
  const int n_q_tiles = (S_tot + AT_BM - 1) / AT_BM;
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * n_q_tiles < (1ll << 31));
  // one batch row: its stride is never stepped
  CUtensorMap tmQ, tmK, tmV, tmPK, tmPV;
  int rc = make_tmap_heads(&tmQ, q, S_tot, H, 1, q_stride_h * H, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPK, prefix_k, P, H, 1, prefix_stride_h * H, prefix_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPV, prefix_v, P, H, 1, prefix_stride_h * H, prefix_stride_h);
  if (rc) return rc;
  AttnParams p{};
  p.B = 1;
  p.H = H;
  p.Tq = S_tot;
  p.Tk = S_tot;
  p.out_hd = AT_D;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.n_q_tiles = n_q_tiles;
  const SharedPrefixParams sp{cu_seqlens, B, P};
  constexpr int smem = AttnCfg<128>::SMEM;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, attn_prefill_shared_prefix_kernel<false>, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  attn_prefill_shared_prefix_kernel<false><<<H * n_q_tiles, AT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      tmQ, tmK, tmV, tmPK, tmPV, p, sp);
  return check_launch("attn_prefill_shared_prefix_kernel");
}

extern "C" int aria_attention_prefill_paged_prefix(const void* q, const void* k, const void* v, const void* k_pool,
                                                   const void* v_pool, const int32_t* pages, int32_t n_pages_list, int32_t n_pages,
                                                   const int32_t* cu_seqlens, void* out, int32_t B, int32_t H, int32_t S_tot,
                                                   int32_t P, int64_t q_stride_h, int64_t kv_stride_h, int64_t page_stride,
                                                   int64_t pool_stride_h, float scale, aria_stream_t stream_) {
  ARIA_CHECK_ARG(q && k && v && k_pool && v_pool && cu_seqlens && out && (pages || P == 0));
  ARIA_CHECK_ARG(B > 0 && H > 0 && S_tot >= B && n_pages > 0 && n_pages_list >= 0);
  ARIA_CHECK_ARG(P >= 0 && P % DEC_SPLIT_KEYS == 0 && P / DEC_SPLIT_KEYS <= n_pages_list);
  ARIA_CHECK_ARG(q_stride_h >= static_cast<int64_t>(S_tot) * AT_D && kv_stride_h >= static_cast<int64_t>(S_tot) * AT_D);
  ARIA_CHECK_ARG(pool_stride_h >= DEC_SPLIT_KEYS * AT_D && page_stride >= pool_stride_h * H);  // pages do not overlap
  ARIA_CHECK_ARG(q_stride_h % 8 == 0 && kv_stride_h % 8 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  const int n_q_tiles = (S_tot + AT_BM - 1) / AT_BM;
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * n_q_tiles < (1ll << 31));
  CUtensorMap tmQ, tmK, tmV, tmPK, tmPV;
  int rc = make_tmap_heads(&tmQ, q, S_tot, H, 1, q_stride_h * H, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPK, k_pool, DEC_SPLIT_KEYS, H, n_pages, page_stride, pool_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPV, v_pool, DEC_SPLIT_KEYS, H, n_pages, page_stride, pool_stride_h);
  if (rc) return rc;
  AttnParams p{};
  p.B = 1;
  p.H = H;
  p.Tq = S_tot;
  p.Tk = S_tot;
  p.out_hd = AT_D;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.n_q_tiles = n_q_tiles;
  const PagedPrefixParams pp{cu_seqlens, B, P, pages};
  constexpr int smem = AttnCfg<128>::SMEM;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, attn_prefill_paged_prefix_kernel, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  attn_prefill_paged_prefix_kernel<<<H * n_q_tiles, AT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      tmQ, tmK, tmV, tmPK, tmPV, p, pp);
  return check_launch("attn_prefill_paged_prefix_kernel");
}

extern "C" int aria_attention_prefill_paged_varlen(const void* q, const void* k, const void* v, const void* k_pool,
                                                   const void* v_pool, const int32_t* page_table, int64_t page_table_stride,
                                                   int32_t n_pages, const int32_t* prefix_lens, const int32_t* cu_seqlens, void* out,
                                                   int32_t n_seg, int32_t H, int32_t S_tot, int64_t q_stride_h, int64_t kv_stride_h,
                                                   int64_t page_stride, int64_t pool_stride_h, float scale, aria_stream_t stream_) {
  ARIA_CHECK_ARG(q && k && v && k_pool && v_pool && page_table && prefix_lens && cu_seqlens && out);
  ARIA_CHECK_ARG(n_seg > 0 && H > 0 && S_tot >= n_seg && n_pages > 0 && page_table_stride > 0);
  ARIA_CHECK_ARG(q_stride_h >= static_cast<int64_t>(S_tot) * AT_D && kv_stride_h >= static_cast<int64_t>(S_tot) * AT_D);
  ARIA_CHECK_ARG(pool_stride_h >= DEC_SPLIT_KEYS * AT_D && page_stride >= pool_stride_h * H);  // pages do not overlap
  ARIA_CHECK_ARG(q_stride_h % 8 == 0 && kv_stride_h % 8 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  // each segment of len rows has ceil(len / 128) tiles <= (len + 127) / 128, and the lens sum to S_tot
  const int64_t n_q_tiles = (static_cast<int64_t>(S_tot) + static_cast<int64_t>(AT_BM - 1) * n_seg) / AT_BM;
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * n_q_tiles < (1ll << 31) && static_cast<int64_t>(n_seg) * page_table_stride < (1ll << 31));
  CUtensorMap tmQ, tmK, tmV, tmPK, tmPV;
  int rc = make_tmap_heads(&tmQ, q, S_tot, H, 1, q_stride_h * H, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, S_tot, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPK, k_pool, DEC_SPLIT_KEYS, H, n_pages, page_stride, pool_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmPV, v_pool, DEC_SPLIT_KEYS, H, n_pages, page_stride, pool_stride_h);
  if (rc) return rc;
  AttnParams p{};
  p.B = 1;
  p.H = H;
  p.Tq = S_tot;
  p.Tk = S_tot;
  p.out_hd = AT_D;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.n_q_tiles = static_cast<int>(n_q_tiles);
  const PagedVarlenParams vl{cu_seqlens, prefix_lens, page_table, page_table_stride, n_seg};
  constexpr int smem = AttnCfg<128>::SMEM;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, attn_prefill_paged_varlen_kernel, smem) != cudaSuccess) return ARIA_ERR_CUDA;
  attn_prefill_paged_varlen_kernel<<<static_cast<int>(H * n_q_tiles), AT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      tmQ, tmK, tmV, tmPK, tmPV, p, vl);
  return check_launch("attn_prefill_paged_varlen_kernel");
}

extern "C" int aria_attention_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int32_t* cu_seqlens,
                                         int32_t n_seg, int32_t H, int32_t N, int64_t q_stride_h, int64_t kv_stride_h, float scale,
                                         aria_stream_t stream_) {
  ARIA_CHECK_ARG(q && k && v && out && cu_seqlens);
  ARIA_CHECK_ARG(n_seg > 0 && H > 0 && N >= n_seg);
  ARIA_CHECK_ARG(q_stride_h >= static_cast<int64_t>(N) * AT_D && kv_stride_h >= static_cast<int64_t>(N) * AT_D);
  ARIA_CHECK_ARG(q_stride_h % 8 == 0 && kv_stride_h % 8 == 0);
  ARIA_CHECK_ARG(!lse || (reinterpret_cast<uintptr_t>(lse) & 3) == 0);
  const int n_q_tiles = (N + AT_BM - 1) / AT_BM;
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * n_q_tiles < (1ll << 31));
  // the shared-prefix pipeline with no prefix: the prefix maps are never read
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_heads(&tmQ, q, N, H, 1, q_stride_h * H, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, N, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, N, H, 1, kv_stride_h * H, kv_stride_h);
  if (rc) return rc;
  AttnParams p{};
  p.B = 1;
  p.H = H;
  p.Tq = N;
  p.Tk = N;
  p.out_hd = AT_D;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.lse = lse;
  p.n_q_tiles = n_q_tiles;
  const SharedPrefixParams sp{cu_seqlens, n_seg, 0};
  constexpr int smem = AttnCfg<128>::SMEM;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (lse) {
    static bool attr_set[kMaxDevices] = {};
    if (ensure_dynamic_smem(attr_set, attn_prefill_shared_prefix_kernel<true>, smem) != cudaSuccess) return ARIA_ERR_CUDA;
    attn_prefill_shared_prefix_kernel<true><<<H * n_q_tiles, AT_THREADS, smem, stream>>>(tmQ, tmK, tmV, tmK, tmV, p, sp);
  } else {
    static bool attr_set[kMaxDevices] = {};
    if (ensure_dynamic_smem(attr_set, attn_prefill_shared_prefix_kernel<false>, smem) != cudaSuccess) return ARIA_ERR_CUDA;
    attn_prefill_shared_prefix_kernel<false><<<H * n_q_tiles, AT_THREADS, smem, stream>>>(tmQ, tmK, tmV, tmK, tmV, p, sp);
  }
  return check_launch("attn_prefill_shared_prefix_kernel");
}

extern "C" int64_t aria_attention_decode_workspace_bytes(int32_t B, int32_t H, int32_t Tk) {
  const int64_t splits = (Tk + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  return static_cast<int64_t>(B) * H * splits * (AT_D + 2) * sizeof(float);
}

extern "C" int aria_attention_decode(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tk,
                                     int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h,
                                     float scale, void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k && v && out && workspace && B > 0 && H > 0 && Tk > 0 && q_stride_b % 4 == 0 && q_stride_h % 4 == 0);
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(B, H, Tk));
  const int splits = (Tk + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  dim3 grid(B * H, splits);
  attn_decode_partial<false><<<grid, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
                                                       static_cast<const __nv_bfloat16*>(v), key_mask, static_cast<float*>(workspace), H, Tk,
                                                       q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, scale * 1.4426950408889634f,
                                                       splits, nullptr, 0);
  int rc = check_launch("attn_decode_partial");
  if (rc) return rc;
  attn_decode_merge<false><<<B * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out), splits,
                                                      nullptr, H);
  return check_launch("attn_decode_merge");
}

extern "C" int aria_attention_decode_devlen(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask,
                                            int64_t key_mask_stride, const int32_t* lens, int32_t B, int32_t H, int32_t T_max,
                                            int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h,
                                            float scale, void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k && v && out && lens && workspace && B > 0 && H > 0 && T_max > 0 && q_stride_b % 4 == 0 && q_stride_h % 4 == 0);
  ARIA_CHECK_ARG(!key_mask || (key_mask_stride >= T_max && key_mask_stride < (1ll << 31)));
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(B, H, T_max));
  const int splits = (T_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  dim3 grid(B * H, splits);
  attn_decode_partial<true><<<grid, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
                                                      static_cast<const __nv_bfloat16*>(v), key_mask, static_cast<float*>(workspace), H,
                                                      T_max, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h,
                                                      scale * 1.4426950408889634f, splits, lens, static_cast<int>(key_mask_stride));
  int rc = check_launch("attn_decode_partial");
  if (rc) return rc;
  attn_decode_merge<true><<<B * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out), splits,
                                                     lens, H);
  return check_launch("attn_decode_merge");
}

extern "C" int aria_attention_decode_paged(const void* q, const void* k_pool, const void* v_pool, const int32_t* block_table,
                                           int64_t block_table_stride, int32_t max_pages, int32_t n_pages, const int32_t* lens,
                                           void* out, int32_t R, int32_t H, int64_t q_stride_b, int64_t q_stride_h,
                                           int64_t page_stride, int64_t pool_stride_h, float scale, void* workspace,
                                           int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k_pool && v_pool && block_table && lens && out && workspace && R > 0 && H > 0 && n_pages > 0);
  ARIA_CHECK_ARG(max_pages > 0 && max_pages <= 65535 && block_table_stride >= max_pages);  // splits are grid.y
  ARIA_CHECK_ARG(q_stride_b % 4 == 0 && q_stride_h % 4 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  ARIA_CHECK_ARG(pool_stride_h >= DEC_SPLIT_KEYS * AT_D && page_stride >= pool_stride_h * H);  // pages do not overlap
  const int T_max = max_pages * DEC_SPLIT_KEYS;
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(R, H, T_max));
  attn_decode_partial_paged<<<dim3(R * H, max_pages), 128, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k_pool), static_cast<const __nv_bfloat16*>(v_pool),
      static_cast<float*>(workspace), H, T_max, q_stride_b, q_stride_h, page_stride, pool_stride_h, scale * 1.4426950408889634f,
      max_pages, lens, block_table, block_table_stride, n_pages);
  int rc = check_launch("attn_decode_partial_paged");
  if (rc) return rc;
  attn_decode_merge<true><<<R * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out),
                                                     max_pages, lens, H);
  return check_launch("attn_decode_merge");
}

extern "C" int aria_attention_decode_multi(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask,
                                           int64_t key_mask_stride, const int32_t* lens, int32_t B, int32_t Q, int32_t H,
                                           int32_t T_max, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_q,
                                           int64_t kv_stride_b, int64_t kv_stride_h, float scale, void* workspace,
                                           int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k && v && out && lens && workspace);
  ARIA_CHECK_ARG(B > 0 && Q > 0 && Q <= 16 && H > 0 && T_max > 0 && static_cast<int64_t>(B) * Q * H < (1ll << 31));
  ARIA_CHECK_ARG(T_max <= 65535 * DEC_SPLIT_KEYS);  // splits are grid.y
  ARIA_CHECK_ARG(q_stride_b % 4 == 0 && q_stride_h % 4 == 0 && q_stride_q % 4 == 0);
  ARIA_CHECK_ARG(kv_stride_b % 8 == 0 && kv_stride_h % 8 == 0);  // the CTAs stage 16-byte vectors of each key and value row
  ARIA_CHECK_ARG(!key_mask || (key_mask_stride >= T_max && key_mask_stride < (1ll << 31)));
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(B * Q, H, T_max));
  const int splits = (T_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, attn_decode_multi_partial, SP_SMEM) != cudaSuccess) return ARIA_ERR_CUDA;
  attn_decode_multi_partial<<<dim3(B * H, splits), 128 * min(Q, SP_TEAMS), SP_SMEM, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v), lens,
      key_mask, static_cast<int>(key_mask_stride), static_cast<float*>(workspace), Q, H, T_max, q_stride_b, q_stride_h, q_stride_q,
      kv_stride_b, kv_stride_h, scale * 1.4426950408889634f, splits);
  int rc = check_launch("attn_decode_multi_partial");
  if (rc) return rc;
  attn_decode_merge<true><<<B * Q * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out),
                                                         splits, lens, H);
  return check_launch("attn_decode_merge");
}

extern "C" int64_t aria_attention_decode_shared_prefix_workspace_bytes(int32_t G, int32_t n, int32_t H, int32_t P_max, int32_t N_max) {
  if (G <= 0 || n <= 0 || H <= 0 || P_max <= 0 || N_max <= 0) return -1;
  const int64_t splits = (P_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS + (N_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  return static_cast<int64_t>(G) * n * H * splits * (AT_D + 2) * sizeof(float);
}

extern "C" int aria_attention_decode_shared_prefix(const void* q, const void* prefix_k, const void* prefix_v, const int32_t* prefix_lens,
                                                   const uint8_t* prefix_mask, int64_t prefix_mask_stride, const void* tail_k,
                                                   const void* tail_v, const int32_t* tail_lens, void* out, int32_t G, int32_t n,
                                                   int32_t H, int32_t P_max, int32_t N_max, int64_t q_stride_b, int64_t q_stride_h,
                                                   int64_t prefix_stride_b, int64_t prefix_stride_h, int64_t tail_stride_b,
                                                   int64_t tail_stride_h, float scale, void* workspace, int64_t workspace_bytes,
                                                   aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && prefix_k && prefix_v && prefix_lens && tail_k && tail_v && tail_lens && out && workspace);
  ARIA_CHECK_ARG(G > 0 && n > 0 && H > 0 && P_max > 0 && N_max > 0 && static_cast<int64_t>(G) * n * H < (1ll << 31));
  ARIA_CHECK_ARG(P_max <= 65535 * DEC_SPLIT_KEYS && N_max <= 65535 * DEC_SPLIT_KEYS);  // splits are grid.y
  ARIA_CHECK_ARG(q_stride_b % 4 == 0 && q_stride_h % 4 == 0);
  // the prefix CTAs stage 16-byte vectors of each key and value row
  ARIA_CHECK_ARG(prefix_stride_b % 8 == 0 && prefix_stride_h % 8 == 0 && tail_stride_b % 8 == 0 && tail_stride_h % 8 == 0);
  ARIA_CHECK_ARG(!prefix_mask || (prefix_mask_stride >= P_max && prefix_mask_stride < (1ll << 31)));
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_shared_prefix_workspace_bytes(G, n, H, P_max, N_max));
  const int R = G * n;
  const int p_splits = (P_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS, t_splits = (N_max + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  float* ws_prefix = static_cast<float*>(workspace);
  float* ws_tail = ws_prefix + static_cast<int64_t>(R) * H * p_splits * (AT_D + 2);
  const float scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, attn_decode_prefix_partial, SP_SMEM) != cudaSuccess) return ARIA_ERR_CUDA;
  attn_decode_prefix_partial<<<dim3(G * H, p_splits), 128 * SP_TEAMS, SP_SMEM, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(prefix_k), static_cast<const __nv_bfloat16*>(prefix_v),
      prefix_lens, prefix_mask, static_cast<int>(prefix_mask_stride), ws_prefix, n, H, P_max, q_stride_b, q_stride_h, prefix_stride_b,
      prefix_stride_h, scale_log2, p_splits);
  int rc = check_launch("attn_decode_prefix_partial");
  if (rc) return rc;
  attn_decode_partial<true><<<dim3(R * H, t_splits), 128, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(tail_k), static_cast<const __nv_bfloat16*>(tail_v),
      nullptr, ws_tail, H, N_max, q_stride_b, q_stride_h, tail_stride_b, tail_stride_h, scale_log2, t_splits, tail_lens, 0);
  rc = check_launch("attn_decode_partial");
  if (rc) return rc;
  attn_decode_merge_shared<<<R * H, 128, 0, stream>>>(ws_prefix, ws_tail, static_cast<__nv_bfloat16*>(out), p_splits, t_splits,
                                                      prefix_lens, tail_lens, n, H);
  return check_launch("attn_decode_merge_shared");
}

// The fp8 entries check what the bf16 ones check, plus the scales, and e4m3 cache strides in multiples of 16 codes (16-byte rows)
template <bool DEVLEN>
static int attention_decode_fp8(const void* q, const void* k, const void* v, const float* k_scale, const float* v_scale, void* out,
                                const uint8_t* key_mask, int64_t key_mask_stride, const int32_t* lens, int32_t B, int32_t H,
                                int32_t Tk, int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h,
                                int64_t scale_stride_b, int64_t scale_stride_h, float scale, void* workspace,
                                int64_t workspace_bytes, cudaStream_t stream) {
  ARIA_CHECK_ARG(q && k && v && k_scale && v_scale && out && workspace && (!DEVLEN || lens));
  ARIA_CHECK_ARG(B > 0 && H > 0 && Tk > 0 && q_stride_b % 4 == 0 && q_stride_h % 4 == 0);
  ARIA_CHECK_ARG(kv_stride_b % 16 == 0 && kv_stride_h % 16 == 0 && scale_stride_b >= 0 && scale_stride_h >= 0);
  ARIA_CHECK_ARG(!DEVLEN || !key_mask || (key_mask_stride >= Tk && key_mask_stride < (1ll << 31)));
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(B, H, Tk));
  const int splits = (Tk + DEC_SPLIT_KEYS - 1) / DEC_SPLIT_KEYS;
  dim3 grid(B * H, splits);
  attn_decode_partial_fp8<DEVLEN><<<grid, 128, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const uint8_t*>(k), static_cast<const uint8_t*>(v), k_scale, v_scale, key_mask,
      static_cast<float*>(workspace), H, Tk, q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, scale_stride_b, scale_stride_h,
      scale * 1.4426950408889634f, splits, lens, static_cast<int>(key_mask_stride));
  int rc = check_launch("attn_decode_partial_fp8");
  if (rc) return rc;
  attn_decode_merge<DEVLEN><<<B * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out), splits,
                                                       lens, H);
  return check_launch("attn_decode_merge");
}

extern "C" int aria_attention_decode_fp8(const void* q, const void* k, const void* v, const float* k_scale, const float* v_scale,
                                         void* out, const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tk, int64_t q_stride_b,
                                         int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, int64_t scale_stride_b,
                                         int64_t scale_stride_h, float scale, void* workspace, int64_t workspace_bytes,
                                         aria_stream_t stream_) {
  return attention_decode_fp8<false>(q, k, v, k_scale, v_scale, out, key_mask, 0, nullptr, B, H, Tk, q_stride_b, q_stride_h,
                                     kv_stride_b, kv_stride_h, scale_stride_b, scale_stride_h, scale, workspace, workspace_bytes,
                                     reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int aria_attention_decode_devlen_fp8(const void* q, const void* k, const void* v, const float* k_scale, const float* v_scale,
                                                void* out, const uint8_t* key_mask, int64_t key_mask_stride, const int32_t* lens,
                                                int32_t B, int32_t H, int32_t T_max, int64_t q_stride_b, int64_t q_stride_h,
                                                int64_t kv_stride_b, int64_t kv_stride_h, int64_t scale_stride_b,
                                                int64_t scale_stride_h, float scale, void* workspace, int64_t workspace_bytes,
                                                aria_stream_t stream_) {
  return attention_decode_fp8<true>(q, k, v, k_scale, v_scale, out, key_mask, key_mask_stride, lens, B, H, T_max, q_stride_b,
                                    q_stride_h, kv_stride_b, kv_stride_h, scale_stride_b, scale_stride_h, scale, workspace,
                                    workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int aria_attention_decode_paged_fp8(const void* q, const void* k_pool, const void* v_pool, const float* k_scale,
                                               const float* v_scale, const int32_t* block_table, int64_t block_table_stride,
                                               int32_t max_pages, int32_t n_pages, const int32_t* lens, void* out, int32_t R,
                                               int32_t H, int64_t q_stride_b, int64_t q_stride_h, int64_t page_stride,
                                               int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h, float scale,
                                               void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k_pool && v_pool && k_scale && v_scale && block_table && lens && out && workspace && R > 0 && H > 0 &&
                 n_pages > 0);
  ARIA_CHECK_ARG(max_pages > 0 && max_pages <= 65535 && block_table_stride >= max_pages);  // splits are grid.y
  ARIA_CHECK_ARG(q_stride_b % 4 == 0 && q_stride_h % 4 == 0 && page_stride % 16 == 0 && pool_stride_h % 16 == 0);
  ARIA_CHECK_ARG(pool_stride_h >= DEC_SPLIT_KEYS * AT_D && page_stride >= pool_stride_h * H);  // pages do not overlap
  ARIA_CHECK_ARG(scale_stride_h >= DEC_SPLIT_KEYS && scale_page_stride >= scale_stride_h * H);
  const int T_max = max_pages * DEC_SPLIT_KEYS;
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_decode_workspace_bytes(R, H, T_max));
  attn_decode_partial_paged_fp8<<<dim3(R * H, max_pages), 128, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const uint8_t*>(k_pool), static_cast<const uint8_t*>(v_pool), k_scale,
      v_scale, static_cast<float*>(workspace), H, T_max, q_stride_b, q_stride_h, page_stride, pool_stride_h, scale_page_stride,
      scale_stride_h, scale * 1.4426950408889634f, max_pages, lens, block_table, block_table_stride, n_pages);
  int rc = check_launch("attn_decode_partial_paged_fp8");
  if (rc) return rc;
  attn_decode_merge<true><<<R * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out),
                                                     max_pages, lens, H);
  return check_launch("attn_decode_merge");
}
