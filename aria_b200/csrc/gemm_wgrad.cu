// Weight-gradient ("wgrad") grouped GEMM for sm_90a: the contraction runs over the (ragged) token rows.
//
//     dW[g][m][n] = sum_{r in group g} A[r][m] * B[r][n]        A = [rows, Md] (layer input), B = [rows, Nd] (grad of output)
//
// Backward of the reference's expert GEMMs (autograd through `gmm`, aria/model/moe_lm.py:484; weight [E, in, out]) and,
// with one group, of the nn.Linear layers (dW[out,in] = dY^T X).  Both operands are consumed MN-major straight from the
// row-major activation tensors (wgmma transpose bits set for A and B): no transposes are materialised.
//
// Ragged groups: group row offsets are any non-decreasing values.  TMA fetches 64-row slabs starting at the group's first
// row; for the last slab of a group only the 16-row k-steps that reach into the group are issued, so whole k-steps of the
// next group that share the slab are never multiplied.  When a group's row count is not a multiple of 16, its last
// k-step also holds the first rows of the next group (or rows past the last group): before that k-step's MMAs each
// consumer warpgroup zeroes those rows in its own 64-column A chunk, so they contribute 0 * B.  In the MN-major SW128
// layout a contraction row is one whole 128-byte line, so the swizzle does not move rows.  16-aligned groups (what the
// training dispatcher's row_align = 16 produces) take no zeroing and issue exactly the same MMAs.
#include "gemm_common.cuh"

namespace aria {

struct WgradParams {
  int Md, Nd, G;
  int n_src;            // row groups are (source, g) pairs, source-major: offs has n_src*G+1 entries and out[g] sums over sources
  const int32_t* offs;  // [n_src*G+1], non-decreasing
  __nv_bfloat16* out;   // [G, Md, Nd]
  int rows;             // ACC_F32: one group over rows [0, rows)
  float* out_f32;       // ACC_F32: [Md, Nd], accumulated into
};

constexpr int WG_BN = 128;
constexpr int WG_STAGES = 6;
constexpr int WG_STAGE_BYTES = 64 * BM * 2 + 64 * WG_BN * 2;  // A slab [64 rows][128 m] + B slab [64 rows][128 n]

// ACC_F32: one group, no offsets array; the epilogue adds the fp32 accumulators into out_f32 instead of storing bf16.  A
// tile belongs to one CTA, so the read-modify-write needs no atomics.
template <bool ACC_F32>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const WgradParams p) {
  uint8_t* smem = smem_1024();
  const BarrierRing<WG_STAGES> bar(smem + WG_STAGES * WG_STAGE_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    bar.init(1, CONSUMER_WARPS);
    fence_mbar_init();
  }
  __syncthreads();

  const int mt = (p.Md + BM - 1) / BM, nt = (p.Nd + WG_BN - 1) / WG_BN;
  const int tiles_per_group = mt * nt;
  const int total = p.G * tiles_per_group;
  // tile t -> (group, m tile, n tile); n innermost so concurrent CTAs share the A slab of the group
  auto decode = [&](int t, int& g, int& mi, int& ni) {
    g = t / tiles_per_group;
    const int r = t - g * tiles_per_group;
    mi = r / nt;
    ni = r - mi * nt;
  };
  // rows of (source s, group g): start row and row count
  auto span = [&](int s, int g, int& r0, int& n) {
    if constexpr (ACC_F32) {
      r0 = 0;
      n = p.rows;
    } else {
      r0 = p.offs[s * p.G + g];
      n = p.offs[s * p.G + g + 1] - r0;
    }
  };

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      RingPos<WG_STAGES> rp;
      for (int t = blockIdx.x; t < total; t += gridDim.x) {
        int g, mi, ni;
        decode(t, g, mi, ni);
        for (int src = 0; src < p.n_src; ++src) {
          int r0, n;
          span(src, g, r0, n);
          const int slabs = (n + 63) / 64;
          for (int s = 0; s < slabs; ++s) {
            mbar_wait(&bar.empty[rp.stage], rp.phase ^ 1);
            uint8_t* sa = smem + rp.stage * WG_STAGE_BYTES;
            uint8_t* sb = sa + 64 * BM * 2;
            uint64_t* fb = &bar.full[rp.stage];
            mbar_arrive_expect_tx(fb, WG_STAGE_BYTES);
            const int row = r0 + s * 64;
#pragma unroll
            for (int c = 0; c < BM / 64; ++c) tma_load_2d(sa + c * 8192, &tmA, fb, mi * BM + c * 64, row);
#pragma unroll
            for (int c = 0; c < WG_BN / 64; ++c) tma_load_2d(sb + c * 8192, &tmB, fb, ni * WG_BN + c * 64, row);
            rp.next();
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1, tid = threadIdx.x & 127;
    // both operands MN-major: A = 64-column chunk cw of the slab (this warpgroup's 64 m), B = both 64-column chunks (LBO 8 KB)
    const uint64_t dA0 = make_smem_desc(smem_u32(smem) + cw * 8192, 8192, 1024);  // stage 0, k-step 0; later ones are + (bytes >> 4)
    const uint64_t dB0 = make_smem_desc(smem_u32(smem) + 64 * BM * 2, 8192, 1024);
    const ConsumerThread ct = consumer_thread(cw, lane);
    RingPos<WG_STAGES> rp;
    for (int t = blockIdx.x; t < total; t += gridDim.x) {
      int g, mi, ni;
      decode(t, g, mi, ni);
      float acc[WG_BN / 2];
#pragma unroll
      for (int i = 0; i < WG_BN / 2; ++i) acc[i] = 0.f;  // an empty group stores zeros
      int prev = -1;
      for (int src = 0; src < p.n_src; ++src) {
        int r0, n;
        span(src, g, r0, n);
        const int slabs = (n + 63) / 64;
        for (int s = 0; s < slabs; ++s) {
          mbar_wait(&bar.full[rp.stage], rp.phase);
          const uint64_t da = dA0 + rp.stage * (WG_STAGE_BYTES >> 4), db = dB0 + rp.stage * (WG_STAGE_BYTES >> 4);
          // the last slab of a group: only the 16-row k-steps that reach into the group (rows of the next group share the slab)
          const int valid = n - s * 64;                 // rows of this group in the slab (> 0)
          const int kmax = min(4, (valid + 15) >> 4);
          if (valid < 16 * kmax) {
            // partial last k-step: zero A rows [valid, 16 * kmax) of this warpgroup's chunk (one 128-byte line per row);
            // the proxy fence orders these generic stores before the wgmma reads and before TMA refills the slot
            uint4* ca = reinterpret_cast<uint4*>(smem + rp.stage * WG_STAGE_BYTES + cw * 8192);
            for (int i = valid * 8 + tid; i < kmax * 128; i += 128) ca[i] = make_uint4(0u, 0u, 0u, 0u);
            fence_proxy_async_smem();
            if (cw == 0) named_bar_sync(1, 128);    // literal ids: ptxas reserves 3 hardware barriers, not all 16
            else named_bar_sync(2, 128);
          }
          wgmma_fence();
          for (int k = 0; k < kmax; ++k) wgmma_m64n128_ss<1, 1>(acc, da + k * (2048 >> 4), db + k * (2048 >> 4), 1u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&bar.empty[prev]);
          prev = static_cast<int>(rp.stage);
          rp.next();
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&bar.empty[prev]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = mi * BM + ct.frag_row + 8 * h;
        if (m >= p.Md) continue;
        if constexpr (ACC_F32) {
          float* orow = p.out_f32 + static_cast<int64_t>(m) * p.Nd + ni * WG_BN;
#pragma unroll
          for (int j = 0; j < WG_BN / 8; ++j) {
            if (ni * WG_BN + 8 * j + 8 <= p.Nd) {
              float2* o = reinterpret_cast<float2*>(orow + 8 * j + ct.frag_col);
              float2 c = *o;
              c.x += acc[4 * j + 2 * h];
              c.y += acc[4 * j + 2 * h + 1];
              *o = c;
            }
          }
          continue;
        }
        __nv_bfloat16* orow = p.out + (static_cast<int64_t>(g) * p.Md + m) * p.Nd + ni * WG_BN;
#pragma unroll
        for (int j = 0; j < WG_BN / 8; ++j) {
          if (ni * WG_BN + 8 * j + 8 <= p.Nd)
            *reinterpret_cast<uint32_t*>(orow + 8 * j + ct.frag_col) = pack_bf16(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

}  // namespace aria

using namespace aria;

extern "C" int aria_grouped_wgrad(const void* a, int64_t lda, const void* b, int64_t ldb, void* out, const int32_t* group_offsets,
                                  int64_t rows, int64_t md, int64_t nd, int32_t num_groups, int32_t num_sources,
                                  aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(a && b && out && group_offsets && rows >= 0 && md > 0 && nd > 0 && num_groups >= 1 && num_sources >= 1);
  ARIA_CHECK_ARG(md % 8 == 0 && nd % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 && lda >= md && ldb >= nd);
  CUtensorMap tmA, tmB;
  // row-major [rows, Md]: inner = feature dim (the MMA's M / N), outer = rows (the contraction)
  int rc = make_tmap_2d(&tmA, a, md, rows > 0 ? rows : 1, lda * 2, 64, 64);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, b, nd, rows > 0 ? rows : 1, ldb * 2, 64, 64);
  if (rc) return rc;
  WgradParams p{};
  p.Md = static_cast<int>(md);
  p.Nd = static_cast<int>(nd);
  p.G = num_groups;
  p.n_src = num_sources;
  p.offs = group_offsets;
  p.out = static_cast<__nv_bfloat16*>(out);
  constexpr int SMEM = WG_STAGES * WG_STAGE_BYTES + 1024 + 256;
  const int64_t tiles = static_cast<int64_t>(num_groups) * ((md + BM - 1) / BM) * ((nd + WG_BN - 1) / WG_BN);
  return launch_persistent<wgrad_kernel<false>>("wgrad_kernel", GEMM_THREADS, SMEM, tiles, stream, tmA, tmB, p);
}

extern "C" int aria_wgrad_accumulate_f32(const void* a, int64_t lda, const void* b, int64_t ldb, float* out, int64_t rows,
                                         int64_t md, int64_t nd, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(a && b && out && rows >= 0 && rows <= INT32_MAX && md > 0 && nd > 0 && md <= INT32_MAX && nd <= INT32_MAX);
  ARIA_CHECK_ARG(md % 8 == 0 && nd % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 && lda >= md && ldb >= nd);
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 7) == 0);
  if (rows == 0) return ARIA_OK;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_2d(&tmA, a, md, rows, lda * 2, 64, 64);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, b, nd, rows, ldb * 2, 64, 64);
  if (rc) return rc;
  WgradParams p{};
  p.Md = static_cast<int>(md);
  p.Nd = static_cast<int>(nd);
  p.G = 1;
  p.n_src = 1;
  p.rows = static_cast<int>(rows);
  p.out_f32 = out;
  constexpr int SMEM = WG_STAGES * WG_STAGE_BYTES + 1024 + 256;
  const int64_t tiles = ((md + BM - 1) / BM) * ((nd + WG_BN - 1) / WG_BN);
  return launch_persistent<wgrad_kernel<true>>("wgrad_accumulate_f32_kernel", GEMM_THREADS, SMEM, tiles, stream, tmA, tmB, p);
}
