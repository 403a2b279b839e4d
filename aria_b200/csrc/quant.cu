// aria_quantize_fp8_cols: per-(expert, output column) e4m3 quantisation of the routed-expert weights (GroupedGEMM.weight,
// [G, K, N] bf16, N contiguous) for the fp8-weight grouped GEMMs (gemm.cu, aria_grouped_gemm_fp8 / _w8a8).
// aria_permute_quantize_fp8_rows: the same formula per row of the activations, for aria_grouped_gemm_w8a8.
//
//   scale[g, n] = max_k |w[g, k, n]| / 448        (fp32, IEEE division; an all-zero column gets scale 1)
//   q[g, k, n]  = e4m3(w[g, k, n] / scale[g, n])  (IEEE division, round to nearest even, saturating)
//
// Bit for bit what torch computes as (w.float() / scale).to(torch.float8_e4m3fn).  Two HBM-bound passes: a column-amax
// reduction over k, then an elementwise cast that re-reads w.
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aria_b200.h"
#include "common.cuh"
#include "fp8.cuh"

namespace {

using aria::cast8_e4m3;
using aria::E4M3_MAX;

constexpr int AMAX_TX = 32;  // threads across the columns of a block (8 columns each: one 16-byte load per row)
constexpr int AMAX_TY = 8;   // row slices of a block, reduced through shared memory

__global__ void __launch_bounds__(AMAX_TX * AMAX_TY) col_amax_kernel(const __nv_bfloat16* __restrict__ w, float* __restrict__ scale,
                                                                     int K, int N) {
  const int g = blockIdx.y;
  const int c0 = (blockIdx.x * AMAX_TX + threadIdx.x) * 8;
  const bool ok = c0 < N;
  const __nv_bfloat16* src = w + static_cast<int64_t>(g) * K * N + c0;
  float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (ok) {
#pragma unroll 4
    for (int k = threadIdx.y; k < K; k += AMAX_TY) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(k) * N));
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m[2 * j] = fmaxf(m[2 * j], fabsf(__uint_as_float(u[j] << 16)));
        m[2 * j + 1] = fmaxf(m[2 * j + 1], fabsf(__uint_as_float(u[j] & 0xFFFF0000u)));
      }
    }
  }
  __shared__ float red[AMAX_TY][AMAX_TX * 8 + 4];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x * 8 + j] = m[j];
  __syncthreads();
  if (threadIdx.y == 0 && ok) {
#pragma unroll
    for (int y = 1; y < AMAX_TY; ++y)
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], red[y][threadIdx.x * 8 + j]);
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = m[j] > 0.f ? __fdiv_rn(m[j], E4M3_MAX) : 1.f;
    float4* dst = reinterpret_cast<float4*>(scale + static_cast<int64_t>(g) * N + c0);
    dst[0] = make_float4(s[0], s[1], s[2], s[3]);
    dst[1] = make_float4(s[4], s[5], s[6], s[7]);
  }
}

// one thread per 8 consecutive elements of a row: 16-byte load of w, 8-byte store of q
__global__ void __launch_bounds__(256) cast_e4m3_kernel(const __nv_bfloat16* __restrict__ w, const float* __restrict__ scale,
                                                        uint8_t* __restrict__ q, int64_t chunks, int K, int N) {
  const int nc = N / 8;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < chunks;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = i / nc;  // row of the flattened [G*K, N] view
    const int c0 = static_cast<int>(i - row * nc) * 8;
    const int g = static_cast<int>(row / K);
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(w + row * N + c0));
    const float4* sp = reinterpret_cast<const float4*>(scale + static_cast<int64_t>(g) * N + c0);
    const float4 s0 = __ldg(sp), s1 = __ldg(sp + 1);
    const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t packed[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = __fdiv_rn(__uint_as_float(u[j] << 16), s[2 * j]);
      const float x1 = __fdiv_rn(__uint_as_float(u[j] & 0xFFFF0000u), s[2 * j + 1]);
      const uint32_t pair = __nv_cvt_float2_to_fp8x2(make_float2(x0, x1), __NV_SATFINITE, __NV_E4M3);  // low byte = x0
      packed[j >> 1] |= (pair & 0xFFFFu) << (16 * (j & 1));
    }
    *reinterpret_cast<uint2*>(q + row * N + c0) = make_uint2(packed[0], packed[1]);
  }
}

// Per-row e4m3 quantisation of the activations of the W8A8 expert GEMMs, fused with the token gather:
//   scale[r] = max |x[src(r)]| / 448 (1 for an all-zero row),  q[r] = e4m3(x[src(r)] / scale[r])
// src(r) = src_token[r], or r without a gather.  One warp per row; the row stays in registers between the amax and the cast, so
// every source byte is read once.
constexpr int QROW_MAX_VEC = 16;  // 16-byte chunks per lane: d <= 32 * 16 * 8 = 4096

__global__ void __launch_bounds__(256) permute_quantize_rows_kernel(const uint4* __restrict__ x, const int32_t* __restrict__ src_token,
                                                                    uint8_t* __restrict__ q, float* __restrict__ scale,
                                                                    int64_t rows, int vec_per_row) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); r < rows;
       r += static_cast<int64_t>(gridDim.x) * wpb) {
    const int64_t st = src_token ? src_token[r] : r;  // st < 0: alignment pad row of the training layout, quantised as zeros
    uint4 v[QROW_MAX_VEC];
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < QROW_MAX_VEC; ++i) {
      const int c = lane + 32 * i;
      v[i] = (st >= 0 && c < vec_per_row) ? __ldg(x + st * vec_per_row + c) : make_uint4(0, 0, 0, 0);
      const uint32_t u[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        m = fmaxf(m, fmaxf(fabsf(__uint_as_float(u[j] << 16)), fabsf(__uint_as_float(u[j] & 0xFFFF0000u))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float s = m > 0.f ? __fdiv_rn(m, E4M3_MAX) : 1.f;
    if (lane == 0) scale[r] = s;
    uint2* dst = reinterpret_cast<uint2*>(q + r * vec_per_row * 8);
#pragma unroll
    for (int i = 0; i < QROW_MAX_VEC; ++i) {
      const int c = lane + 32 * i;
      if (c < vec_per_row) dst[c] = cast8_e4m3(v[i], s);
    }
  }
}

}  // namespace

extern "C" int aria_permute_quantize_fp8_rows(const void* x, const int32_t* src_token, void* q, float* scale, int64_t rows,
                                              int32_t d, aria_stream_t stream_) {
  ARIA_CHECK_ARG(x && q && scale);
  ARIA_CHECK_ARG(rows >= 0 && d > 0 && d % 8 == 0 && d <= 32 * QROW_MAX_VEC * 8);
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(scale) & 3) == 0);
  if (rows == 0) return ARIA_OK;
  int64_t blocks = (rows + 7) / 8;
  const int64_t cap = static_cast<int64_t>(aria::sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  permute_quantize_rows_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint4*>(x), src_token, static_cast<uint8_t*>(q), scale, rows, d / 8);
  return aria::check_launch("permute_quantize_rows_kernel");
}

extern "C" int aria_quantize_fp8_cols(const void* w, void* q, float* scale, int32_t G, int64_t K, int64_t N,
                                      aria_stream_t stream_) {
  ARIA_CHECK_ARG(w && q && scale);
  ARIA_CHECK_ARG(G >= 1 && K > 0 && N > 0 && K % 64 == 0 && N % 64 == 0);
  ARIA_CHECK_ARG(K <= (1 << 30) && N <= (1 << 30) && static_cast<int64_t>(G) * K <= (int64_t(1) << 40) / N);
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(scale) & 15) == 0);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const __nv_bfloat16* wb = static_cast<const __nv_bfloat16*>(w);
  dim3 ablock(AMAX_TX, AMAX_TY);
  dim3 agrid(static_cast<unsigned>((N + AMAX_TX * 8 - 1) / (AMAX_TX * 8)), static_cast<unsigned>(G));
  col_amax_kernel<<<agrid, ablock, 0, stream>>>(wb, scale, static_cast<int>(K), static_cast<int>(N));
  int rc = aria::check_launch("col_amax_kernel");
  if (rc) return rc;
  const int64_t chunks = static_cast<int64_t>(G) * K * (N / 8);
  int64_t blocks = (chunks + 255) / 256;
  const int64_t cap = static_cast<int64_t>(aria::sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  cast_e4m3_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(wb, scale, static_cast<uint8_t*>(q), chunks,
                                                                     static_cast<int>(K), static_cast<int>(N));
  return aria::check_launch("cast_e4m3_kernel");
}
