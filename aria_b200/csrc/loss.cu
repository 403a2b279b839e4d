// Cross-entropy over rows of bf16 logits, the loss half of the fused lm_head loss (aria_b200/loss.py):
//
//     loss[r]     = logsumexp(x[r, :]) - x[r, label[r]]                              fp32
//     x[r, :]    <- (softmax(x[r, :]) - onehot(label[r])) * (*grad_scale)            bf16, in place
//
// One CTA per row, 128-bit accesses.  Pass 1 streams the row once and keeps an online (max, sum of exp) per thread in fp32;
// the per-thread pairs are merged in a fixed order (xor butterfly in each warp, then the same over the warps' pairs), so two
// runs are bit-identical; there are no atomics.  Pass 2 reads the row again and overwrites it with the gradient.
//
// Exponents are taken as (x - max) - log(sum): for the terms that matter x and max are close, so x - max is exact in fp32,
// and the rounding of a large logsumexp never enters an exponent.
#include <math.h>

#include "common.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int CE_THREADS = 512;
constexpr int CE_WARPS = CE_THREADS / 32;

// (m, s) <- the pair over the union; an empty side has m = -inf.  Symmetric in its two operands, so every lane of a
// butterfly ends with the same bits.
ARIA_DEVICE void max_sum_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) {
    m = m2;
    s = s2;
    return;
  }
  const float M = fmaxf(m, m2);
  s = s * __expf(m - M) + s2 * __expf(m2 - M);
  m = M;
}

ARIA_DEVICE void max_sum_add(float& m, float& s, const uint4 q) {
  const uint32_t a[4] = {q.x, q.y, q.z, q.w};
  float x[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    x[2 * j] = bf16_lo(a[j]);
    x[2 * j + 1] = bf16_hi(a[j]);
  }
  float vm = x[0];
#pragma unroll
  for (int j = 1; j < 8; ++j) vm = fmaxf(vm, x[j]);
  if (vm > m) {
    s *= __expf(m - vm);  // m = -inf: exp(-inf) = 0 and s is 0 already
    m = vm;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s += __expf(x[j] - m);
}

__global__ void __launch_bounds__(CE_THREADS, 2)
cross_entropy_rows_kernel(__nv_bfloat16* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels,
                          const float* __restrict__ grad_scale, float* __restrict__ loss, int V) {
  __shared__ float red_m[CE_WARPS], red_s[CE_WARPS];
  __shared__ float label_logit;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r = blockIdx.x;
  uint4* row = reinterpret_cast<uint4*>(logits + r * ld);
  const int vpr = V / 8;
  const int64_t label = labels[r];
  const bool label_ok = label >= 0 && label < V;
  if (tid == 0) label_logit = label_ok ? __bfloat162float(logits[r * ld + label]) : 0.f;

  // pass 1: four 128-bit loads in flight per thread, then the tail
  float m = -INFINITY, s = 0.f;
  int v = tid;
  for (; v + 3 * CE_THREADS < vpr; v += 4 * CE_THREADS) {
    uint4 q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = row[v + i * CE_THREADS];
#pragma unroll
    for (int i = 0; i < 4; ++i) max_sum_add(m, s, q[i]);
  }
  for (; v < vpr; v += CE_THREADS) max_sum_add(m, s, row[v]);
#pragma unroll
  for (int o = 16; o; o >>= 1) max_sum_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) {
    red_m[warp] = m;
    red_s[warp] = s;
  }
  __syncthreads();  // also orders thread 0's read of the label logit before any thread's pass-2 store
  m = lane < CE_WARPS ? red_m[lane] : -INFINITY;
  s = lane < CE_WARPS ? red_s[lane] : 0.f;
#pragma unroll
  for (int o = 16; o; o >>= 1) max_sum_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
  const float log_s = logf(s);  // s >= 1: the maximum contributes exp(0)
  if (tid == 0) loss[r] = label_ok ? (m - label_logit) + log_s : __int_as_float(0x7fc00000);

  // pass 2: the gradient, in place
  const float gs = *grad_scale;
  const int label_vec = label_ok ? static_cast<int>(label >> 3) : -1;
  for (v = tid; v < vpr; v += CE_THREADS) {
    const uint4 q = row[v];
    const uint32_t a[4] = {q.x, q.y, q.z, q.w};
    float g[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      g[2 * j] = __expf((bf16_lo(a[j]) - m) - log_s) * gs;
      g[2 * j + 1] = __expf((bf16_hi(a[j]) - m) - log_s) * gs;
    }
    if (v == label_vec) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j == static_cast<int>(label & 7)) g[j] -= gs;
    }
    row[v] = make_uint4(pack_bf16(g[0], g[1]), pack_bf16(g[2], g[3]), pack_bf16(g[4], g[5]), pack_bf16(g[6], g[7]));
  }
}

}  // namespace aria

using namespace aria;

extern "C" int aria_cross_entropy_rows(void* logits, int64_t ld, const int64_t* labels, const float* grad_scale, float* loss,
                                       int64_t rows, int32_t vocab, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(logits && labels && grad_scale && loss && rows >= 0 && rows <= INT32_MAX);
  ARIA_CHECK_ARG(vocab > 0 && vocab % 8 == 0 && ld >= vocab && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  if (rows == 0) return ARIA_OK;
  cross_entropy_rows_kernel<<<static_cast<unsigned>(rows), CE_THREADS, 0, stream>>>(
      static_cast<__nv_bfloat16*>(logits), ld, labels, grad_scale, loss, vocab);
  return check_launch("cross_entropy_rows_kernel");
}
