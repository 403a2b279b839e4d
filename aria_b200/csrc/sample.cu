// Next-token sampling for generation, sm_90a.
//
// aria_sample_tokens: Hugging Face's warper chain on an fp32 copy of bf16 logits, one CTA of 1024 threads per row:
//   TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> softmax -> multinomial.
//   top-k: radix select on the 16-bit order-preserving key of each bf16 logit (two 8-bit histogram passes).  Division by a
//     positive temperature is monotone, so the k-th largest scaled logit is the scaled k-th largest bf16 logit; every logit
//     equal to it (the pivot) is kept, as TopKLogitsWarper keeps ties.
//   top-p: the logits strictly above the pivot (< k <= 1024 of them) are compacted to shared memory and bitonic-sorted
//     ascending by (value, index); the pivot ties, all of the same probability, come first in that order.  A block scan of
//     the sorted probabilities gives HF's cumulative sums; entries whose sum is <= 1 - p are removed, ties in the order of a
//     stable sort (lowest index first), and the largest entry is always kept.
//   sampling: Gumbel-max over the kept set, argmax of (scaled logit + Gumbel noise): the same distribution as softmax +
//     multinomial and as gpt-fast's exponential race.  The noise is Philox4x32-10 keyed by the host seed, counter
//     (vocabulary index, row, device step offset), so a CUDA-graph replay draws fresh numbers once the offset advances.
//     It is not torch's RNG stream.
//   temperature 0 is greedy: argmax of the logits, ties to the lowest id (torch.argmax's rule).
// Every sum is reduced in a fixed order, so a row's result depends only on its logits, the seed and the offset.
//
// aria_sample_tokens_rows: the same kernel with a noise row and an offset per logits row, so that logits row b * (K + 1) + i
// of a prompt-lookup verification step draws the noise generation row b draws for its token n_out[b] + i.
// aria_sample_tokens_slots: aria_sample_tokens_rows with the temperature, top_k, top_p and seed of each row also read from
// device arrays (continuous batching: every slot samples with its own request's parameters).
#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace aria {

constexpr int SP_THREADS = 1024;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_MAX_K = 1024;
constexpr int32_t SP_MAX_ROWS = 1 << 20;
constexpr int32_t SP_MAX_VOCAB = 1 << 24;

struct SampleParams {
  const uint16_t* logits;  // bf16 bits, row r at logits + r * stride
  int64_t stride;
  int64_t* next_ids;
  float* probs;            // [B, V] or NULL
  int V;
  float temperature;
  int top_k;
  float top_p;
  uint32_t seed_lo, seed_hi;
  const uint64_t* rng_offset;  // device, or NULL (offset 0)
};

// order-preserving 16-bit key of a bf16 bit pattern (larger key = larger value) and its inverse
__device__ __forceinline__ uint32_t bf16_key(uint32_t u) { return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u); }
__device__ __forceinline__ float key_to_float(uint32_t k) {
  const uint32_t u = (k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu);
  return __uint_as_float(u << 16);
}

// Philox4x32-10 (Salmon et al., SC'11); the first output word
__device__ __forceinline__ uint32_t philox_x0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// standard Gumbel noise from 23 random bits: u in [2^-24, 1 - 2^-24], -log(-log u) finite
__device__ __forceinline__ float gumbel(uint32_t x) {
  const float u = (static_cast<float>(x >> 9) + 0.5f) * (1.0f / 8388608.0f);
  return -logf(-logf(u));
}

// (score, index) argmax: larger score wins, equal scores go to the lower index
__device__ __forceinline__ bool arg_better(float s, int i, float bs, int bi) { return s > bs || (s == bs && i < bi); }

struct SampleSmem {
  uint32_t hist[256];
  unsigned long long list[SP_MAX_K];  // (key << 32) | index, keys strictly above the pivot
  float red_f[SP_WARPS];
  int red_i[SP_WARPS];
  int n_list;
  int bin, above;
  int cut;
};

__device__ float block_sum(float v, SampleSmem& sm) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm.red_f[warp] = v;
  __syncthreads();
  v = lane < SP_WARPS ? sm.red_f[lane] : 0.f;
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ void block_argmax(float& s, int& i, SampleSmem& sm) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (arg_better(os, oi, s, i)) s = os, i = oi;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm.red_f[warp] = s, sm.red_i[warp] = i;
  __syncthreads();
  s = lane < SP_WARPS ? sm.red_f[lane] : -INFINITY;
  i = lane < SP_WARPS ? sm.red_i[lane] : INT_MAX;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (arg_better(os, oi, s, i)) s = os, i = oi;
  }
}

// Inclusive scan over the block in thread order.
__device__ float block_scan(float v, SampleSmem& sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  __syncthreads();
  if (lane == 31) sm.red_f[warp] = v;
  __syncthreads();
  float w = lane < SP_WARPS ? sm.red_f[lane] : 0.f;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, w, o);
    if (lane >= o) w += n;
  }
  const float before = __shfl_sync(0xffffffffu, w, (warp + 31) & 31);
  return warp ? v + before : v;
}

// Warp 0 finds the histogram bin holding the need-th largest key: sm.bin, and sm.above = the count in higher bins.
__device__ void find_bin(SampleSmem& sm, int need) {
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    uint32_t c[8], tot = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) tot += (c[j] = sm.hist[8 * lane + j]);
    uint32_t suffix = tot;  // inclusive suffix sum over the lanes
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t n = __shfl_down_sync(0xffffffffu, suffix, o);
      if (lane + o < 32) suffix += n;
    }
    uint32_t cum = suffix - tot;  // keys in the bins of the higher lanes
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (cum < static_cast<uint32_t>(need) && cum + c[j] >= static_cast<uint32_t>(need)) {
        sm.bin = 8 * lane + j;
        sm.above = static_cast<int>(cum);
      }
      cum += c[j];
    }
  }
  __syncthreads();
}

// Per-row sampling parameters of aria_sample_tokens_slots, device arrays [R]
struct SlotSampling {
  const float* temperature;
  const int32_t* top_k;
  const float* top_p;
  const uint64_t* seed;
};

// ROWS (aria_sample_tokens_rows): logits row `row` draws the noise of row noise_rows[row] at offset offsets[row] instead of
// (row, *p.rng_offset).  SLOTS (with ROWS): the row's temperature, top_k, top_p and seed come from `slots`, brought into the
// ranges aria_sample_tokens accepts (a caller checks them; this keeps a bad entry from reading past shared memory).
// Everything else is the same code.
template <bool ROWS, bool SLOTS = false>
__device__ __forceinline__ void sample_body(SampleParams p, const int32_t* __restrict__ noise_rows,
                                            const uint64_t* __restrict__ offsets, const SlotSampling slots = {}) {
  __shared__ SampleSmem sm;
  if constexpr (SLOTS) {
    const int r = blockIdx.x;
    const float t = slots.temperature[r];
    p.temperature = t > 0.f && t <= FLT_MAX ? t : 0.f;
    p.top_k = min(max(slots.top_k[r], 0), SP_MAX_K);
    const float tp = slots.top_p[r];
    p.top_p = p.top_k > 0 && tp > 0.f && tp < 1.f ? tp : 1.f;
    const uint64_t seed = slots.seed[r];
    p.seed_lo = static_cast<uint32_t>(seed);
    p.seed_hi = static_cast<uint32_t>(seed >> 32);
  }
  const int tid = threadIdx.x, row = blockIdx.x, V = p.V;
  const uint16_t* x = p.logits + static_cast<int64_t>(row) * p.stride;
  float* probs = p.probs ? p.probs + static_cast<int64_t>(row) * V : nullptr;

  if (p.temperature == 0.f) {  // greedy
    float bs = -INFINITY;
    int bi = INT_MAX;
    for (int i = tid; i < V; i += SP_THREADS) {
      const float k = static_cast<float>(bf16_key(x[i]));  // keys < 2^16 are exact in fp32
      if (arg_better(k, i, bs, bi)) bs = k, bi = i;
    }
    block_argmax(bs, bi, sm);
    if (tid == 0) p.next_ids[row] = bi;
    if (probs)
      for (int i = tid; i < V; i += SP_THREADS) probs[i] = i == bi ? 1.f : 0.f;
    return;
  }

  const float temp = p.temperature;  // HF divides: scores / temperature
  const int k = min(p.top_k, V);
  uint32_t pivot = 0;                 // keys >= pivot survive top-k (0: every key)
  int n_tie = 0, n_gt = 0;
  float m, z_kept;                    // max kept scaled logit, sum of exp(s - m) over the final kept set
  int r_tie = 0, fk = 0;              // pivot ties removed by top-p; first kept entry of the sorted list
  int idx_cut = -1;                   // pivot ties with index <= idx_cut are removed
  unsigned long long fk_comp = 0;     // (key, index) of the smallest kept list entry

  if (k > 0) {
    // ---- radix select of the k-th largest key: high byte, then low byte
    for (int i = tid; i < 256; i += SP_THREADS) sm.hist[i] = 0;
    if (tid == 0) sm.n_list = 0;
    __syncthreads();
    for (int i = tid; i < V; i += SP_THREADS) atomicAdd(&sm.hist[bf16_key(x[i]) >> 8], 1u);
    find_bin(sm, k);
    const uint32_t hb = sm.bin;
    const int above_hi = sm.above;
    for (int i = tid; i < 256; i += SP_THREADS) sm.hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < V; i += SP_THREADS) {
      const uint32_t key = bf16_key(x[i]);
      if ((key >> 8) == hb) atomicAdd(&sm.hist[key & 0xFF], 1u);
    }
    find_bin(sm, k - above_hi);
    pivot = (hb << 8) | sm.bin;
    n_gt = above_hi + sm.above;
    n_tie = static_cast<int>(sm.hist[sm.bin]);
    // ---- compact the keys above the pivot (n_gt < k of them) and sort them ascending by (key, index)
    for (int i = tid; i < V; i += SP_THREADS) {
      const uint32_t key = bf16_key(x[i]);
      if (key > pivot) sm.list[atomicAdd(&sm.n_list, 1)] = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(i);
    }
    __syncthreads();
    int P = 1;
    while (P < n_gt) P <<= 1;
    for (int i = n_gt + tid; i < P; i += SP_THREADS) sm.list[i] = ~0ull;
    for (int size = 2; size <= P; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        __syncthreads();
        const int i = tid, j = tid ^ stride;
        if (i < P && j > i) {
          const unsigned long long a = sm.list[i], b = sm.list[j];
          if ((a > b) == ((i & size) == 0)) {
            sm.list[i] = b;
            sm.list[j] = a;
          }
        }
      }
    }
    __syncthreads();
    // ---- softmax over the top-k set: pivot ties (probability q_piv each) first, then the sorted list
    const float s_piv = key_to_float(pivot) / temp;
    const bool mine = tid < n_gt;
    const float s_t = mine ? key_to_float(static_cast<uint32_t>(sm.list[tid] >> 32)) / temp : -INFINITY;
    m = n_gt > 0 ? key_to_float(static_cast<uint32_t>(sm.list[n_gt - 1] >> 32)) / temp : s_piv;
    const float e_t = mine ? expf(s_t - m) : 0.f;
    const float e_piv = expf(s_piv - m);
    const float cum_t = block_scan(e_t, sm);
    const float z = n_tie * e_piv + block_sum(e_t, sm);
    if (p.top_p < 1.f) {
      // ---- top-p with HF's rule: ascending cumulative probability <= 1 - p is removed, the largest entry always stays
      const float thr = 1.f - p.top_p;
      const float q_piv = e_piv / z;
      if (q_piv <= 0.f) {
        r_tie = n_tie;
      } else {
        const float rf = floorf(thr / q_piv);
        r_tie = rf >= static_cast<float>(n_tie) ? n_tie : static_cast<int>(rf);
      }
      if (n_gt == 0) r_tie = min(r_tie, n_tie - 1);
      if (r_tie == n_tie) {
        const bool removed = mine && (n_tie * e_piv + cum_t) / z <= thr;
        fk = min(__syncthreads_count(removed), n_gt - 1);
      }
      if (r_tie > 0 && r_tie < n_tie) {
        // index of the r_tie-th pivot tie in index order (a stable sort puts the lower indices first)
        const int lane = tid & 31, warp = tid >> 5;
        int base = 0;
        for (int i0 = 0; i0 < V && base < r_tie; i0 += SP_THREADS) {
          const int i = i0 + tid;
          const bool t = i < V && bf16_key(x[i]) == pivot;
          const unsigned bal = __ballot_sync(0xffffffffu, t);
          __syncthreads();
          if (lane == 0) sm.red_i[warp] = __popc(bal);
          __syncthreads();
          int before = base + __popc(bal & ((1u << lane) - 1u)), total = 0;
          for (int w = 0; w < SP_WARPS; ++w) {
            const int c = sm.red_i[w];
            if (w < warp) before += c;
            total += c;
          }
          if (t && before + 1 == r_tie) sm.cut = i;
          base += total;
        }
        __syncthreads();
        idx_cut = sm.cut;
      } else if (r_tie == n_tie) {
        idx_cut = INT_MAX;
      }
    }
    fk_comp = fk < n_gt ? sm.list[fk] : ~0ull;
    z_kept = (n_tie - r_tie) * e_piv + block_sum(tid >= fk ? e_t : 0.f, sm);
  } else {
    // ---- no top-k (then p == 1): the full softmax
    float bs = -INFINITY;
    int bi = INT_MAX;
    for (int i = tid; i < V; i += SP_THREADS) {
      const float kf = static_cast<float>(bf16_key(x[i]));
      if (arg_better(kf, i, bs, bi)) bs = kf, bi = i;
    }
    block_argmax(bs, bi, sm);
    m = key_to_float(static_cast<uint32_t>(bs)) / temp;
    float zs = 0.f;
    for (int i = tid; i < V; i += SP_THREADS) zs += expf(__uint_as_float(static_cast<uint32_t>(x[i]) << 16) / temp - m);
    z_kept = block_sum(zs, sm);
  }

  // ---- Gumbel-max over the kept set; the normalised distribution to probs_out
  const uint64_t off = ROWS ? offsets[row] : p.rng_offset ? *p.rng_offset : 0ull;
  const uint32_t noise_row = ROWS ? static_cast<uint32_t>(noise_rows[row]) : static_cast<uint32_t>(row);
  const float inv_z = 1.f / z_kept;
  float bs = -INFINITY;
  int bi = INT_MAX;
  for (int i = tid; i < V; i += SP_THREADS) {
    const uint32_t key = bf16_key(x[i]);
    bool keep = true;
    if (k > 0) {
      const unsigned long long comp = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(i);
      keep = key > pivot ? comp >= fk_comp : (key == pivot && i > idx_cut);
    }
    float pr = 0.f;
    if (keep) {
      const float s = key_to_float(key) / temp;
      pr = expf(s - m) * inv_z;
      const float g = gumbel(philox_x0(static_cast<uint32_t>(i), noise_row, static_cast<uint32_t>(off),
                                       static_cast<uint32_t>(off >> 32), p.seed_lo, p.seed_hi));
      const float sc = s + g;
      if (arg_better(sc, i, bs, bi)) bs = sc, bi = i;
    }
    if (probs) probs[i] = pr;
  }
  block_argmax(bs, bi, sm);
  if (tid == 0) p.next_ids[row] = bi;
}

__global__ void __launch_bounds__(SP_THREADS, 1) sample_kernel(const SampleParams p) {
  sample_body<false>(p, nullptr, nullptr);
}

__global__ void __launch_bounds__(SP_THREADS, 1) sample_rows_kernel(const SampleParams p, const int32_t* __restrict__ noise_rows,
                                                                    const uint64_t* __restrict__ offsets) {
  sample_body<true>(p, noise_rows, offsets);
}

__global__ void __launch_bounds__(SP_THREADS, 1) sample_slots_kernel(const SampleParams p, const int32_t* __restrict__ noise_rows,
                                                                     const uint64_t* __restrict__ offsets, const SlotSampling slots) {
  sample_body<true, true>(p, noise_rows, offsets, slots);
}

}  // namespace aria

using namespace aria;

// the checks and parameters the two entries share
static int sample_params(SampleParams& p, const void* logits, int64_t logits_stride, int64_t* next_ids, float* probs_out, int32_t B,
                         int32_t V, float temperature, int32_t top_k, float top_p, uint64_t seed, const uint64_t* rng_offset) {
  ARIA_CHECK_ARG(logits && next_ids);
  ARIA_CHECK_ARG(B > 0 && B <= SP_MAX_ROWS && V > 0 && V <= SP_MAX_VOCAB && logits_stride >= 0);
  ARIA_CHECK_ARG(temperature >= 0.f && temperature <= FLT_MAX);  // also rejects NaN and +inf
  ARIA_CHECK_ARG(top_k >= 0 && top_k <= SP_MAX_K);
  ARIA_CHECK_ARG(top_p > 0.f && top_p <= 1.f);
  if (top_k == 0 && top_p < 1.f) return ARIA_ERR_UNSUPPORTED;  // a full-vocabulary nucleus needs a full sort
  p.logits = static_cast<const uint16_t*>(logits);
  p.stride = logits_stride;
  p.next_ids = next_ids;
  p.probs = probs_out;
  p.V = V;
  p.temperature = temperature;
  p.top_k = top_k;
  p.top_p = top_p;
  p.seed_lo = static_cast<uint32_t>(seed);
  p.seed_hi = static_cast<uint32_t>(seed >> 32);
  p.rng_offset = rng_offset;
  return ARIA_OK;
}

extern "C" int aria_sample_tokens(const void* logits, int64_t logits_stride, int64_t* next_ids, float* probs_out, int32_t B,
                                  int32_t V, float temperature, int32_t top_k, float top_p, uint64_t seed,
                                  const uint64_t* rng_offset, aria_stream_t stream_) {
  SampleParams p{};
  const int rc = sample_params(p, logits, logits_stride, next_ids, probs_out, B, V, temperature, top_k, top_p, seed, rng_offset);
  if (rc) return rc;
  sample_kernel<<<B, SP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("sample_kernel");
}

extern "C" int aria_sample_tokens_rows(const void* logits, int64_t logits_stride, int64_t* next_ids, int32_t R, int32_t V,
                                       float temperature, int32_t top_k, float top_p, uint64_t seed, const int32_t* noise_rows,
                                       const uint64_t* offsets, aria_stream_t stream_) {
  ARIA_CHECK_ARG(noise_rows && offsets);
  SampleParams p{};
  const int rc = sample_params(p, logits, logits_stride, next_ids, nullptr, R, V, temperature, top_k, top_p, seed, nullptr);
  if (rc) return rc;
  sample_rows_kernel<<<R, SP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p, noise_rows, offsets);
  return check_launch("sample_rows_kernel");
}

extern "C" int aria_sample_tokens_slots(const void* logits, int64_t logits_stride, int64_t* next_ids, int32_t R, int32_t V,
                                        const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seed,
                                        const int32_t* noise_rows, const uint64_t* offsets, aria_stream_t stream_) {
  ARIA_CHECK_ARG(noise_rows && offsets && temperature && top_k && top_p && seed);
  SampleParams p{};
  const int rc = sample_params(p, logits, logits_stride, next_ids, nullptr, R, V, 0.f, 0, 1.f, 0, nullptr);
  if (rc) return rc;
  sample_slots_kernel<<<R, SP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p, noise_rows, offsets,
                                                                                      SlotSampling{temperature, top_k, top_p, seed});
  return check_launch("sample_slots_kernel");
}
