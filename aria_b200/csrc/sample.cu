// Next-token sampling for generation, sm_90a.
//
// aria_sample_tokens: Hugging Face's warper chain on an fp32 copy of bf16 logits, one CTA of 1024 threads per row:
//   TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> softmax -> multinomial.
//   Values compare as torch compares them: -0 and +0 are one value, tied like any other equal logits.
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
//
// aria_sample_tokens_processed: aria_sample_tokens_slots behind Hugging Face's logits processors, each row with its own:
//   RepetitionPenaltyLogitsProcessor -> MinNewTokensLengthLogitsProcessor -> (sampling) the warpers above -> MinPLogitsWarper.
//   Every score is the fp32 value of the bf16 logit, divided (IEEE, __fdiv_rn) or multiplied by the penalty when the id is set in
//   the row's presence bitmap (loaded to shared memory), or -inf for an EOS id while fewer than min_new tokens are out.  Such
//   scores are no longer bf16 values, so the select, the top-p list and the argmax run on the 32-bit order-preserving key of the
//   fp32 score (four 8-bit histogram passes); for a bf16-valued score it orders exactly as the 16-bit key, so a row whose
//   processors are off gets aria_sample_tokens' token and probabilities bit for bit.  Min-p is a cut in the final pass: kept
//   entries with p < min_p * p_max, p over the top-k / top-p survivors, are removed (the largest has p_max).
// aria_presence_set: the bits of an id matrix into those bitmaps.
//
// aria_token_logprobs: the log-probability of a token under a row's raw distribution and the row's top n (n <= 20) by (value
// desc, id asc), one CTA per row, reusing the radix select above (see token_logprobs_kernel).
#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace aria {

constexpr int SP_THREADS = 1024;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr int SP_MAX_K = 1024;
constexpr int32_t SP_MAX_ROWS = 1 << 20;
constexpr int32_t SP_MAX_VOCAB = 1 << 24;
constexpr int32_t SP_PROC_MAX_VOCAB = 1 << 18;  // the presence bitmap (V / 32 words) fits the shared memory left beside SampleSmem
constexpr int SP_MAX_EOS = 8;

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

// order-preserving 16-bit key of a bf16 bit pattern (larger key = larger value) and its inverse.  -0 is keyed as +0: the two
// compare equal in torch and transformers, so they tie (argmax and top-k ties, the stable top-p order, the top-n list).
__device__ __forceinline__ uint32_t bf16_key(uint32_t u) {
  u = u == 0x8000u ? 0u : u;
  return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
  const uint32_t u = (k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu);
  return __uint_as_float(u << 16);
}
// the same for an fp32 value: the 32-bit key of the processed scores (-0 keyed as +0 here too)
__device__ __forceinline__ uint32_t f32_key(float f) {
  uint32_t u = __float_as_uint(f);
  u = u == 0x80000000u ? 0u : u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_key_to_float(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

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
  unsigned long long red_u[SP_WARPS];
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

// Block maximum of (key << 32) | ~index entries: the largest key, ties to the lowest index.
__device__ unsigned long long block_max_u64(unsigned long long v, SampleSmem& sm) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sm.red_u[warp] = v;
  __syncthreads();
  v = lane < SP_WARPS ? sm.red_u[lane] : 0ull;
#pragma unroll
  for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
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

// Per-row logits processors of aria_sample_tokens_processed
struct Processing {
  const float* min_p;          // [R]
  const float* penalty;        // [R], repetition penalty
  const int32_t* min_new;      // [R]
  const uint32_t* presence;    // [R, words] bitmaps
  const int32_t* n_emitted;    // [R] (emitted_per_row) or [1]: tokens the row has emitted
  int emitted_per_row, offset_per_row, words, n_eos;
  int eos[SP_MAX_EOS];         // EOS ids inside [0, V)
};

// ROWS (aria_sample_tokens_rows): logits row `row` draws the noise of row noise_rows[row] at offset offsets[row] instead of
// (row, *p.rng_offset).  SLOTS (with ROWS): the row's temperature, top_k, top_p and seed come from `slots`, brought into the
// ranges aria_sample_tokens accepts (a caller checks them; this keeps a bad entry from reading past shared memory).
// PROC (with SLOTS): the row's scores are its processed logits (`proc`), keyed by 32 bits; the noise row is noise_rows[row] or
// row when noise_rows is NULL, the offset offsets[row] or offsets[0].  Everything else is the same code.
template <bool ROWS, bool SLOTS = false, bool PROC = false>
__device__ __forceinline__ void sample_body(SampleParams p, const int32_t* __restrict__ noise_rows,
                                            const uint64_t* __restrict__ offsets, const SlotSampling slots = {},
                                            const Processing& proc = {}) {
  __shared__ SampleSmem sm;
  extern __shared__ uint32_t presence_sm[];  // PROC: the row's presence bitmap
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

  float penalty = 1.f, min_p = 0.f;
  bool no_eos = false;
  if constexpr (PROC) {
    const float pen = proc.penalty[row], mp = proc.min_p[row];
    penalty = pen > 0.f && pen <= FLT_MAX ? pen : 1.f;
    min_p = mp > 0.f && mp <= 1.f ? mp : 0.f;
    no_eos = proc.n_eos > 0 && proc.n_emitted[proc.emitted_per_row ? row : 0] < proc.min_new[row];
    if (penalty != 1.f) {
      const uint32_t* src = proc.presence + static_cast<int64_t>(row) * proc.words;
      for (int w = tid; w < proc.words; w += SP_THREADS) presence_sm[w] = src[w];
    }
    __syncthreads();
  }
  // the score of id i (Hugging Face's fp32 copy of the logit, processed) and its order-preserving key; key_value inverts it
  auto score = [&](int i) -> float {
    float v = __uint_as_float(static_cast<uint32_t>(x[i]) << 16);
    if constexpr (PROC) {
      if (penalty != 1.f && ((presence_sm[i >> 5] >> (i & 31)) & 1u)) v = v < 0.f ? __fmul_rn(v, penalty) : __fdiv_rn(v, penalty);
      if (no_eos) {
#pragma unroll
        for (int e = 0; e < SP_MAX_EOS; ++e)
          if (e < proc.n_eos && i == proc.eos[e]) v = -INFINITY;
      }
    }
    return v;
  };
  auto key_at = [&](int i) -> uint32_t {
    if constexpr (PROC) return f32_key(score(i));
    else return bf16_key(x[i]);
  };
  auto key_value = [&](uint32_t key) -> float {
    if constexpr (PROC) return f32_key_to_float(key);
    else return key_to_float(key);
  };
  // the largest key of the row, ties to the lowest id -> (key, id)
  auto argmax_key = [&](uint32_t& key, int& id) {
    unsigned long long b = 0;
    for (int i = tid; i < V; i += SP_THREADS) b = max(b, (static_cast<unsigned long long>(key_at(i)) << 32) | (0xFFFFFFFFu - i));
    b = block_max_u64(b, sm);
    key = static_cast<uint32_t>(b >> 32);
    id = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(b));
  };

  if (p.temperature == 0.f) {  // greedy
    uint32_t bk;
    int bi;
    argmax_key(bk, bi);
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
    // ---- radix select of the k-th largest key, one byte at a time from the top (16-bit keys: two passes, 32-bit: four)
    constexpr int KEY_BITS = PROC ? 32 : 16;
    if (tid == 0) sm.n_list = 0;
#pragma unroll
    for (int shift = KEY_BITS - 8; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += SP_THREADS) sm.hist[i] = 0;
      __syncthreads();
      for (int i = tid; i < V; i += SP_THREADS) {
        const uint32_t key = key_at(i);
        if (shift == KEY_BITS - 8 || (key >> (shift + 8)) == pivot) atomicAdd(&sm.hist[(key >> shift) & 0xFF], 1u);
      }
      find_bin(sm, k - n_gt);
      pivot = (pivot << 8) | sm.bin;  // the key prefix selected so far
      n_gt += sm.above;
    }
    n_tie = static_cast<int>(sm.hist[sm.bin]);
    // ---- compact the keys above the pivot (n_gt < k of them) and sort them ascending by (key, index)
    for (int i = tid; i < V; i += SP_THREADS) {
      const uint32_t key = key_at(i);
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
    const float s_piv = key_value(pivot) / temp;
    const bool mine = tid < n_gt;
    const float s_t = mine ? key_value(static_cast<uint32_t>(sm.list[tid] >> 32)) / temp : -INFINITY;
    m = n_gt > 0 ? key_value(static_cast<uint32_t>(sm.list[n_gt - 1] >> 32)) / temp : s_piv;
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
          const bool t = i < V && key_at(i) == pivot;
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
    uint32_t bk;
    int bi;
    argmax_key(bk, bi);
    m = key_value(bk) / temp;
    float zs = 0.f;
    for (int i = tid; i < V; i += SP_THREADS) zs += expf(score(i) / temp - m);
    z_kept = block_sum(zs, sm);
  }

  // ---- Gumbel-max over the kept set; the normalised distribution to probs_out
  uint64_t off;
  uint32_t noise_row;
  if constexpr (PROC) {
    off = offsets[proc.offset_per_row ? row : 0];
    noise_row = noise_rows ? static_cast<uint32_t>(noise_rows[row]) : static_cast<uint32_t>(row);
  } else {
    off = ROWS ? offsets[row] : p.rng_offset ? *p.rng_offset : 0ull;
    noise_row = ROWS ? static_cast<uint32_t>(noise_rows[row]) : static_cast<uint32_t>(row);
  }
  const float inv_z = 1.f / z_kept;
  // whether id i (key `key`) is in the final set; then s = its scaled score and e = exp(s - m).  Min-p: p = e / z_kept over the
  // top-k / top-p set, whose largest entry has e = 1, so p < min_p * p_max is e * inv_z < min_p * inv_z (never with min_p 0)
  auto kept = [&](int i, uint32_t key, float& s, float& e) -> bool {
    if (k > 0) {
      const unsigned long long comp = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(i);
      if (!(key > pivot ? comp >= fk_comp : (key == pivot && i > idx_cut))) return false;
    }
    s = key_value(key) / temp;
    e = expf(s - m);
    if constexpr (PROC) return !(e * inv_z < min_p * inv_z);
    return true;
  };
  float inv_zp = inv_z;  // the normaliser of probs_out: min-p renormalises over what it keeps
  if constexpr (PROC) {
    if (probs && min_p > 0.f) {
      float zs = 0.f;
      for (int i = tid; i < V; i += SP_THREADS) {
        float s, e;
        if (kept(i, key_at(i), s, e)) zs += e;
      }
      inv_zp = 1.f / block_sum(zs, sm);
    }
  }
  float bs = -INFINITY;
  int bi = INT_MAX;
  for (int i = tid; i < V; i += SP_THREADS) {
    float pr = 0.f, s, e;
    if (kept(i, key_at(i), s, e)) {
      pr = e * inv_zp;
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

// ---------------------------------------------------------------------------------------------------- token log-probabilities
constexpr int LP_MAX_N = 20;

struct LogprobParams {
  const uint16_t* logits;  // bf16 bits, row r at logits + r * stride
  int64_t stride;
  const int64_t* tokens;   // [R]
  const int32_t* n_row;    // [R] or NULL (every row n_max); -1 skips the row
  const int32_t* col;      // output column: col[r] (col_per_row) or col[0]; NULL: column 0
  int col_per_row;
  int ring;                // > 0: column col mod ring
  const uint8_t* finished; // [R] or NULL
  int finished_fill;       // finished rows: 1 write the filler, 0 leave untouched
  float* lp;               // [R, cols]
  int32_t* top_ids;        // [R, cols, n_max]
  float* top_lp;           // [R, cols, n_max]
  int cols, n_max, V;
};

// (m, s) <- the pair over the union; an empty side has m = -inf.  The compiler may contract one of the two products into an
// FMA, so the two lanes of a butterfly exchange can round differently: the caller takes one lane's result (lp_pass1).  expf,
// not __expf: the sum decides every logprob's last bits.
__device__ __forceinline__ void lp_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) {
    m = m2;
    s = s2;
    return;
  }
  const float M = fmaxf(m, m2);
  s = s * expf(m - M) + s2 * expf(m2 - M);
  m = M;
}

// one 8-element chunk of the row into the thread's (max, sum of exp) and, with HIST, the high-byte key histogram
template <bool HIST>
__device__ __forceinline__ void lp_add8(float& m, float& s, const uint32_t (&u)[8], int valid, SampleSmem& sm) {
  float x[8];
  float vm = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    x[j] = j < valid ? __uint_as_float(u[j] << 16) : -INFINITY;
    vm = fmaxf(vm, x[j]);
    if (HIST && j < valid) atomicAdd(&sm.hist[bf16_key(u[j]) >> 8], 1u);
  }
  if (vm == -INFINITY) return;  // nothing to add (also keeps -inf - -inf out of the exponents)
  if (vm > m) {
    s *= expf(m - vm);          // m = -inf: s is 0 already
    m = vm;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s += expf(x[j] - m);
}

// Chunk c (elements 8c .. 8c + 7) of a row always belongs to thread c mod SP_THREADS and is added in increasing c, whether it
// is read with one 128-bit load (a 16-byte aligned row) or with scalar loads, so the sum does not depend on the row's address.
template <bool HIST>
__device__ void lp_pass1(const uint16_t* __restrict__ x, int V, float& m, float& s, SampleSmem& sm) {
  const int tid = threadIdx.x, n_full = V >> 3;
  m = -INFINITY;
  s = 0.f;
  uint32_t u[8];
  if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const uint4* row = reinterpret_cast<const uint4*>(x);
    int c = tid;
    for (; c + 3 * SP_THREADS < n_full; c += 4 * SP_THREADS) {
      uint4 q[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = __ldg(row + c + i * SP_THREADS);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t a[4] = {q[i].x, q[i].y, q[i].z, q[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) u[2 * j] = a[j] & 0xFFFFu, u[2 * j + 1] = a[j] >> 16;
        lp_add8<HIST>(m, s, u, 8, sm);
      }
    }
    for (; c < n_full; c += SP_THREADS) {
      const uint4 q = __ldg(row + c);
      const uint32_t a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) u[2 * j] = a[j] & 0xFFFFu, u[2 * j + 1] = a[j] >> 16;
      lp_add8<HIST>(m, s, u, 8, sm);
    }
  } else {
    for (int c = tid; c < n_full; c += SP_THREADS) {
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = x[8 * c + j];
      lp_add8<HIST>(m, s, u, 8, sm);
    }
  }
  if ((V & 7) && tid == n_full % SP_THREADS) {  // the scalar tail, the last chunk of its thread
#pragma unroll
    for (int j = 0; j < 8; ++j) u[j] = 8 * n_full + j < V ? x[8 * n_full + j] : 0u;
    lp_add8<HIST>(m, s, u, V & 7, sm);
  }
  // fixed-order merge: xor butterfly in each warp, then the same over the warps' pairs
#pragma unroll
  for (int o = 16; o; o >>= 1) lp_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
  const int lane = tid & 31, warp = tid >> 5;
  __syncthreads();
  if (lane == 0) sm.red_f[warp] = m, sm.red_i[warp] = __float_as_int(s);
  __syncthreads();
  m = lane < SP_WARPS ? sm.red_f[lane] : -INFINITY;
  s = lane < SP_WARPS ? __int_as_float(sm.red_i[lane]) : 0.f;
#pragma unroll
  for (int o = 16; o; o >>= 1) lp_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
  // lane 0 of every warp ran the same operations on the same values: its pair is the row's, in every thread, so the token's
  // logprob (thread 0) and each top entry's (thread j) use the same m and log(s)
  m = __shfl_sync(0xffffffffu, m, 0);
  s = __shfl_sync(0xffffffffu, s, 0);
}

// logprob of token t in row x: (x_t - m) - log(s), the row's raw distribution.  Top n: the n largest logits by (value desc, id
// asc), found by the radix select of sample_body (find_bin on the high, then the low byte of the 16-bit key); the keys above
// the pivot (< n of them) and the lowest-id pivot ties are compacted and bitonic-sorted.  A row's result depends only on its
// logits, its token and its n.
__global__ void __launch_bounds__(SP_THREADS, 1) token_logprobs_kernel(const LogprobParams p) {
  __shared__ SampleSmem sm;
  const int tid = threadIdx.x, row = blockIdx.x, V = p.V;
  int n = p.n_max;
  if (p.n_row) {
    n = p.n_row[row];
    if (n < 0) return;
    n = min(n, p.n_max);
  }
  int c = 0;
  if (p.col) {
    c = p.col[p.col_per_row ? row : 0];
    if (p.ring > 0) c = ((c % p.ring) + p.ring) % p.ring;
    if (c < 0 || c >= p.cols) return;
  }
  const int64_t o = static_cast<int64_t>(row) * p.cols + c;
  float* top_lp = p.top_lp + o * p.n_max;
  int32_t* top_ids = p.top_ids + o * p.n_max;
  if (p.finished && p.finished[row]) {
    if (!p.finished_fill) return;
    if (tid == 0) p.lp[o] = 0.f;
    for (int j = tid; j < p.n_max; j += SP_THREADS) top_ids[j] = -1, top_lp[j] = -INFINITY;
    return;
  }
  const uint16_t* x = p.logits + static_cast<int64_t>(row) * p.stride;
  const int ne = min(n, V);  // real top entries; [ne, n_max) get the filler
  if (ne > 0)
    for (int i = tid; i < 256; i += SP_THREADS) sm.hist[i] = 0;
  if (tid == 0) sm.n_list = 0;
  __syncthreads();
  float m, s;
  if (ne > 0)
    lp_pass1<true>(x, V, m, s, sm);
  else
    lp_pass1<false>(x, V, m, s, sm);
  const float log_s = logf(s);  // s >= 1: the maximum contributes exp(0)
  if (tid == 0) {
    const int64_t t = p.tokens[row];
    p.lp[o] = t >= 0 && t < V ? (__uint_as_float(static_cast<uint32_t>(x[t]) << 16) - m) - log_s : __int_as_float(0x7fc00000);
  }
  for (int j = ne + tid; j < p.n_max; j += SP_THREADS) top_ids[j] = -1, top_lp[j] = -INFINITY;
  if (ne == 0) return;

  // ---- the ne-th largest key: high byte (histogram filled by pass 1), then the low byte within it
  find_bin(sm, ne);
  const uint32_t hb = sm.bin;
  const int above_hi = sm.above;
  for (int i = tid; i < 256; i += SP_THREADS) sm.hist[i] = 0;
  __syncthreads();
  for (int i = tid; i < V; i += SP_THREADS) {
    const uint32_t key = bf16_key(x[i]);
    if ((key >> 8) == hb) atomicAdd(&sm.hist[key & 0xFF], 1u);
  }
  find_bin(sm, ne - above_hi);
  const uint32_t pivot = (hb << 8) | sm.bin;
  const int n_gt = above_hi + sm.above;        // < ne
  const int n_tie = static_cast<int>(sm.hist[sm.bin]);
  const int need = ne - n_gt;                  // pivot ties taken, the lowest ids first
  // ---- compact: entries (~key << 32 | id) sort ascending as (value desc, id asc)
  const bool all_ties = n_tie <= SP_MAX_K - LP_MAX_N;  // else only the first `need` ties in id order, by an ordered scan
  for (int i = tid; i < V; i += SP_THREADS) {
    const uint32_t key = bf16_key(x[i]);
    if (key > pivot || (all_ties && key == pivot))
      sm.list[atomicAdd(&sm.n_list, 1)] = (static_cast<unsigned long long>(0xFFFFu - key) << 32) | static_cast<uint32_t>(i);
  }
  int total = n_gt + n_tie;
  if (!all_ties) {
    total = ne;
    const int lane = tid & 31, warp = tid >> 5;
    const unsigned long long piv = static_cast<unsigned long long>(0xFFFFu - pivot) << 32;
    int base = 0;
    for (int i0 = 0; i0 < V && base < need; i0 += SP_THREADS) {
      const int i = i0 + tid;
      const bool t = i < V && bf16_key(x[i]) == pivot;
      const unsigned bal = __ballot_sync(0xffffffffu, t);
      __syncthreads();
      if (lane == 0) sm.red_i[warp] = __popc(bal);
      __syncthreads();
      int before = base + __popc(bal & ((1u << lane) - 1u)), sum = 0;
      for (int w = 0; w < SP_WARPS; ++w) {
        const int cnt = sm.red_i[w];
        if (w < warp) before += cnt;
        sum += cnt;
      }
      if (t && before < need) sm.list[n_gt + before] = piv | static_cast<uint32_t>(i);
      base += sum;
    }
  }
  __syncthreads();
  int P = 1;
  while (P < total) P <<= 1;
  for (int i = total + tid; i < P; i += SP_THREADS) sm.list[i] = ~0ull;
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
  if (tid < ne) {
    const unsigned long long e = sm.list[tid];
    const uint32_t key = 0xFFFFu - static_cast<uint32_t>(e >> 32);
    top_ids[tid] = static_cast<int32_t>(e & 0xFFFFFFFFu);
    top_lp[tid] = (key_to_float(key) - m) - log_s;
  }
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

__global__ void __launch_bounds__(SP_THREADS, 1) sample_processed_kernel(const SampleParams p, const int32_t* __restrict__ noise_rows,
                                                                         const uint64_t* __restrict__ offsets,
                                                                         const SlotSampling slots, const Processing proc) {
  sample_body<true, true, true>(p, noise_rows, offsets, slots, proc);
}

// One CTA per row: optionally clear the row's bitmap, then set the bits of its first n ids (ids outside [0, V) are skipped).
constexpr int PS_THREADS = 256;
__global__ void __launch_bounds__(PS_THREADS) presence_set_kernel(const int64_t* __restrict__ ids, int64_t ids_stride, int32_t T,
                                                                  const int32_t* __restrict__ lengths, int32_t clear,
                                                                  uint32_t* __restrict__ bitmap, int32_t V, int32_t words) {
  const int r = blockIdx.x;
  uint32_t* bm = bitmap + static_cast<int64_t>(r) * words;
  if (clear) {
    for (int w = threadIdx.x; w < words; w += PS_THREADS) bm[w] = 0u;
    __syncthreads();
  }
  const int n = lengths ? min(max(lengths[r], 0), T) : T;
  const int64_t* row = ids + static_cast<int64_t>(r) * ids_stride;
  for (int t = threadIdx.x; t < n; t += PS_THREADS) {
    const int64_t id = row[t];
    if (id >= 0 && id < V) atomicOr(bm + (id >> 5), 1u << (id & 31));
  }
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

extern "C" int aria_sample_tokens_processed(const void* logits, int64_t logits_stride, int64_t* next_ids, float* probs_out,
                                            int32_t R, int32_t V, const float* temperature, const int32_t* top_k, const float* top_p,
                                            const float* min_p, const uint64_t* seed, const float* repetition_penalty,
                                            const int32_t* min_new_tokens, const uint32_t* presence, const int32_t* noise_rows,
                                            const uint64_t* rng_offset, int32_t offset_per_row, const int32_t* n_emitted,
                                            int32_t emitted_per_row, const int64_t* eos_ids, int32_t n_eos, aria_stream_t stream_) {
  ARIA_CHECK_ARG(temperature && top_k && top_p && min_p && seed && repetition_penalty && min_new_tokens && presence && rng_offset &&
                 n_emitted);
  ARIA_CHECK_ARG(V > 0 && V <= SP_PROC_MAX_VOCAB);
  ARIA_CHECK_ARG(n_eos >= 0 && n_eos <= SP_MAX_EOS && (n_eos == 0 || eos_ids));
  SampleParams p{};
  const int rc = sample_params(p, logits, logits_stride, next_ids, probs_out, R, V, 0.f, 0, 1.f, 0, nullptr);
  if (rc) return rc;
  Processing proc{};
  proc.min_p = min_p;
  proc.penalty = repetition_penalty;
  proc.min_new = min_new_tokens;
  proc.presence = presence;
  proc.n_emitted = n_emitted;
  proc.emitted_per_row = emitted_per_row != 0;
  proc.offset_per_row = offset_per_row != 0;
  proc.words = (V + 31) / 32;
  for (int e = 0; e < n_eos; ++e)  // host array; an id outside the vocabulary has no score to mask
    if (eos_ids[e] >= 0 && eos_ids[e] < V) proc.eos[proc.n_eos++] = static_cast<int>(eos_ids[e]);
  const size_t smem = sizeof(uint32_t) * proc.words;
  sample_processed_kernel<<<R, SP_THREADS, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      p, noise_rows, rng_offset, SlotSampling{temperature, top_k, top_p, seed}, proc);
  return check_launch("sample_processed_kernel");
}

extern "C" int aria_presence_set(const int64_t* ids, int64_t ids_stride, int32_t R, int32_t T, const int32_t* lengths,
                                 int32_t clear, uint32_t* bitmap, int32_t V, aria_stream_t stream_) {
  ARIA_CHECK_ARG(ids && bitmap);
  ARIA_CHECK_ARG(R > 0 && R <= SP_MAX_ROWS && T > 0 && ids_stride >= 0 && V > 0 && V <= SP_PROC_MAX_VOCAB);
  presence_set_kernel<<<R, PS_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(ids, ids_stride, T, lengths, clear != 0,
                                                                                     bitmap, V, (V + 31) / 32);
  return check_launch("presence_set_kernel");
}

extern "C" int aria_token_logprobs(const void* logits, int64_t logits_stride, const int64_t* tokens, int32_t R, int32_t V,
                                   int32_t n_max, const int32_t* n_row, const int32_t* col, int32_t col_per_row, int32_t ring,
                                   const uint8_t* finished, int32_t finished_fill, float* logprobs, int32_t* top_ids,
                                   float* top_logprobs, int32_t cols, aria_stream_t stream_) {
  ARIA_CHECK_ARG(logits && tokens && logprobs);
  ARIA_CHECK_ARG(R > 0 && R <= SP_MAX_ROWS && V > 0 && V <= SP_MAX_VOCAB && logits_stride >= 0);
  ARIA_CHECK_ARG(n_max >= 0 && n_max <= LP_MAX_N && (n_max == 0 || (top_ids && top_logprobs)));
  ARIA_CHECK_ARG(cols >= 1 && ring >= 0 && ring <= cols && (col || (ring == 0 && col_per_row == 0)));
  ARIA_CHECK_ARG(finished_fill == 0 || finished_fill == 1);
  LogprobParams p{};
  p.logits = static_cast<const uint16_t*>(logits);
  p.stride = logits_stride;
  p.tokens = tokens;
  p.n_row = n_row;
  p.col = col;
  p.col_per_row = col_per_row != 0;
  p.ring = ring;
  p.finished = finished;
  p.finished_fill = finished_fill;
  p.lp = logprobs;
  p.top_ids = top_ids;
  p.top_lp = top_logprobs;
  p.cols = cols;
  p.n_max = n_max;
  p.V = V;
  token_logprobs_kernel<<<R, SP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("token_logprobs_kernel");
}
