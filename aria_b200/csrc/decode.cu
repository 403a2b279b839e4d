// The two small kernels that let one captured decode step be replayed token after token: every position they use is read
// from device memory, so nothing in the step is a host integer.
//
// aria_kv_append: copies the step's k and v rows ([B, H, 128] staging rows written by the q/k/v projection) into the cache
//   at the device row pos[b].
// aria_kv_scatter_tails: copies the packed suffix k and v rows of a shared-prefix prefill into the n tails of each prompt.
// aria_decode_advance: after the sampler, feeds next_ids back as the next step's input, records the token, applies
//   Hugging Face's EOS rule and advances the RoPE positions, the cache rows, the step index and the RNG offset.
#include <cuda_bf16.h>

#include "common.cuh"

namespace aria {

constexpr int KV_ROW_VECS = 16;  // a 128-wide bf16 row is 16 x 16 bytes

__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_append_kernel(const __nv_bfloat16* __restrict__ k_new,
                                                                    const __nv_bfloat16* __restrict__ v_new, int64_t new_sb,
                                                                    int64_t new_sh, __nv_bfloat16* __restrict__ kc,
                                                                    __nv_bfloat16* __restrict__ vc, int64_t c_sb, int64_t c_sh,
                                                                    const int32_t* __restrict__ pos, int H, int T_max) {
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int p = pos[b];
  if (p < 0 || p >= T_max) return;  // never past the cache
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const __nv_bfloat16* src = (is_v ? v_new : k_new) + b * new_sb + h * new_sh;
  __nv_bfloat16* dst = (is_v ? vc : kc) + b * c_sb + h * c_sh + static_cast<int64_t>(p) * 128;
  reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
}

// One CTA per (packed row s, head h): row s of segment b goes to tail row s - cu[b] of rows b * n .. b * n + n - 1
__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_scatter_tails_kernel(const __nv_bfloat16* __restrict__ k,
                                                                           const __nv_bfloat16* __restrict__ v, int64_t src_sh,
                                                                           __nv_bfloat16* __restrict__ tk, __nv_bfloat16* __restrict__ tv,
                                                                           int64_t t_sb, int64_t t_sh, const int32_t* __restrict__ cu,
                                                                           int B, int n, int H, int N_max) {
  const int s = blockIdx.x / H, h = blockIdx.x % H;
  const int b = packed_segment(cu, B, s);
  const int row = s - cu[b];
  if (row < 0 || row >= N_max) return;  // never past the tails
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const uint4 x = reinterpret_cast<const uint4*>((is_v ? v : k) + h * src_sh + static_cast<int64_t>(s) * 128)[j];
  __nv_bfloat16* dst = (is_v ? tv : tk) + h * t_sh + static_cast<int64_t>(row) * 128;
  for (int c = 0; c < n; ++c) reinterpret_cast<uint4*>(dst + static_cast<int64_t>(b * n + c) * t_sb)[j] = x;
}

constexpr int ADV_MAX_EOS = 8;
constexpr int ADV_MAX_B = 1024;

struct AdvanceParams {
  const int64_t* next_ids;
  int64_t* ids_in;
  int64_t* out_tokens;  // [B, max_steps]
  int32_t max_steps;
  int32_t* step;
  int32_t* rope_pos;
  int32_t* write_pos;
  int32_t* kv_len;
  uint64_t* rng_offset;
  uint8_t* finished;
  int32_t* done_step;
  int64_t eos[ADV_MAX_EOS];
  int32_t n_eos;
  int64_t pad;
  int32_t B;
};

__global__ void __launch_bounds__(ADV_MAX_B) decode_advance_kernel(const AdvanceParams p) {
  const int b = threadIdx.x;
  const int t = *p.step;
  bool fin = true;
  if (b < p.B) {
    // GenerationMixin._sample: a finished row emits pad; a row finishes when the token it emits is an EOS id
    const bool was = p.finished[b] != 0;
    const int64_t tok = was ? p.pad : p.next_ids[b];
    if (t < p.max_steps) p.out_tokens[static_cast<int64_t>(b) * p.max_steps + t] = tok;
    p.ids_in[b] = tok;
    bool now = was;
    for (int e = 0; e < p.n_eos; ++e) now |= tok == p.eos[e];
    p.finished[b] = now;
    fin = now;
    ++p.rope_pos[b];
    ++p.write_pos[b];
    ++p.kv_len[b];
  }
  const bool all = __syncthreads_and(fin);  // every thread has read *p.step
  if (b == 0) {
    *p.step = t + 1;
    *p.rng_offset += 1;
    if (all && p.n_eos > 0 && *p.done_step < 0) *p.done_step = t;
  }
}

}  // namespace aria

using namespace aria;

extern "C" int aria_kv_append(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_cache,
                              void* v_cache, int64_t cache_stride_b, int64_t cache_stride_h, const int32_t* pos, int32_t B,
                              int32_t H, int32_t T_max, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_new && v_new && k_cache && v_cache && pos);
  ARIA_CHECK_ARG(B > 0 && H > 0 && T_max > 0 && static_cast<int64_t>(B) * H < (1ll << 31));
  ARIA_CHECK_ARG(new_stride_b % 8 == 0 && new_stride_h % 8 == 0 && cache_stride_b % 8 == 0 && cache_stride_h % 8 == 0);
  kv_append_kernel<<<B * H, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k_new), static_cast<const __nv_bfloat16*>(v_new), new_stride_b, new_stride_h,
      static_cast<__nv_bfloat16*>(k_cache), static_cast<__nv_bfloat16*>(v_cache), cache_stride_b, cache_stride_h, pos, H, T_max);
  return check_launch("kv_append_kernel");
}

extern "C" int aria_kv_scatter_tails(const void* k, const void* v, int64_t src_stride_h, void* tail_k, void* tail_v,
                                     int64_t tail_stride_b, int64_t tail_stride_h, const int32_t* cu_seqlens, int32_t B, int32_t n,
                                     int32_t H, int32_t S_tot, int32_t N_max, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k && v && tail_k && tail_v && cu_seqlens);
  ARIA_CHECK_ARG(B > 0 && n > 0 && H > 0 && S_tot >= B && N_max > 0);
  ARIA_CHECK_ARG(static_cast<int64_t>(S_tot) * H < (1ll << 31) && static_cast<int64_t>(B) * n < (1ll << 31));
  ARIA_CHECK_ARG(src_stride_h >= static_cast<int64_t>(S_tot) * 128 && tail_stride_h >= static_cast<int64_t>(N_max) * 128);
  ARIA_CHECK_ARG(tail_stride_b >= tail_stride_h * H);  // tails of different rows do not overlap
  ARIA_CHECK_ARG(src_stride_h % 8 == 0 && tail_stride_b % 8 == 0 && tail_stride_h % 8 == 0);
  kv_scatter_tails_kernel<<<S_tot * H, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v), src_stride_h, static_cast<__nv_bfloat16*>(tail_k),
      static_cast<__nv_bfloat16*>(tail_v), tail_stride_b, tail_stride_h, cu_seqlens, B, n, H, N_max);
  return check_launch("kv_scatter_tails_kernel");
}

extern "C" int aria_decode_advance(const int64_t* next_ids, int64_t* ids_in, int64_t* out_tokens, int32_t max_steps, int32_t* step,
                                   int32_t* rope_pos, int32_t* write_pos, int32_t* kv_len, uint64_t* rng_offset, uint8_t* finished,
                                   int32_t* done_step, const int64_t* eos_ids, int32_t n_eos, int64_t pad_token_id, int32_t B,
                                   aria_stream_t stream_) {
  ARIA_CHECK_ARG(next_ids && ids_in && out_tokens && step && rope_pos && write_pos && kv_len && rng_offset && finished && done_step);
  ARIA_CHECK_ARG(B > 0 && B <= ADV_MAX_B && max_steps > 0);
  ARIA_CHECK_ARG(n_eos >= 0 && n_eos <= ADV_MAX_EOS && (n_eos == 0 || eos_ids));
  AdvanceParams p{};
  p.next_ids = next_ids;
  p.ids_in = ids_in;
  p.out_tokens = out_tokens;
  p.max_steps = max_steps;
  p.step = step;
  p.rope_pos = rope_pos;
  p.write_pos = write_pos;
  p.kv_len = kv_len;
  p.rng_offset = rng_offset;
  p.finished = finished;
  p.done_step = done_step;
  for (int e = 0; e < n_eos; ++e) p.eos[e] = eos_ids[e];  // host array, copied into the launch parameters
  p.n_eos = n_eos;
  p.pad = pad_token_id;
  p.B = B;
  const int threads = (B + 31) / 32 * 32;
  decode_advance_kernel<<<1, threads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("decode_advance_kernel");
}
