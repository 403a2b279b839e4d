// The two small kernels that let one captured decode step be replayed token after token: every position they use is read
// from device memory, so nothing in the step is a host integer.
//
// aria_kv_append: copies the step's k and v rows ([B, H, 128] staging rows written by the q/k/v projection) into the cache
//   at the device row pos[b].
// aria_kv_scatter_tails: copies the packed suffix k and v rows of a shared-prefix prefill into the n tails of each prompt.
// aria_decode_advance_slots: after the sampler, feeds each row's token back as the next step's input, records it, applies
//   Hugging Face's EOS rule and the row's budget, and advances the row's RoPE position, cache row, output count and RNG offset.
//
// Continuous batching (serving.Engine) over a paged KV cache, pools [n_pages, H, 256, 128] and a block table [R, max_pages]:
// aria_kv_append_paged: kv_append into the page block_table[r, write_pos[r] / 256], row write_pos[r] % 256.  A negative
//   write_pos, or one outside the row's mapped pages, writes nothing: idle and finished slots never touch another's pages.
// aria_kv_pages_store: copies rows [0, T) of a one-row prefill cache into a request's pages.
// aria_kv_pages_store_varlen: the same for packed segments, each into its own pages after its own prefix.
//
// Prompt-lookup decoding (generate(prompt_lookup_num_tokens=K)): a step verifies Q = K + 1 tokens per row.
// aria_kv_append_rows: kv_append for the Q rows of each row, at cache rows pos[b] + i.
// aria_ngram_draft: Hugging Face's PromptLookupCandidateGenerator.get_candidates on each row's history, one CTA per row.
// aria_lookup_accept_advance: accepts each row's drafts against the sampled targets, emits the accepted run plus one token,
//   applies the EOS rule and moves the row's positions on by the count emitted.
#include <climits>

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

// One CTA per (row b, head h, query i): row i of the step goes to cache row pos[b] + i
__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_append_rows_kernel(const __nv_bfloat16* __restrict__ k_new,
                                                                         const __nv_bfloat16* __restrict__ v_new, int64_t new_sb,
                                                                         int64_t new_sh, int64_t new_sq, __nv_bfloat16* __restrict__ kc,
                                                                         __nv_bfloat16* __restrict__ vc, int64_t c_sb, int64_t c_sh,
                                                                         const int32_t* __restrict__ pos, int H, int Q, int T_max) {
  const int i = blockIdx.x % Q, bh = blockIdx.x / Q, b = bh / H, h = bh % H;
  const int p = pos[b] + i;
  if (p < 0 || p >= T_max) return;  // never past the cache
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const __nv_bfloat16* src = (is_v ? v_new : k_new) + b * new_sb + h * new_sh + i * new_sq;
  __nv_bfloat16* dst = (is_v ? vc : kc) + b * c_sb + h * c_sh + static_cast<int64_t>(p) * 128;
  reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
}

constexpr int ADV_MAX_EOS = 8;
constexpr int ADV_MAX_B = 1024;

// One CTA per (slot r, head h)
__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_append_paged_kernel(const __nv_bfloat16* __restrict__ k_new,
                                                                          const __nv_bfloat16* __restrict__ v_new, int64_t new_sb,
                                                                          int64_t new_sh, __nv_bfloat16* __restrict__ kp,
                                                                          __nv_bfloat16* __restrict__ vp, int64_t page_stride,
                                                                          int64_t pool_sh, const int32_t* __restrict__ bt,
                                                                          int64_t bt_stride, int max_pages, int n_pages,
                                                                          const int32_t* __restrict__ pos, int H) {
  const int r = blockIdx.x / H, h = blockIdx.x % H;
  const int p = pos[r];
  const int page = page_of(bt + r * bt_stride, max_pages, n_pages, p);
  if (page < 0) return;
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const __nv_bfloat16* src = (is_v ? v_new : k_new) + r * new_sb + h * new_sh;
  __nv_bfloat16* dst = (is_v ? vp : kp) + page * page_stride + h * pool_sh + static_cast<int64_t>(p % PAGE_ROWS) * 128;
  reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
}

// One CTA per (row t, head h) of the prefill cache
__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_pages_store_kernel(const __nv_bfloat16* __restrict__ k,
                                                                         const __nv_bfloat16* __restrict__ v, int64_t src_sh,
                                                                         __nv_bfloat16* __restrict__ kp, __nv_bfloat16* __restrict__ vp,
                                                                         int64_t page_stride, int64_t pool_sh,
                                                                         const int32_t* __restrict__ pages, int max_pages,
                                                                         int n_pages, int H) {
  const int t = blockIdx.x / H, h = blockIdx.x % H;
  const int page = page_of(pages, max_pages, n_pages, t);
  if (page < 0) return;
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const uint4 x = reinterpret_cast<const uint4*>((is_v ? v : k) + h * src_sh + static_cast<int64_t>(t) * 128)[j];
  __nv_bfloat16* dst = (is_v ? vp : kp) + page * page_stride + h * pool_sh + static_cast<int64_t>(t % PAGE_ROWS) * 128;
  reinterpret_cast<uint4*>(dst)[j] = x;
}

// One CTA per (packed row t, head h): row t of segment b is position P_b + t - cu[b] of its request
__global__ void __launch_bounds__(2 * KV_ROW_VECS) kv_pages_store_varlen_kernel(
    const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v, int64_t src_sh, __nv_bfloat16* __restrict__ kp,
    __nv_bfloat16* __restrict__ vp, int64_t page_stride, int64_t pool_sh, const int32_t* __restrict__ page_table,
    int64_t table_stride, int max_pages, int n_pages, const int32_t* __restrict__ prefix_lens, const int32_t* __restrict__ cu,
    int n_seg, int H) {
  const int t = blockIdx.x / H, h = blockIdx.x % H;
  const int b = packed_segment(cu, n_seg, t);
  const int pos = prefix_lens[b] + t - cu[b];
  const int page = page_of(page_table + b * table_stride, max_pages, n_pages, pos);
  if (page <= 0) return;  // unmapped, outside the pool, or the null page
  const bool is_v = threadIdx.x >= KV_ROW_VECS;
  const int j = threadIdx.x % KV_ROW_VECS;
  const uint4 x = reinterpret_cast<const uint4*>((is_v ? v : k) + h * src_sh + static_cast<int64_t>(t) * 128)[j];
  __nv_bfloat16* dst = (is_v ? vp : kp) + page * page_stride + h * pool_sh + static_cast<int64_t>(pos % PAGE_ROWS) * 128;
  reinterpret_cast<uint4*>(dst)[j] = x;
}

struct SlotAdvanceParams {
  const int64_t* next_ids;
  int64_t* ids_in;
  int32_t* out_tokens;  // [R, out_stride]
  int64_t out_stride;
  int32_t* n_out;
  const int32_t* max_new;
  int32_t* rope_pos;
  int32_t* write_pos;
  int32_t* kv_len;
  uint64_t* rng_offset;
  uint8_t* finished;
  int64_t eos[ADV_MAX_EOS];
  int32_t n_eos;
  int64_t pad;
  int32_t R;
};

// Slot r emits its token n_out[r] (the one sampled at offset rng_offset[r] = n_out[r]) and finishes on an EOS id or when its
// budget is spent; a finished slot keeps every value, and is fed pad, until the host retires it.
__global__ void __launch_bounds__(ADV_MAX_B) decode_advance_slots_kernel(const SlotAdvanceParams p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.R || p.finished[r]) return;
  const int64_t tok = p.next_ids[r];
  const int t = p.n_out[r];
  if (t < p.out_stride) p.out_tokens[r * p.out_stride + t] = static_cast<int32_t>(tok);
  bool fin = t + 1 >= p.max_new[r];
  for (int e = 0; e < p.n_eos; ++e) fin |= tok == p.eos[e];
  p.ids_in[r] = fin ? p.pad : tok;
  p.n_out[r] = t + 1;
  p.finished[r] = fin;
  ++p.rope_pos[r];
  ++p.write_pos[r];
  ++p.kv_len[r];
  ++p.rng_offset[r];
}

constexpr int LK_MAX_K = 15;  // drafts per row
constexpr int LK_MAX_M = 16;  // longest n-gram
constexpr int DRAFT_THREADS = 256;

__device__ __forceinline__ bool is_eos(int64_t t, const int64_t* eos, int n_eos) {
  bool r = false;
  for (int e = 0; e < n_eos; ++e) r |= t == eos[e];
  return r;
}

struct DraftParams {
  const int64_t* hist;  // [B, hist_stride]: row b's real tokens, hist_len[b] of them
  int64_t hist_stride;
  const int32_t* hist_len;
  const uint8_t* finished;
  const int32_t* n_out;
  int32_t max_new;
  int64_t* drafts;  // [B, K] at row stride draft_stride
  int64_t draft_stride;
  int32_t* draft_len;
  int32_t* any_draft;
  int32_t K, M;
  int64_t eos[ADV_MAX_EOS];
  int32_t n_eos;
};

// For every end e in [1, len) (the continuation starts at e, so it is never empty), c(e) is the number of tokens before e that
// equal the row's last tokens, up to n_max = min(M, len - 1).  The earliest match of the last n tokens is then the smallest e
// with c(e) >= n, so one pass gives the first match of every n, and the largest n with a match wins, as in get_candidates.
__global__ void __launch_bounds__(DRAFT_THREADS) ngram_draft_kernel(const DraftParams p) {
  __shared__ int64_t suf[LK_MAX_M];
  __shared__ int first_e[LK_MAX_M + 1];
  __shared__ int s_e, s_len;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t* h = p.hist + b * p.hist_stride;
  const int len = p.hist_len[b];
  const int room = p.finished[b] ? 0 : min(p.K, p.max_new - 1 - p.n_out[b]);  // tokens a step can still emit, minus one
  const int n_max = min(p.M, len - 1);
  int e_found = -1, dl = 0;
  if (room > 0 && n_max >= 1) {  // uniform over the CTA
    if (tid < n_max) suf[tid] = h[len - n_max + tid];
    if (tid <= LK_MAX_M) first_e[tid] = INT_MAX;
    __syncthreads();
    for (int e = 1 + tid; e < len; e += DRAFT_THREADS) {
      const int lim = min(n_max, e);
      int c = 0;
      while (c < lim && h[e - 1 - c] == suf[n_max - 1 - c]) ++c;
      for (int n = 1; n <= c; ++n)
        if (e < first_e[n]) atomicMin(&first_e[n], e);
    }
    __syncthreads();
    if (tid == 0) {
      int n = n_max;
      while (n >= 1 && first_e[n] == INT_MAX) --n;
      int d = 0, e = -1;
      if (n >= 1) {
        e = first_e[n];
        const int end = min(e + p.K, len);
        while (e + d < end && !is_eos(h[e + d], p.eos, p.n_eos)) ++d;  // the draft stops before its first EOS
      }
      s_e = e;
      s_len = min(d, room);
    }
    __syncthreads();
    e_found = s_e;
    dl = s_len;
  }
  if (tid < p.K) p.drafts[b * p.draft_stride + tid] = tid < dl ? h[e_found + tid] : h[max(len - 1, 0)];
  if (tid == 0) {
    p.draft_len[b] = dl;
    if (dl > 0) atomicExch(p.any_draft, 1);
  }
}

struct AcceptParams {
  const int64_t* targets;   // [B * Q] sampled at each of the step's positions
  const int64_t* step_ids;  // [B, Q] the step's input: the last token, then the drafts
  const int32_t* draft_len;
  int32_t Q;
  int64_t* ids1;            // [B] the next 1-wide step's input
  int64_t* idsk;            // [B, Kp1] the next K-wide step's input (column 0; the draft kernel writes the rest)
  int32_t Kp1;
  int32_t* pos_k;           // [B * Kp1] RoPE positions of the next K-wide step
  int32_t* lens_k;          // [B * Kp1] key counts of its queries
  uint64_t* off1;           // [B] Philox offsets of the next 1-wide step
  uint64_t* offk;           // [B * Kp1]
  int64_t* out_tokens;      // [B, max_new]
  int32_t max_new;
  int64_t* hist;
  int64_t hist_stride;
  int32_t* hist_len;
  int32_t* n_out;
  uint8_t* finished;
  int32_t* rope_pos;
  int32_t* write_pos;
  int32_t* kv_len;
  int32_t* status;                  // [0]: every row finished or at max_new; [1]: any draft (reset here, set by the draft kernel)
  unsigned long long* counters;     // [0]: draft tokens verified, [1]: draft tokens accepted
  int64_t eos[ADV_MAX_EOS];
  int32_t n_eos;
  int32_t B;
};

__global__ void __launch_bounds__(ADV_MAX_B) lookup_accept_kernel(const AcceptParams p) {
  const int b = threadIdx.x;
  bool done = true;
  if (b < p.B) {
    int n = p.n_out[b];
    bool fin = p.finished[b] != 0;
    if (!fin && n < p.max_new) {
      const int dl = p.Q > 1 ? p.draft_len[b] : 0;
      const int64_t* t = p.targets + static_cast<int64_t>(b) * p.Q;
      const int64_t* d = p.step_ids + static_cast<int64_t>(b) * p.Q + 1;
      int a = 0;
      while (a < dl && d[a] == t[a]) ++a;  // _assisted_decoding: drafts accepted while they equal the target before them
      int e = 0, hl = p.hist_len[b];
      int64_t last = 0;
      for (int i = 0; i <= a && n < p.max_new && !fin; ++i) {
        last = t[i];
        p.out_tokens[static_cast<int64_t>(b) * p.max_new + n] = last;
        if (hl < p.hist_stride) p.hist[b * p.hist_stride + hl++] = last;
        ++n;
        ++e;
        fin = is_eos(last, p.eos, p.n_eos);  // GenerationMixin: the row stops after its first EOS
      }
      p.hist_len[b] = hl;
      p.n_out[b] = n;
      p.finished[b] = fin;
      p.rope_pos[b] += e;
      p.write_pos[b] += e;
      p.kv_len[b] += e;
      p.ids1[b] = last;
      p.idsk[static_cast<int64_t>(b) * p.Kp1] = last;
      if (dl > 0) {
        atomicAdd(&p.counters[0], static_cast<unsigned long long>(dl));
        atomicAdd(&p.counters[1], static_cast<unsigned long long>(e - 1));
      }
    }
    const int rp = p.rope_pos[b], kl = p.kv_len[b];
    for (int i = 0; i < p.Kp1; ++i) {
      p.pos_k[b * p.Kp1 + i] = rp + i;
      p.lens_k[b * p.Kp1 + i] = kl + i;
      p.offk[b * p.Kp1 + i] = static_cast<uint64_t>(n + i);
    }
    p.off1[b] = static_cast<uint64_t>(n);
    done = fin || n >= p.max_new;
  }
  const bool all = __syncthreads_and(done);
  if (b == 0) {
    p.status[0] = all;
    p.status[1] = 0;
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

extern "C" int aria_kv_append_paged(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_pool,
                                    void* v_pool, int64_t page_stride, int64_t pool_stride_h, const int32_t* block_table,
                                    int64_t block_table_stride, int32_t max_pages, int32_t n_pages, const int32_t* write_pos,
                                    int32_t R, int32_t H, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_new && v_new && k_pool && v_pool && block_table && write_pos);
  ARIA_CHECK_ARG(R > 0 && H > 0 && max_pages > 0 && n_pages > 0 && block_table_stride >= max_pages);
  ARIA_CHECK_ARG(static_cast<int64_t>(R) * H < (1ll << 31) && static_cast<int64_t>(R) * block_table_stride < (1ll << 31));
  ARIA_CHECK_ARG(pool_stride_h >= PAGE_ROWS * 128 && page_stride >= pool_stride_h * H);
  ARIA_CHECK_ARG(new_stride_b % 8 == 0 && new_stride_h % 8 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  kv_append_paged_kernel<<<R * H, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k_new), static_cast<const __nv_bfloat16*>(v_new), new_stride_b, new_stride_h,
      static_cast<__nv_bfloat16*>(k_pool), static_cast<__nv_bfloat16*>(v_pool), page_stride, pool_stride_h, block_table,
      block_table_stride, max_pages, n_pages, write_pos, H);
  return check_launch("kv_append_paged_kernel");
}

extern "C" int aria_kv_pages_store(const void* k, const void* v, int64_t src_stride_h, int32_t T, void* k_pool, void* v_pool,
                                   int64_t page_stride, int64_t pool_stride_h, const int32_t* pages, int32_t max_pages,
                                   int32_t n_pages, int32_t H, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k && v && k_pool && v_pool && pages);
  ARIA_CHECK_ARG(T > 0 && H > 0 && n_pages > 0 && max_pages > 0 && T <= static_cast<int64_t>(max_pages) * PAGE_ROWS);
  ARIA_CHECK_ARG(static_cast<int64_t>(T) * H < (1ll << 31) && src_stride_h >= static_cast<int64_t>(T) * 128);
  ARIA_CHECK_ARG(pool_stride_h >= PAGE_ROWS * 128 && page_stride >= pool_stride_h * H);
  ARIA_CHECK_ARG(src_stride_h % 8 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  kv_pages_store_kernel<<<T * H, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v), src_stride_h, static_cast<__nv_bfloat16*>(k_pool),
      static_cast<__nv_bfloat16*>(v_pool), page_stride, pool_stride_h, pages, max_pages, n_pages, H);
  return check_launch("kv_pages_store_kernel");
}

extern "C" int aria_kv_pages_store_varlen(const void* k, const void* v, int64_t src_stride_h, int32_t S_tot, void* k_pool,
                                          void* v_pool, int64_t page_stride, int64_t pool_stride_h, const int32_t* page_table,
                                          int64_t page_table_stride, int32_t max_pages, int32_t n_pages, const int32_t* prefix_lens,
                                          const int32_t* cu_seqlens, int32_t n_seg, int32_t H, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k && v && k_pool && v_pool && page_table && prefix_lens && cu_seqlens);
  ARIA_CHECK_ARG(S_tot >= n_seg && n_seg > 0 && H > 0 && n_pages > 0 && max_pages > 0 && page_table_stride >= max_pages);
  ARIA_CHECK_ARG(static_cast<int64_t>(S_tot) * H < (1ll << 31) && src_stride_h >= static_cast<int64_t>(S_tot) * 128);
  ARIA_CHECK_ARG(static_cast<int64_t>(n_seg) * page_table_stride < (1ll << 31));
  ARIA_CHECK_ARG(pool_stride_h >= PAGE_ROWS * 128 && page_stride >= pool_stride_h * H);
  ARIA_CHECK_ARG(src_stride_h % 8 == 0 && page_stride % 8 == 0 && pool_stride_h % 8 == 0);
  kv_pages_store_varlen_kernel<<<S_tot * H, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v), src_stride_h, static_cast<__nv_bfloat16*>(k_pool),
      static_cast<__nv_bfloat16*>(v_pool), page_stride, pool_stride_h, page_table, page_table_stride, max_pages, n_pages,
      prefix_lens, cu_seqlens, n_seg, H);
  return check_launch("kv_pages_store_varlen_kernel");
}

extern "C" int aria_decode_advance_slots(const int64_t* next_ids, int64_t* ids_in, int32_t* out_tokens, int64_t out_stride,
                                         int32_t* n_out, const int32_t* max_new, int32_t* rope_pos, int32_t* write_pos,
                                         int32_t* kv_len, uint64_t* rng_offset, uint8_t* finished, const int64_t* eos_ids,
                                         int32_t n_eos, int64_t pad_token_id, int32_t R, aria_stream_t stream_) {
  ARIA_CHECK_ARG(next_ids && ids_in && out_tokens && n_out && max_new && rope_pos && write_pos && kv_len && rng_offset && finished);
  ARIA_CHECK_ARG(R > 0 && R <= ADV_MAX_B && out_stride > 0);
  ARIA_CHECK_ARG(n_eos >= 0 && n_eos <= ADV_MAX_EOS && (n_eos == 0 || eos_ids));
  SlotAdvanceParams p{};
  p.next_ids = next_ids;
  p.ids_in = ids_in;
  p.out_tokens = out_tokens;
  p.out_stride = out_stride;
  p.n_out = n_out;
  p.max_new = max_new;
  p.rope_pos = rope_pos;
  p.write_pos = write_pos;
  p.kv_len = kv_len;
  p.rng_offset = rng_offset;
  p.finished = finished;
  for (int e = 0; e < n_eos; ++e) p.eos[e] = eos_ids[e];  // host array, copied into the launch parameters
  p.n_eos = n_eos;
  p.pad = pad_token_id;
  p.R = R;
  decode_advance_slots_kernel<<<1, (R + 31) / 32 * 32, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("decode_advance_slots_kernel");
}

extern "C" int aria_kv_append_rows(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h,
                                   int64_t new_stride_q, void* k_cache, void* v_cache, int64_t cache_stride_b,
                                   int64_t cache_stride_h, const int32_t* pos, int32_t B, int32_t Q, int32_t H, int32_t T_max,
                                   aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_new && v_new && k_cache && v_cache && pos);
  ARIA_CHECK_ARG(B > 0 && Q > 0 && H > 0 && T_max > 0 && static_cast<int64_t>(B) * H * Q < (1ll << 31));
  ARIA_CHECK_ARG(new_stride_b % 8 == 0 && new_stride_h % 8 == 0 && new_stride_q % 8 == 0 && cache_stride_b % 8 == 0 &&
                 cache_stride_h % 8 == 0);
  kv_append_rows_kernel<<<B * H * Q, 2 * KV_ROW_VECS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k_new), static_cast<const __nv_bfloat16*>(v_new), new_stride_b, new_stride_h, new_stride_q,
      static_cast<__nv_bfloat16*>(k_cache), static_cast<__nv_bfloat16*>(v_cache), cache_stride_b, cache_stride_h, pos, H, Q, T_max);
  return check_launch("kv_append_rows_kernel");
}

extern "C" int aria_ngram_draft(const int64_t* hist, int64_t hist_stride, const int32_t* hist_len, const uint8_t* finished,
                                const int32_t* n_out, int32_t max_new, int64_t* drafts, int64_t draft_stride, int32_t* draft_len,
                                int32_t* any_draft, int32_t B, int32_t K, int32_t M, const int64_t* eos_ids, int32_t n_eos,
                                aria_stream_t stream_) {
  ARIA_CHECK_ARG(hist && hist_len && finished && n_out && drafts && draft_len && any_draft);
  ARIA_CHECK_ARG(B > 0 && B <= 65535 * 32 && K >= 1 && K <= LK_MAX_K && M >= 1 && M <= LK_MAX_M && max_new > 0);
  ARIA_CHECK_ARG(hist_stride > 0 && hist_stride < (1ll << 31) && draft_stride >= K);
  ARIA_CHECK_ARG(n_eos >= 0 && n_eos <= ADV_MAX_EOS && (n_eos == 0 || eos_ids));
  DraftParams p{};
  p.hist = hist;
  p.hist_stride = hist_stride;
  p.hist_len = hist_len;
  p.finished = finished;
  p.n_out = n_out;
  p.max_new = max_new;
  p.drafts = drafts;
  p.draft_stride = draft_stride;
  p.draft_len = draft_len;
  p.any_draft = any_draft;
  p.K = K;
  p.M = M;
  for (int e = 0; e < n_eos; ++e) p.eos[e] = eos_ids[e];  // host array, copied into the launch parameters
  p.n_eos = n_eos;
  ngram_draft_kernel<<<B, DRAFT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("ngram_draft_kernel");
}

extern "C" int aria_lookup_accept_advance(const int64_t* targets, const int64_t* step_ids, const int32_t* draft_len, int32_t Q,
                                          int64_t* ids1, int64_t* idsk, int32_t Kp1, int32_t* pos_k, int32_t* lens_k, uint64_t* off1,
                                          uint64_t* offk, int64_t* out_tokens, int32_t max_new, int64_t* hist, int64_t hist_stride,
                                          int32_t* hist_len, int32_t* n_out, uint8_t* finished, int32_t* rope_pos, int32_t* write_pos,
                                          int32_t* kv_len, int32_t* status, uint64_t* counters, const int64_t* eos_ids,
                                          int32_t n_eos, int32_t B, aria_stream_t stream_) {
  ARIA_CHECK_ARG(targets && step_ids && draft_len && ids1 && idsk && pos_k && lens_k && off1 && offk && out_tokens && hist);
  ARIA_CHECK_ARG(hist_len && n_out && finished && rope_pos && write_pos && kv_len && status && counters);
  ARIA_CHECK_ARG(B > 0 && B <= ADV_MAX_B && Kp1 >= 2 && Kp1 <= LK_MAX_K + 1 && (Q == 1 || Q == Kp1) && max_new > 0);
  ARIA_CHECK_ARG(hist_stride > 0 && hist_stride < (1ll << 31));
  ARIA_CHECK_ARG(n_eos >= 0 && n_eos <= ADV_MAX_EOS && (n_eos == 0 || eos_ids));
  AcceptParams p{};
  p.targets = targets;
  p.step_ids = step_ids;
  p.draft_len = draft_len;
  p.Q = Q;
  p.ids1 = ids1;
  p.idsk = idsk;
  p.Kp1 = Kp1;
  p.pos_k = pos_k;
  p.lens_k = lens_k;
  p.off1 = off1;
  p.offk = offk;
  p.out_tokens = out_tokens;
  p.max_new = max_new;
  p.hist = hist;
  p.hist_stride = hist_stride;
  p.hist_len = hist_len;
  p.n_out = n_out;
  p.finished = finished;
  p.rope_pos = rope_pos;
  p.write_pos = write_pos;
  p.kv_len = kv_len;
  p.status = status;
  p.counters = reinterpret_cast<unsigned long long*>(counters);
  for (int e = 0; e < n_eos; ++e) p.eos[e] = eos_ids[e];
  p.n_eos = n_eos;
  p.B = B;
  const int threads = (B + 31) / 32 * 32;
  lookup_accept_kernel<<<1, threads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("lookup_accept_kernel");
}
