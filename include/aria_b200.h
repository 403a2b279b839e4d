/* aria_b200 — C ABI of the H100-native Aria hot path (libaria_b200.so).
 *
 * Every entry point is `extern "C"`, takes raw DEVICE pointers + sizes + a cudaStream_t, never allocates or
 * frees, launches asynchronously on the caller's stream and returns 0 or a negative error code.  There is
 * no CPU fallback: unsupported shapes are errors.  Pointers must be 16-byte aligned and rows contiguous.
 *
 * Each function names the reference interface (rhymes-ai/Aria @ 9b25fecb) it replaces.  The reference is
 * pure Python; its "FFI" for this path is the set of third-party kernels it imports (SURVEY.md §2b):
 *   grouped_gemm.ops.gmm (aria/model/moe_lm.py:432,484), flash-attn / SDPA behind the HF attention classes
 *   (moe_lm.py:594, vision_encoder.py:120), and the ATen ops of the router / dispatcher (moe_lm.py:261-269,
 *   329-332, 350-363).  INTEGRATION.md shows the ctypes binding a maintainer adds on the reference side.
 */
#ifndef ARIA_B200_H
#define ARIA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* aria_stream_t; /* == cudaStream_t */

#define ARIA_OK 0
#define ARIA_ERR_BAD_ARG (-1)
#define ARIA_ERR_UNSUPPORTED (-2)
#define ARIA_ERR_CUDA (-3)

/* Library/ABI version and build target ("sm_90a"). */
int aria_abi_version(void);
const char* aria_build_arch(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM family (wgmma + TMA, bf16 in, fp32 accumulate, bf16 out).
 * One descriptor drives: nn.Linear-layout dense GEMMs, the reference's grouped expert GEMM, and the fused
 * epilogues of the hot path.  Rounding points mirror the reference's op-by-op bf16 rounding.
 * ------------------------------------------------------------------------------------------------ */
enum { ARIA_B_NK = 0,  /* B[n_seg][N,K], K contiguous — torch.nn.Linear.weight                        */
       ARIA_B_GKN = 1, /* B[G,K,N],      N contiguous — GroupedGEMM.weight (moe_lm.py:465)            */
       ARIA_B_GNK = 2  /* B[G,N,K],      K contiguous — the same expert weight used transposed (dgrad) */ };
enum { ARIA_EPI_LINEAR = 0, /* out = act(acc + bias) (+ residual)                                      */
       ARIA_EPI_SWIGLU = 1, /* out = silu(acc_gate) * acc_up  (moe_lm.py:505-507 `glu`, LlamaMLP)      */
       ARIA_EPI_HEADS = 2   /* (+bias) (+RoPE) and scatter to [B, H, T, head_ld] head-major buffers    */ };
enum { ARIA_ACT_NONE = 0, ARIA_ACT_GELU_TANH = 1, /* F.gelu(approximate="tanh") — Idefics2 MLP       */
       ARIA_ACT_GELU_NEW = 2                       /* transformers NewGELU, op-by-op bf16 — projector  */ };

typedef struct aria_gemm_desc {
  /* A: activations [m, k] bf16, row stride lda (elements). For grouped GEMMs rows are grouped by expert. */
  const void* a;
  int64_t lda;
  int64_t m, n, k;   /* n = OUTPUT columns per segment (SWIGLU: B carries 2n columns: gate then up)       */
  /* B: weights. NK layout: up to 3 segments (e.g. q,k,v projections, or gate,up for SWIGLU), each [n,k]
   * (SWIGLU: b[0] = gate [n,k], b[1] = up [n,k]).  GKN layout: b[0] = [G, k, n] (SWIGLU: [G, k, 2n]).  */
  const void* b[3];
  int32_t n_seg;
  int32_t b_layout;
  /* grouping: num_groups = 1 and group_offsets = NULL for a dense GEMM; else group_offsets[G+1] (device,
   * int32) are the row offsets of each expert's contiguous row block inside A / out.                   */
  int32_t num_groups;
  const int32_t* group_offsets;
  int32_t group_mod;       /* grouped weights: group g uses weight block g % group_mod (> 0), g / -group_mod (< 0), g (0).
                            * Expert parallelism receives rows grouped by (source rank, local expert): num_groups = W*E_loc,
                            * mod = E_loc; or by (local expert, source rank): mod = -W, which keeps the W groups that share
                            * an expert's weights next to each other in the tile order (one HBM read, W-1 L2 hits) */
  /* epilogue */
  int32_t epilogue;
  int32_t act;
  const void* bias[3];     /* per segment [n] bf16 or NULL                                               */
  const void* residual;    /* [m, n] bf16 or NULL (LINEAR only), row stride ldr                          */
  int64_t ldr;
  void* out[3];            /* LINEAR/SWIGLU: out[0] = [m, n_seg*n] row stride ldo; HEADS: one per segment */
  int64_t ldo;
  /* HEADS epilogue: row r of A is (batch r / rows_per_batch, token r % rows_per_batch); column c of
   * segment s is (head c / head_dim, d c % head_dim); destination element
   *   out[s] + batch*stride_b + head*stride_h + (pos0 + token)*head_ld + d                              */
  int32_t head_dim, head_ld, rows_per_batch, pos0;
  int64_t stride_b, stride_h;
  int32_t rope_mask;       /* bit s set: apply rotate-half RoPE to segment s (needs head_dim == 128)     */
  const void* rope_cos;    /* [max_pos, head_dim] bf16 tables (aria_rope_table)                          */
  const void* rope_sin;
  const int32_t* position_ids; /* [m] or NULL (then position = pos0 + token)                              */
  /* Expert parallelism over NVLink peer memory (fused compute + collective, SURVEY.md §8e):
   *   group_counts  non-NULL: group g = rows [group_offsets[g], group_offsets[g] + group_counts[g]) — fixed-capacity
   *                 regions a peer GPU fills without knowing the other senders' counts; a_rows = rows of the A buffer
   *                 (m then only feeds the tile-shape heuristics: pass the expected row count).
   *   out_group_base / out_group_row0 (LINEAR): row r of group g is stored at
   *                 (bf16*)out_group_base[g] + (out_group_row0[g] + r) * ldo — e.g. the SOURCE rank's combine buffer, so the
   *                 fc2 epilogue IS the return all-to-all (16-byte stores through NVSwitch). */
  const int32_t* group_counts;
  int64_t a_rows;
  const void* out_group_base;      /* uint64 device addresses [G] */
  const int32_t* out_group_row0;   /* [G] */
} aria_gemm_desc_t;

/* Generic entry.  Replaces: torch F.linear / cuBLAS on the path, and grouped_gemm.ops.gmm. */
int aria_gemm(const aria_gemm_desc_t* desc, aria_stream_t stream);

/* Drop-in for `grouped_gemm.ops.gmm(a, b, batch_sizes)` as called at moe_lm.py:484 (`experts_gemm`), except
 * that the per-expert row offsets stay on the device (no .cpu() sync, moe_lm.py:478):
 *   out[off[e]:off[e+1]] = a[off[e]:off[e+1]] @ b[e],  a [rows,k], b [G,k,n], out [rows,n], all bf16.      */
int aria_grouped_gemm(const void* a, const void* b, void* out, const int32_t* group_offsets, int64_t rows,
                      int64_t k, int64_t n, int32_t num_groups, aria_stream_t stream);

/* FP8 expert weights (weight-only, e4m3 with one fp32 scale per (expert, output column); activations stay bf16).
 *
 * aria_quantize_fp8_cols: w [G, K, N] bf16 (GroupedGEMM.weight layout) ->
 *   scale [G, N] fp32 = max_k |w[g,k,n]| / 448 (IEEE division; an all-zero column gets 1),
 *   q [G, K, N] e4m3 = w / scale, round to nearest even, saturating — bit for bit (w.float() / scale).to(float8_e4m3fn).
 *   K % 64 == 0, N % 64 == 0; w, q, scale 16-byte aligned.
 *
 * aria_grouped_gemm_fp8: aria_grouped_gemm with e4m3 weights b_fp8 [G, k, N_b] and scales b_scale [G, N_b]:
 *   epilogue ARIA_EPI_LINEAR (N_b = n) or ARIA_EPI_SWIGLU (N_b = 2n, gate then up, out [rows, n]).  The result is aria_gemm's
 *   with ARIA_B_GKN weights q.to(bf16), except that the fp32 accumulator of column c of group g is multiplied by
 *   b_scale[g, c] before the epilogue's first bf16 rounding; every rounding point is the same.  k % 64 == 0, n % 64 == 0. */
int aria_quantize_fp8_cols(const void* w, void* q, float* scale, int32_t G, int64_t K, int64_t N, aria_stream_t stream);
int aria_grouped_gemm_fp8(const void* a, const void* b_fp8, const float* b_scale, void* out, const int32_t* group_offsets,
                          int64_t rows, int64_t k, int64_t n, int32_t num_groups, int32_t epilogue, aria_stream_t stream);

/* FP8 activations and weights (W8A8) for the routed experts.
 *
 * aria_permute_quantize_fp8_rows: x [*, d] bf16 -> q [rows, d] e4m3, scale [rows] fp32, row r taken from x[src_token[r]]
 *   (x[r] when src_token is NULL; src_token[r] < 0 gives a zero row):
 *   scale[r] = max |x_row| / 448 (IEEE division; an all-zero row gets 1), q = e4m3(x_row / scale[r]), round to nearest even,
 *   saturating — bit for bit (x.float() / scale[:, None]).to(float8_e4m3fn).  d % 8 == 0, d <= 4096; x, q 16-byte aligned.
 *
 * aria_grouped_gemm_w8a8: out[off[g]:off[g+1]] = epilogue(a[rows of g] . b[g]^T * a_scale[row] * b_scale[g, col]), with
 *   a_fp8 [rows, k] e4m3 and a_scale [rows] from aria_permute_quantize_fp8_rows, b_fp8_nk [G, N_b, k] e4m3 (K-major: the
 *   transpose of the [G, k, N_b] weights of aria_quantize_fp8_cols, same codes) and b_scale [G, N_b].  Epilogue ARIA_EPI_LINEAR
 *   (N_b = n) or ARIA_EPI_SWIGLU (N_b = 2n, gate then up, out [rows, n]).  Both scales multiply the fp32 accumulator before the
 *   epilogue's first bf16 rounding; every rounding point after that is aria_gemm's.  The tensor cores accumulate one
 *   128-element k-block at a time, which is then added to an fp32 accumulator.  k % 128 == 0, n % 64 == 0. */
int aria_permute_quantize_fp8_rows(const void* x, const int32_t* src_token, void* q, float* scale, int64_t rows, int32_t d,
                                   aria_stream_t stream);
int aria_grouped_gemm_w8a8(const void* a_fp8, const float* a_scale, const void* b_fp8_nk, const float* b_scale, void* out,
                           const int32_t* group_offsets, int64_t rows, int64_t k, int64_t n, int32_t num_groups, int32_t epilogue,
                           aria_stream_t stream);

/* W8A8 dense GEMM for nn.Linear weights: aria_gemm's descriptor (b_layout ARIA_B_NK, num_groups 1, no group offsets or
 * counts) with a = e4m3 [m, k] (row stride lda, in elements = bytes) and b[s] = e4m3 [n, k] weights, one per segment.
 * a_scale [m] fp32 is the row scale of a (aria_permute_quantize_fp8_rows or aria_rmsnorm_quantize_fp8); b_scale[s] [n] fp32
 * the column scales of b[s] (aria_permute_quantize_fp8_rows on the [n, k] weight: one scale per output channel).  The fp32
 * accumulator of (row r, column c of segment s) is multiplied by a_scale[r] * b_scale[s][c] before the epilogue's first bf16
 * rounding; every rounding point after that is aria_gemm's.  Epilogues: ARIA_EPI_LINEAR (bias, act, residual), ARIA_EPI_SWIGLU
 * (n_seg = 2: b[0] = gate, b[1] = up) and ARIA_EPI_HEADS (RoPE at pos0 or position_ids).  k % 128 == 0, n % 64 == 0
 * (n % 128 == 0 for HEADS and for LINEAR with n_seg > 1); a, out, b[s] and residual 16-byte aligned, b_scale[s] 16-byte
 * aligned, lda % 16 == 0.  Every argument is checked before any CUDA call. */
int aria_gemm_w8a8(const aria_gemm_desc_t* desc, const float* a_scale, const float* const b_scale[3], aria_stream_t stream);

/* Weight gradient of a (grouped) linear layer — backward of gmm / F.linear:
 *   out[g, m, n] = sum_{r in group g} a[r, m] * b[r, n]   a [rows, md] (row stride lda), b [rows, nd] (ldb), out [G, md, nd] bf16.
 * group_offsets: device int32 row offsets, non-decreasing, any values (densely packed groups as the reference's dispatcher
 * produces them, or the 16-aligned blocks of aria_build_permutation with row_align = 16).  Rows past the last offset are
 * never multiplied into a result.  When a group's row count is not a multiple of 16, the (up to 15) rows of b that follow
 * it are multiplied by zeros, so they must be finite (rows past `rows` are read as zeros).
 * num_sources = 1: offsets[G+1].  num_sources = S > 1 (expert parallelism): rows are grouped (source rank, g),
 * source-major, offsets[S*G+1], and out[g] sums the S partial products — no separate reduction pass. */
int aria_grouped_wgrad(const void* a, int64_t lda, const void* b, int64_t ldb, void* out, const int32_t* group_offsets,
                       int64_t rows, int64_t md, int64_t nd, int32_t num_groups, int32_t num_sources, aria_stream_t stream);
/* One-group weight gradient accumulated in fp32: out[m, n] += sum_{r < rows} a[r, m] * b[r, n]; out [md, nd] fp32, 8-byte
 * aligned.  The same kernel as aria_grouped_wgrad with an epilogue that adds its fp32 accumulators to out, so a weight gradient
 * can be built up over chunks of rows without a bf16 rounding per chunk.  Each output tile has one owner: no atomics, and
 * the result does not depend on the launch.  rows = 0 launches nothing. */
int aria_wgrad_accumulate_f32(const void* a, int64_t lda, const void* b, int64_t ldb, float* out, int64_t rows, int64_t md,
                              int64_t nd, aria_stream_t stream);

/* Cross-entropy rows for the fused lm_head loss: for each of `rows` rows of bf16 logits (row stride ld, vocab % 8 == 0,
 * ld % 8 == 0, logits 16-byte aligned) and its int64 label in [0, vocab):
 *   loss[r] = logsumexp(logits[r, :]) - logits[r, label[r]]                 (fp32, softmax in fp32)
 *   logits[r, :] <- (softmax(logits[r, :]) - onehot(label[r])) * (*grad_scale)  (bf16, in place)
 * grad_scale: DEVICE fp32 scalar (1 / n for a mean, 1 for a sum).  A label outside [0, vocab) gives loss NaN and no one-hot
 * term (callers check labels first).  One CTA per row; two runs give identical bits. */
int aria_cross_entropy_rows(void* logits, int64_t ld, const int64_t* labels, const float* grad_scale, float* loss, int64_t rows,
                            int32_t vocab, aria_stream_t stream);

/* int64 counts (tokens_per_expert as the reference passes it, moe_lm.py:264-269) -> int32 offsets[G+1]. */
int aria_offsets_from_counts(const int64_t* counts, int32_t* offsets, int32_t num_groups, aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * MoE routing / dispatch (HBM-bound kernels)
 * ------------------------------------------------------------------------------------------------ */
/* TopKRouter.forward (moe_lm.py:275-293 = gating :190-201 + routing :261-269), eval path.
 *   x [T, d] bf16, w_router [E, d] bf16 -> logits [T, E] bf16 (required: the top-k runs on the rounded values),
 *   top_idx [T, k] int32 (descending logit, ties: lowest expert id), scores [T, k] bf16 (fp32 softmax over
 *   the k selected bf16 logits, rounded to bf16), counts [E] int32 (must be zeroed by this call: it is).
 * E <= 64, k <= 8. */
int aria_router_topk(const void* x, const void* w_router, void* logits_out, int32_t* top_idx, void* scores,
                     int32_t* counts, int64_t T, int32_t d, int32_t E, int32_t k, aria_stream_t stream);
/* Same routing from precomputed bf16 logits (exact integer/bit parity path; torch.topk + softmax + histc). */
int aria_route_from_logits(const void* logits, int32_t* top_idx, void* scores, int32_t* counts, int64_t T,
                           int32_t E, int32_t k, aria_stream_t stream);

/* Routing with the expert choice GIVEN (parity / replay hook): top_idx [T, k] int32 is an INPUT; scores = fp32 softmax over the
 * logits at those ids (same arithmetic as above), counts = their histogram.  Lets a test inject the oracle's top-k into the
 * CUDA path so that bf16 near-ties in the router cannot hide other differences. */
int aria_route_given_indices(const void* logits, const int32_t* top_idx, void* scores, int32_t* counts, int64_t T,
                             int32_t E, int32_t k, aria_stream_t stream);

/* TokenDispatcher.token_permutation (moe_lm.py:313-334): stable counting sort of the T*k expert ids.
 *   offsets [E+1] int32 (exclusive scan of counts), dest_row [T*k] int32 (row of flattened (token,slot) in
 *   the expert-sorted order == inverse of the reference's `sorted_indices`), src_token [T*k] int32 (token of
 *   each sorted row == sorted_indices // k).  Order inside an expert = ascending flattened index (stable). */
/* row_align = 1: dense layout (inference).  row_align = 16 (training): every expert's block starts on a multiple of 16
 * rows; src_token then needs T*k + E*(row_align-1) slots and pad rows carry -1 (permute_rows writes zeros for them). */
int aria_build_permutation(const int32_t* top_idx, const int32_t* counts, int32_t* offsets, int32_t* dest_row,
                           int32_t* src_token, int64_t T, int32_t E, int32_t k, int32_t row_align, aria_stream_t stream);
/*   permuted[r, :] = x[src_token[r], :]  (index_select, moe_lm.py:330) */
int aria_permute_rows(const void* x, const int32_t* src_token, void* permuted, int64_t rows, int32_t d,
                      aria_stream_t stream);
/* TokenDispatcher.token_unpermutation (moe_lm.py:336-365) fused with `output += shared` (moe_lm.py:576):
 *   out[t] = bf16( sum_j bf16(y[dest_row[t*k+j]] * scores[t,j]) ) (+ shared[t]) ; fp32 accumulate. */
int aria_unpermute_combine(const void* y, const int32_t* dest_row, const void* scores, const void* shared,
                           void* out, int64_t T, int32_t d, int32_t k, aria_stream_t stream);

/* MoELayer.forward as ONE call (moe_lm.py:548-577; SURVEY.md §8b "moe_block_fwd"): router -> stable sort by expert ->
 * grouped fc1 + glu -> grouped fc2 -> unpermute + score-weighted sum + shared experts.  Launches the kernels of the entries
 * above in order from C (no Python between them), the shared-expert branch on `side_stream` when one is given (forked from /
 * joined to `stream` with events: becomes a parallel branch under CUDA-graph capture), counts and offsets never leave the
 * device (the reference's tokens_per_expert.cpu(), moe_lm.py:478, is gone).
 *   x [T, d]; w_router [E, d]; fc1_w [E, d, 2I] / fc2_w [E, I, d] (GroupedGEMM.weight layout); gate_w / up_w [I_shared, d],
 *   down_w [d, I_shared] (nn.Linear layout; I_shared = 0: no shared experts); out [T, d]; all bf16.
 *   forced_top_idx [T, k] int32 or NULL: expert choice given (parity / replay hook, see aria_route_given_indices).
 *   workspace: aria_moe_block_fwd_workspace_bytes(...) bytes, 16-byte aligned; holds every intermediate. */
int64_t aria_moe_block_fwd_workspace_bytes(int64_t T, int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared);
int aria_moe_block_fwd(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w, const void* gate_w,
                       const void* up_w, const void* down_w, void* out, int64_t T, int32_t d, int32_t E, int32_t k, int32_t I,
                       int32_t I_shared, const int32_t* forced_top_idx, void* workspace, int64_t workspace_bytes,
                       aria_stream_t stream, aria_stream_t side_stream);
/* The same block with e4m3 expert weights: fc1_w [E, d, 2I] / fc2_w [E, I, d] from aria_quantize_fp8_cols, with their scales
 * fc1_scale [E, 2I] / fc2_scale [E, d]; the expert GEMMs are aria_grouped_gemm_fp8.  d % 64 == 0, I % 64 == 0.  Same workspace. */
int aria_moe_block_fwd_fp8(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w, const float* fc1_scale,
                           const float* fc2_scale, const void* gate_w, const void* up_w, const void* down_w, void* out, int64_t T,
                           int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared, const int32_t* forced_top_idx,
                           void* workspace, int64_t workspace_bytes, aria_stream_t stream, aria_stream_t side_stream);
/* The same block with W8A8 experts: fc1_w_nk [E, 2I, d] / fc2_w_nk [E, d, I] are the K-major e4m3 weights (the transposes of
 * aria_quantize_fp8_cols' codes) with the scales fc1_scale [E, 2I] / fc2_scale [E, d].  The gathered tokens and h are
 * quantised per row (aria_permute_quantize_fp8_rows) and the expert GEMMs are aria_grouped_gemm_w8a8.
 * d % 128 == 0, I % 128 == 0, d and I <= 4096, I <= 2 d.  Same workspace. */
int aria_moe_block_fwd_w8a8(const void* x, const void* w_router, const void* fc1_w_nk, const void* fc2_w_nk, const float* fc1_scale,
                            const float* fc2_scale, const void* gate_w, const void* up_w, const void* down_w, void* out, int64_t T,
                            int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared, const int32_t* forced_top_idx,
                            void* workspace, int64_t workspace_bytes, aria_stream_t stream, aria_stream_t side_stream);
/* The same block with W8A8 shared experts, in any expert mode: expert_mode ARIA_MOE_EXPERTS_BF16 (fc1_scale / fc2_scale NULL,
 * as aria_moe_block_fwd), _FP8 (as aria_moe_block_fwd_fp8) or _W8A8 (as aria_moe_block_fwd_w8a8).  gate_w / up_w [I_shared, d]
 * and down_w [d, I_shared] are e4m3 nn.Linear weights with one fp32 scale per output channel, gate_scale / up_scale
 * [I_shared], down_scale [d].  The shared branch quantises x per row, runs aria_gemm_w8a8 (SwiGLU), quantises h per row and
 * runs aria_gemm_w8a8 (LINEAR).  I_shared > 0, d and I_shared % 128 == 0 and <= 4096, plus the expert mode's constraints.
 * workspace: aria_moe_block_fwd_shared_fp8_workspace_bytes(...) bytes, 16-byte aligned. */
enum { ARIA_MOE_EXPERTS_BF16 = 0, ARIA_MOE_EXPERTS_FP8 = 1, ARIA_MOE_EXPERTS_W8A8 = 2 };
int64_t aria_moe_block_fwd_shared_fp8_workspace_bytes(int64_t T, int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared);
int aria_moe_block_fwd_shared_fp8(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w, const float* fc1_scale,
                                  const float* fc2_scale, int32_t expert_mode, const void* gate_w, const void* up_w,
                                  const void* down_w, const float* gate_scale, const float* up_scale, const float* down_scale,
                                  void* out, int64_t T, int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared,
                                  const int32_t* forced_top_idx, void* workspace, int64_t workspace_bytes, aria_stream_t stream,
                                  aria_stream_t side_stream);

/* ---- backward of the MoE block (BASELINE cfg 5; autograd through moe_lm.py:548-577) ---- */
/* h = bf16(bf16(silu(g)) * u) with g = h1[:, :I], u = h1[:, I:]  (unfused `glu`, moe_lm.py:505-507; training keeps h1). */
int aria_swiglu_fwd(const void* h1, void* h, int64_t rows, int32_t I, aria_stream_t stream);
/* dh1 = [dh * u * silu'(g) | dh * silu(g)] */
int aria_swiglu_bwd(const void* h1, const void* dh, void* dh1, int64_t rows, int32_t I, aria_stream_t stream);
/* backward of aria_unpermute_combine w.r.t. y and scores:
 *   dy[dest_row[t*k+j]] = bf16(scores[t,j] * dout[t]),  dscores[t,j] = <dout[t], y[dest_row[t*k+j]]> (fp32).
 * dy rows that no (t,j) maps to (alignment pads) must be pre-zeroed by the caller. */
int aria_combine_bwd(const void* dout, const void* y, const int32_t* dest_row, const void* scores, void* dy, float* dscores,
                     int64_t T, int32_t d, int32_t k, aria_stream_t stream);
/* backward of softmax-over-top-k (moe_lm.py:261-262): dlogits[t, idx[t,j]] = s_j * (g_j - sum_i s_i g_i), zeros elsewhere. */
int aria_router_bwd(const float* dscores, const void* scores, const int32_t* top_idx, void* dlogits, int64_t T, int32_t E,
                    int32_t k, aria_stream_t stream);
/* Training-mode router losses (TopKRouter.apply_z_loss / apply_aux_loss, moe_lm.py:203-241; z_loss_func :128-140,
 * switch_load_balancing_loss_func :143-166).  logits [T,E] bf16, counts [E] int32 (tokens_per_expert), E <= 256.
 *   losses[0] = z_coeff * mean_t(logsumexp(logits_t)^2)
 *   losses[1] = aux_coeff * E/(T*k) * sum_e mean_t(softmax(logits)_te) * counts[e]          (fp32 softmax, :235)
 * The reference uses the values only through MoEAuxLossAutoScaler (:84-125): aria_router_aux_bwd ADDS
 * loss_scale * d(losses[0] + losses[1])/d(logits) to dlogits (bf16 [T,E], e.g. the output of aria_router_bwd);
 * loss_scale is MoEAuxLossAutoScaler.main_loss_backward_scale. */
size_t aria_router_aux_workspace_bytes(int32_t E);
int aria_router_aux_loss(const void* logits, const int32_t* counts, float* losses, int64_t T, int32_t E, int32_t k, float z_coeff,
                         float aux_coeff, void* workspace, size_t ws_bytes, aria_stream_t stream);
int aria_router_aux_bwd(const void* logits, const int32_t* counts, void* dlogits, int64_t T, int32_t E, int32_t k, float z_coeff,
                        float aux_coeff, float loss_scale, aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Norms, RoPE table, embedding, patches
 * ------------------------------------------------------------------------------------------------ */
/* LlamaRMSNorm (moe_lm.py:599-602,631): out = w * bf16(x * rsqrt(mean(x^2) + eps)).
 * If residual != NULL: first h = bf16(x + residual), written to sum_out, and the norm is taken of h. */
int aria_rmsnorm(const void* x, const void* residual, const void* weight, void* out, void* sum_out, int64_t rows,
                 int32_t d, float eps, aria_stream_t stream);
/* aria_rmsnorm whose bf16 output row is quantised per row in the same kernel instead of being stored:
 *   q [rows, d] e4m3, scale [rows] fp32 — bit for bit aria_rmsnorm followed by aria_permute_quantize_fp8_rows (src_token NULL).
 * residual / sum_out as in aria_rmsnorm.  d % 8 == 0, d <= 4096; x, residual, weight, q, sum_out 16-byte aligned. */
int aria_rmsnorm_quantize_fp8(const void* x, const void* residual, const void* weight, void* q, float* scale, void* sum_out,
                              int64_t rows, int32_t d, float eps, aria_stream_t stream);
/* nn.LayerNorm (Idefics2 encoder layers, projector): out = bf16((x-mean)*rstd*w + b). */
int aria_layernorm(const void* x, const void* weight, const void* bias, void* out, int64_t rows, int32_t d,
                   float eps, aria_stream_t stream);
/* LlamaRotaryEmbedding (moe_lm.py:632): cos/sin [n_pos, head_dim] bf16 from fp32 inv_freq[head_dim/2]. */
int aria_rope_table(const float* inv_freq, void* cos_out, void* sin_out, int32_t n_pos, int32_t head_dim,
                    aria_stream_t stream);
/* nn.Embedding gather: out[i] = table[ids[i]]. */
int aria_embedding(const int64_t* ids, const void* table, void* out, int64_t n, int32_t d, aria_stream_t stream);
/* masked_scatter merge (modeling_aria.py:272-283): rows where ids == image_token get consecutive rows of
 * `features`; `slot_index` [n] int32 scratch.  Returns the number of image slots through *count_out (device). */
int aria_merge_image_features(const int64_t* ids, int64_t image_token, const void* features, void* embeds,
                              int32_t* count_out, int64_t n, int32_t d, aria_stream_t stream);
/* Conv2d(3,C,14,14) as im2col: pixel_values [B,3,S,S] bf16 -> patches [B*N, k_pad] (k = 3*P*P zero padded). */
int aria_im2col_patches(const void* pixels, void* patches, int32_t B, int32_t S, int32_t P, int32_t k_pad,
                        aria_stream_t stream);
/* out[r,:] = bf16(x[r,:] + table[pos[r],:]) — position-embedding add of Idefics2VisionEmbeddings. */
int aria_add_pos_embedding(const void* x, const int64_t* pos_ids, const void* table, void* out, int64_t rows,
                           int32_t d, aria_stream_t stream);

/* Multi-GPU: allow kernels on the current device to load/store `peer_device`'s memory over NVLink (idempotent). */
int aria_enable_peer_access(int32_t peer_device);
/* CUDA IPC for peer-mapped arenas: export the 64-byte handle of the allocation containing `ptr` (+ byte offset of ptr in
 * it); open maps a peer's allocation into the current device's context (lazy peer access) and returns its base. */
int aria_ipc_export(const void* ptr, void* handle64, int64_t* offset_out);
int aria_ipc_open(const void* handle64, void** base_out);
int aria_ipc_close(void* base);

/* Expert-parallel exchange over NVLink peer memory (aria_b200/csrc/ep.cu): replaces the all-to-all the reference's
 * dispatcher lost (moe_lm.py:296-297).  `peer_*` arrays are device arrays of W addresses (one per rank, as mapped on THIS
 * GPU).  All calls are asynchronous and need no host sync. */
int aria_peer_barrier(const uint64_t* peer_flags, int32_t rank, int32_t W, int32_t* epoch_dev /* device counter, advanced by the call */,
                      aria_stream_t stream);
/* Fused exchange (fixed-capacity regions; see csrc/ep.cu): gathers the token rows in expert order (src_token / offsets from
 * aria_build_permutation) and stores each into region (e % E_loc, rank) = index (e % E_loc) * W + rank of owner e / E_loc — peer_recv[p] = rank p's receive
 * buffer [W*E_loc][cap][d] as mapped on this GPU — and publishes per-block (row count, first sorted row) into the owners'
 * meta arrays peer_counts[p] / peer_row0[p] ([W*E_loc] int32 each).  A peer barrier must follow before the owner reads. */
int aria_ep_dispatch(const void* x, const int32_t* src_token, const int32_t* offsets, const uint64_t* peer_recv,
                     const uint64_t* peer_counts, const uint64_t* peer_row0, int32_t rank, int32_t W, int32_t E,
                     int32_t cap, int32_t d, int64_t max_rows, aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Attention (wgmma QK^T / PV, fp32 online softmax)
 * ------------------------------------------------------------------------------------------------ */
/* softmax(q k^T * scale + mask) v for head_dim 128 (LM) — replaces flash_attn_func / SDPA behind
 * LLAMA_ATTENTION_CLASSES (moe_lm.py:594) and, with hd padded 72->128, the Idefics2 / projector attention.
 *   q [B, H, Tq, 128], k/v [B, H, Tk_max, 128] head-major bf16 (HF cache layout), first Tk rows valid.
 *   out [B, Tq, H*out_hd] token-major bf16 (only the first out_hd of 128 dims are written).
 *   causal != 0: query i (absolute position Tk - Tq + i) sees keys <= its position.
 *   key_mask [B, Tk] uint8 or NULL: 1 = key is masked OUT (image_attn_mask convention, vision_encoder.py:147). */
int aria_attention_fwd(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask,
                       int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h,
                       int64_t kv_stride_b, int64_t kv_stride_h, int32_t out_hd, float scale, int32_t causal,
                       void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* Scratch bytes aria_attention_fwd wants in `workspace` (0 for this build: one CTA per (batch, head, 128 queries), no partial
 * results to merge).  workspace may be NULL. */
int64_t aria_attention_fwd_workspace_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk, int32_t out_hd, int32_t causal);
/* aria_attention_fwd that also writes lse [B, H, Tq] fp32: the natural-log logsumexp of scale * q.k over the keys the row sees,
 * -inf for a row that sees none (e.g. a left-padded query row).  `out` is bit-identical to aria_attention_fwd's (same kernel). */
int aria_attention_fwd_lse(const void* q, const void* k, const void* v, void* out, float* lse, const uint8_t* key_mask,
                           int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h,
                           int64_t kv_stride_b, int64_t kv_stride_h, int32_t out_hd, float scale, int32_t causal,
                           void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* Backward of aria_attention_fwd for head_dim 128, with the forward's (Tq <= Tk, causal, key_mask) conventions:
 *   q, dq [B, H, Tq, 128] at the q strides; k, v, dk, dv [B, H, Tk, 128] at the kv strides (head-major, 128-element rows);
 *   out, dout [B, Tq, H*128] token-major (the forward's output layout); lse from aria_attention_fwd_lse.
 *   dq = scale * dS k, dk = scale * dS^T q, dv = P^T dout with P = exp(scale * q k^T - lse), dS = P o (dout v^T - rowsum(dout o out)).
 * A query row with lse = -inf contributes nothing; a key that is masked out or that no query sees gets dk = dv = 0.
 * dk and dv are bit-reproducible; dq is summed over key tiles with fp32 atomics, so its last bits depend on their order.
 * workspace: aria_attention_bwd_workspace_bytes(...) bytes, 16-byte aligned.  Three kernel launches. */
int64_t aria_attention_bwd_workspace_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk, int32_t causal);
int aria_attention_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
                       void* dq, void* dk, void* dv, const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tq, int32_t Tk,
                       int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, float scale,
                       int32_t causal, void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* Varlen (packed, padding-free) causal attention over n_seg segments packed along one sequence of N rows: segment s is rows
 * [cu_seqlens[s], cu_seqlens[s+1]) (DEVICE int32 [n_seg+1], nondecreasing from 0 to N, every segment >= 1 row); the query at
 * packed row r of segment s sees the packed keys [cu_seqlens[s], r].  q, k, v [1, H, >= N, 128] head-major (head strides
 * q_stride_h / kv_stride_h, multiples of 8 elements, 128-element rows).  out [N, H*128] bf16; lse [H, N] fp32 natural-log
 * logsumexp, or NULL.  The shared-prefix prefill's pipeline with no prefix: each segment's out and lse are bit-identical to
 * aria_attention_fwd_lse (causal) on that segment alone.  No workspace. */
int aria_attention_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int32_t* cu_seqlens,
                              int32_t n_seg, int32_t H, int32_t N, int64_t q_stride_h, int64_t kv_stride_h, float scale,
                              aria_stream_t stream);
/* Backward of aria_attention_fwd_varlen (same segment convention; lse from it): q, dq at the q head stride, k, v, dk, dv at the
 * kv head stride, out / dout [N, H*128].  One CTA per (head, 128-key tile aligned at its segment's start), heaviest tiles
 * first.  Per segment, dk and dv are bit-identical to aria_attention_bwd (causal) on the segment alone and dq equals it up to
 * the order of fp32 atomic additions; no segment's gradients read another segment's inputs.  Boundaries that break the
 * convention give wrong gradients but no access outside the tensors and the workspace (they are clamped to [0, N]).
 * workspace: aria_attention_bwd_varlen_workspace_bytes(...) bytes, 16-byte aligned.  Four kernel launches. */
int64_t aria_attention_bwd_varlen_workspace_bytes(int32_t n_seg, int32_t H, int32_t N);
int aria_attention_bwd_varlen(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
                              void* dq, void* dk, void* dv, const int32_t* cu_seqlens, int32_t n_seg, int32_t H, int32_t N,
                              int64_t q_stride_h, int64_t kv_stride_h, float scale, void* workspace, int64_t workspace_bytes,
                              aria_stream_t stream);
/* Single-token decode against a KV cache (HBM-bound, split-KV): q element (b,h,:) at q + b*q_stride_b + h*q_stride_h
 * (128 contiguous bf16), cache [B,H,Tk_max,128], out [B, H*128].  workspace: B*H*splits*(128+2) floats.
 * key_mask [B, Tk] uint8 or NULL: 1 = key is masked OUT (padded batch: the HF 2-D attention_mask inverted). */
int aria_attention_decode(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tk,
                          int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, float scale,
                          void* workspace, int64_t workspace_bytes, aria_stream_t stream);
int64_t aria_attention_decode_workspace_bytes(int32_t B, int32_t H, int32_t Tk);
/* aria_attention_decode with the key count of each row in DEVICE memory (one captured decode step replayed token after token):
 * row b attends to cache rows [0, min(lens[b], T_max)), lens = int32 [B].  key_mask [B, T_max] uint8 at row stride
 * key_mask_stride (>= T_max) or NULL.  The grid covers T_max; the result of row b is bit-identical to aria_attention_decode's
 * with Tk = lens[b].  Rows at or past lens[b] are never read.  workspace: aria_attention_decode_workspace_bytes(B, H, T_max). */
int aria_attention_decode_devlen(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask,
                                 int64_t key_mask_stride, const int32_t* lens, int32_t B, int32_t H, int32_t T_max,
                                 int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, float scale,
                                 void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* aria_attention_decode_devlen over a paged KV cache (continuous batching).  k_pool / v_pool [n_pages, H, 256, 128] bf16 (page
 * stride page_stride, head stride pool_stride_h, 128-element rows); block_table int32 [R, >= max_pages] at row stride
 * block_table_stride: row r's keys [256 s, 256 s + 256) are rows [0, 256) of page block_table[r, s].  Row r attends to its keys
 * [0, min(lens[r], 256 max_pages)) (lens: DEVICE int32 [R]); q as aria_attention_decode's with R rows; out [R, H*128].
 * The page size is the decode split, so split s reads exactly page s, with the contiguous kernel's key order and arithmetic:
 * row r is bit-identical to aria_attention_decode_devlen on a contiguous cache holding the same keys.  Splits past
 * ceil(lens[r] / 256) read no page and write (-inf, 0, 0); the merge reads the live splits only.  A live split whose entry is
 * not in [0, n_pages) reads nothing.  workspace: aria_attention_decode_workspace_bytes(R, H, 256 * max_pages). */
int aria_attention_decode_paged(const void* q, const void* k_pool, const void* v_pool, const int32_t* block_table,
                                int64_t block_table_stride, int32_t max_pages, int32_t n_pages, const int32_t* lens, void* out,
                                int32_t R, int32_t H, int64_t q_stride_b, int64_t q_stride_h, int64_t page_stride,
                                int64_t pool_stride_h, float scale, void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* aria_attention_decode_paged over fp8 KV pages: k_pool / v_pool e4m3 codes [n_pages, H, 256, 128] (element = byte strides
 * page_stride / pool_stride_h, multiples of 16) and k_scale / v_scale fp32 [n_pages, H, 256] (strides scale_page_stride /
 * scale_stride_h), one scale per (page, head, row).  Split s of row r reads page block_table[r, s] and its scale rows, with the
 * arithmetic of aria_attention_decode_devlen_fp8: row r is bit-identical to that entry on a contiguous cache holding the same
 * codes and scales (no key mask).  Same block table, lens, q, out and workspace contracts as aria_attention_decode_paged. */
int aria_attention_decode_paged_fp8(const void* q, const void* k_pool, const void* v_pool, const float* k_scale, const float* v_scale,
                                    const int32_t* block_table, int64_t block_table_stride, int32_t max_pages, int32_t n_pages,
                                    const int32_t* lens, void* out, int32_t R, int32_t H, int64_t q_stride_b, int64_t q_stride_h,
                                    int64_t page_stride, int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h,
                                    float scale, void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* aria_attention_decode / aria_attention_decode_devlen over an fp8 KV cache: k, v are e4m3 codes [B,H,T_max,128] (element = byte
 * strides kv_stride_b / kv_stride_h, multiples of 16), k_scale / v_scale fp32 [B,H,T_max] at scale_stride_b / scale_stride_h, one
 * scale per (row, head, token): key t of (b, h) is code * scale.  The key scale multiplies the reduced dot product q.code and the
 * value weight is p * v_scale.  Same split size, key assignment and update order as the bf16 kernels, so with power-of-two
 * scales the output is bit-identical to the bf16 entry run on the bf16 tensors code * scale.  Same workspace query, same
 * key_mask / lens contracts (rows at or past lens[b] are never read). */
int aria_attention_decode_fp8(const void* q, const void* k, const void* v, const float* k_scale, const float* v_scale, void* out,
                              const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tk, int64_t q_stride_b, int64_t q_stride_h,
                              int64_t kv_stride_b, int64_t kv_stride_h, int64_t scale_stride_b, int64_t scale_stride_h, float scale,
                              void* workspace, int64_t workspace_bytes, aria_stream_t stream);
int aria_attention_decode_devlen_fp8(const void* q, const void* k, const void* v, const float* k_scale, const float* v_scale,
                                     void* out, const uint8_t* key_mask, int64_t key_mask_stride, const int32_t* lens, int32_t B,
                                     int32_t H, int32_t T_max, int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b,
                                     int64_t kv_stride_h, int64_t scale_stride_b, int64_t scale_stride_h, float scale,
                                     void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* Single-token decode of R = G*n rows in G groups of n (row r = g*n + j) that share a prompt (prefix) cache.  Row r attends to
 * prefix rows [0, min(prefix_lens[g], P_max)) of prefix_k / prefix_v [G,H,P_max,128] (strides prefix_stride_b / _h) minus the
 * keys of prefix_mask [G, >= P_max] uint8 (row stride prefix_mask_stride, 1 = masked out; or NULL), then to its own tail rows
 * [0, min(tail_lens[r], N_max)) of tail_k / tail_v [R,H,N_max,128].  prefix_lens int32 [G] and tail_lens int32 [R] are DEVICE
 * values (one captured step serves every length); q as aria_attention_decode's with R rows; out [R, H*128].
 * Result: row r is bit-identical to aria_attention_decode_devlen on the expanded layout, a cache of row r that holds the
 * prefix at [0, P_g), masked rows [P_g, S_g) with S_g = 256*ceil(P_g/256), the tail at [S_g, S_g + tail_lens[r]), and
 * lens[r] = S_g + tail_lens[r].  Rows at or past the lengths, and masked prefix rows, are never read.  Each prefix key and value is
 * read from HBM once per (group, head).  Cache strides are multiples of 8 elements.
 * workspace: aria_attention_decode_shared_prefix_workspace_bytes(G, n, H, P_max, N_max) (-1 for a non-positive size). */
int aria_attention_decode_shared_prefix(const void* q, const void* prefix_k, const void* prefix_v, const int32_t* prefix_lens,
                                        const uint8_t* prefix_mask, int64_t prefix_mask_stride, const void* tail_k, const void* tail_v,
                                        const int32_t* tail_lens, void* out, int32_t G, int32_t n, int32_t H, int32_t P_max,
                                        int32_t N_max, int64_t q_stride_b, int64_t q_stride_h, int64_t prefix_stride_b,
                                        int64_t prefix_stride_h, int64_t tail_stride_b, int64_t tail_stride_h, float scale,
                                        void* workspace, int64_t workspace_bytes, aria_stream_t stream);
int64_t aria_attention_decode_shared_prefix_workspace_bytes(int32_t G, int32_t n, int32_t H, int32_t P_max, int32_t N_max);
/* Causal prefill of B suffixes that share one prefix (many questions about one image).  The suffixes are packed along one
 * sequence: q, k, v [1, H, >= S_tot, 128] (head strides q_stride_h / kv_stride_h, 128-element rows), row b's suffix at packed rows
 * [cu_seqlens[b], cu_seqlens[b+1]) (DEVICE int32 [B+1], nondecreasing from 0 to S_tot, every suffix >= 1 row).  The prefix is
 * rows [0, P) of prefix_k / prefix_v [1, H, P_max, 128] (head stride prefix_stride_h).  The query at packed row q of suffix b
 * sees every prefix key (no mask) and the packed keys [cu_seqlens[b], q].  out [S_tot, H*128] bf16 (the o_proj input).
 * One CTA per (head, 128 packed queries) on aria_attention_fwd's pipeline: the prefix in 128-key tiles from key 0, then each
 * suffix present in the query tile in 128-key tiles from its own start.  A row's arithmetic is the prefix tiles, then its own
 * tiles, so with P % 128 == 0 row b is bit-identical to aria_attention_fwd (causal) on its own [prefix, suffix b] layout.
 * Prefix rows at or past P and packed rows at or past S_tot are never read.  Strides are multiples of 8 elements.  No workspace. */
int aria_attention_prefill_shared_prefix(const void* q, const void* k, const void* v, const void* prefix_k, const void* prefix_v,
                                         const int32_t* cu_seqlens, void* out, int32_t B, int32_t H, int32_t S_tot, int32_t P,
                                         int32_t P_max, int64_t q_stride_h, int64_t kv_stride_h, int64_t prefix_stride_h,
                                         float scale, aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Generation: sampling, KV append, decode-state advance (one decode step has no host integer in it)
 * ------------------------------------------------------------------------------------------------ */
/* Next token of each row from bf16 logits [B, V] (row r at logits + r * logits_stride elements; stride 0 repeats one row),
 * following transformers' warper chain on an fp32 copy: TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper ->
 * softmax -> multinomial, written to next_ids [B] int64.
 *   temperature == 0: greedy, argmax with ties to the lowest id (torch.argmax); top_k / top_p are then not applied.
 *   top_k in [1, 1024] keeps every logit >= the k-th largest (ties kept); 0 = off.  top_p in (0, 1]: HF's rule over the top-k
 *   survivors (ascending cumulative probability <= 1 - top_p removed, the largest always kept; boundary ties removed lowest id
 *   first).  top_k == 0 with top_p < 1 (a full-vocabulary nucleus) returns ARIA_ERR_UNSUPPORTED.
 *   Sampling is Gumbel-max with Philox4x32-10 noise keyed by `seed`, counter (vocabulary index, row, *rng_offset): the same
 *   seed and offset give the same tokens; it is NOT torch's generator stream.  rng_offset: device uint64, or NULL for 0.
 *   probs_out [B, V] fp32 or NULL: the final normalised distribution (zero outside the kept set; one-hot when greedy).
 * B <= 2^20, V <= 2^24.  One CTA of 1024 threads per row. */
int aria_sample_tokens(const void* logits, int64_t logits_stride, int64_t* next_ids, float* probs_out, int32_t B, int32_t V,
                       float temperature, int32_t top_k, float top_p, uint64_t seed, const uint64_t* rng_offset,
                       aria_stream_t stream);
/* Copy the new k and v rows k_new / v_new [B, H, 128] (element strides new_stride_b / new_stride_h) into the caches
 * [B, H, T_max, 128] (strides cache_stride_b / cache_stride_h) at the device row pos[b] (int32 [B]); a row outside
 * [0, T_max) is not written.  Strides must be multiples of 8 elements. */
int aria_kv_append(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_cache, void* v_cache,
                   int64_t cache_stride_b, int64_t cache_stride_h, const int32_t* pos, int32_t B, int32_t H, int32_t T_max,
                   aria_stream_t stream);
/* Copy the packed suffix rows k / v [1, H, >= S_tot, 128] (head stride src_stride_h) of an
 * aria_attention_prefill_shared_prefix call into the tails tail_k / tail_v [B*n, H, N_max, 128] (strides tail_stride_b /
 * tail_stride_h): packed row s of suffix b (cu_seqlens as there, DEVICE int32 [B+1]) goes to row s - cu_seqlens[b] of tails
 * b*n .. b*n + n-1.  Tail rows at or past each suffix's length are not written, nor rows past N_max.  Strides are multiples of 8
 * elements, and the tails of different rows do not overlap (tail_stride_b >= H * tail_stride_h). */
int aria_kv_scatter_tails(const void* k, const void* v, int64_t src_stride_h, void* tail_k, void* tail_v, int64_t tail_stride_b,
                          int64_t tail_stride_h, const int32_t* cu_seqlens, int32_t B, int32_t n, int32_t H, int32_t S_tot,
                          int32_t N_max, aria_stream_t stream);
/* fp8 KV cache: e4m3 codes k_cache / v_cache [B, H, T_max, 128] (element = byte strides cache_stride_b / cache_stride_h, multiples
 * of 16) and fp32 scales k_scale / v_scale [B, H, T_max] (strides scale_stride_b / scale_stride_h), one per (row, head, token):
 *   scale = max |x| / 448 (IEEE division; an all-zero row gets 1), code = e4m3(x / scale) (round to nearest even, saturating),
 * bit for bit (x.float() / scale[..., None]).to(torch.float8_e4m3fn).  bf16 sources / outputs have 128-element rows at strides
 * that are multiples of 8 elements.  The store and the append share one device quantiser, so a row gets the same bits from both.
 * aria_kv_store_fp8: source rows [0, n_rows) ([B, H, n_rows, 128]) -> cache rows [row0, row0 + n_rows) (row0 + n_rows <= T_max). */
int aria_kv_store_fp8(const void* k_src, const void* v_src, int64_t src_stride_b, int64_t src_stride_h, void* k_cache, void* v_cache,
                      float* k_scale, float* v_scale, int64_t cache_stride_b, int64_t cache_stride_h, int64_t scale_stride_b,
                      int64_t scale_stride_h, int32_t row0, int32_t n_rows, int32_t B, int32_t H, int32_t T_max, aria_stream_t stream);
/* aria_kv_append for the fp8 cache: k_new / v_new [B, H, 128] -> cache row pos[b] (device int32 [B]); a row outside [0, T_max)
 * is not written. */
int aria_kv_append_fp8(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_cache, void* v_cache,
                       float* k_scale, float* v_scale, int64_t cache_stride_b, int64_t cache_stride_h, int64_t scale_stride_b,
                       int64_t scale_stride_h, const int32_t* pos, int32_t B, int32_t H, int32_t T_max, aria_stream_t stream);
/* Dequantise cache rows [0, n_rows) (n_rows <= T_max) into bf16 k_out / v_out [B, H, >= n_rows, 128]: bf16(code * scale), the
 * fp32 product rounded to nearest even. */
int aria_kv_load_fp8(const void* k_cache, const void* v_cache, const float* k_scale, const float* v_scale, int64_t cache_stride_b,
                     int64_t cache_stride_h, int64_t scale_stride_b, int64_t scale_stride_h, void* k_out, void* v_out,
                     int64_t out_stride_b, int64_t out_stride_h, int32_t n_rows, int32_t B, int32_t H, int32_t T_max,
                     aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Prompt-lookup decoding: a step verifies Q = K + 1 tokens per row (the last token, then K drafts from the row's history)
 * ------------------------------------------------------------------------------------------------ */
/* Decode attention of Q consecutive queries per row: q [B, H, Q, 128] (element strides q_stride_b / q_stride_h / q_stride_q,
 * multiples of 4), cache k / v [B, H, T_max, 128] bf16 (strides kv_stride_b / kv_stride_h, multiples of 8).  Query i of row b sees
 * cache rows [0, lens[b * Q + i]) (DEVICE int32 [B * Q]) minus key_mask (uint8 [B, >= T_max] at row stride key_mask_stride,
 * 1 = masked out, or NULL).  out [B, Q, H*128] bf16.  One CTA per (row, head, 256-key split) stages the split's live keys and
 * values once and serves every query with aria_attention_decode_devlen's per-query arithmetic; the devlen merge follows.  So
 * query i of row b is bit-identical to aria_attention_decode_devlen at lens = lens[b * Q + i].  Q <= 16.
 * workspace_bytes >= aria_attention_decode_workspace_bytes(B * Q, H, T_max). */
int aria_attention_decode_multi(const void* q, const void* k, const void* v, void* out, const uint8_t* key_mask, int64_t key_mask_stride,
                                const int32_t* lens, int32_t B, int32_t Q, int32_t H, int32_t T_max, int64_t q_stride_b,
                                int64_t q_stride_h, int64_t q_stride_q, int64_t kv_stride_b, int64_t kv_stride_h, float scale,
                                void* workspace, int64_t workspace_bytes, aria_stream_t stream);
/* aria_kv_append for Q rows per row: k_new / v_new [B, H, Q, 128] (element strides new_stride_b / new_stride_h / new_stride_q) ->
 * cache rows pos[b] + i (pos DEVICE int32 [B]); rows outside [0, T_max) are not written.  Strides are multiples of 8 elements. */
int aria_kv_append_rows(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, int64_t new_stride_q,
                        void* k_cache, void* v_cache, int64_t cache_stride_b, int64_t cache_stride_h, const int32_t* pos, int32_t B,
                        int32_t Q, int32_t H, int32_t T_max, aria_stream_t stream);
/* aria_sample_tokens over R logits rows, where row r draws the Philox noise of row noise_rows[r] (DEVICE int32 [R]) at offset
 * offsets[r] (DEVICE uint64 [R]) instead of (r, *rng_offset).  Same warper chain, same kernel code; no probs output. */
int aria_sample_tokens_rows(const void* logits, int64_t logits_stride, int64_t* next_ids, int32_t R, int32_t V, float temperature,
                            int32_t top_k, float top_p, uint64_t seed, const int32_t* noise_rows, const uint64_t* offsets,
                            aria_stream_t stream);
/* Continuous batching over a paged KV cache (pools [n_pages, H, 256, 128] bf16 at page_stride / pool_stride_h, block table int32
 * [R, >= max_pages] at row stride block_table_stride, as aria_attention_decode_paged's).
 * aria_kv_append_paged: the k and v rows of slot r, k_new / v_new [R, H, 128] (strides new_stride_b / new_stride_h), go to row
 * write_pos[r] % 256 of page block_table[r, write_pos[r] / 256] (write_pos: DEVICE int32 [R]).  Nothing is written for a
 * negative write_pos, one at or past 256 * max_pages, or a table entry outside [0, n_pages): an idle or padding slot never
 * writes into another request's pages.  Strides are multiples of 8 elements. */
int aria_kv_append_paged(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_pool, void* v_pool,
                         int64_t page_stride, int64_t pool_stride_h, const int32_t* block_table, int64_t block_table_stride,
                         int32_t max_pages, int32_t n_pages, const int32_t* write_pos, int32_t R, int32_t H, aria_stream_t stream);
/* Rows [0, T) of a one-row contiguous cache k / v [1, H, >= T, 128] (head stride src_stride_h) into the pages of one request:
 * row t goes to row t % 256 of page pages[t / 256] (pages: DEVICE int32 [max_pages], a block-table row); a page entry outside
 * [0, n_pages) is not written.  T <= 256 * max_pages. */
int aria_kv_pages_store(const void* k, const void* v, int64_t src_stride_h, int32_t T, void* k_pool, void* v_pool,
                        int64_t page_stride, int64_t pool_stride_h, const int32_t* pages, int32_t max_pages, int32_t n_pages,
                        int32_t H, aria_stream_t stream);
/* aria_attention_prefill_shared_prefix whose prefix is read from pool pages (prefix caching): key 256 i + r of the prefix is row
 * r of page pages[i] (pages: DEVICE int32 [n_pages_list]) of k_pool / v_pool [n_pages, H, 256, 128] (page_stride /
 * pool_stride_h as aria_attention_decode_paged's).  P is a multiple of 256 with P / 256 <= n_pages_list; P = 0 is no prefix
 * (then pages may be NULL), the varlen forward.  q, k, v, cu_seqlens, out, B, S_tot and the head strides as there.  Every
 * output row is bit-identical to aria_attention_prefill_shared_prefix on a contiguous copy of the same prefix (P = 0:
 * aria_attention_fwd_varlen).  A page entry outside [0, n_pages) reads zeros; packed rows at or past S_tot are never read.
 * No workspace. */
int aria_attention_prefill_paged_prefix(const void* q, const void* k, const void* v, const void* k_pool, const void* v_pool,
                                        const int32_t* pages, int32_t n_pages_list, int32_t n_pages, const int32_t* cu_seqlens,
                                        void* out, int32_t B, int32_t H, int32_t S_tot, int32_t P, int64_t q_stride_h,
                                        int64_t kv_stride_h, int64_t page_stride, int64_t pool_stride_h, float scale,
                                        aria_stream_t stream);
/* aria_attention_prefill_paged_prefix over n_seg packed segments, each after a paged prefix of its own (batched admission):
 * segment b is rows [cu_seqlens[b], cu_seqlens[b + 1]) of q / k / v [1, H, S_tot, 128] (DEVICE int32 [n_seg + 1], increasing
 * from 0 to S_tot) and attends to its prefix_lens[b] cached keys (DEVICE int32 [n_seg], multiples of 256; key 256 i + r is row r
 * of page page_table[b * page_table_stride + i], DEVICE int32, at least prefix_lens[b] / 256 entries per row) and causally to its
 * own rows -> out [S_tot, H * 128].  Query tiles do not cross segments, so every row of segment b is bit-identical to
 * aria_attention_prefill_paged_prefix run on segment b alone (B = 1) with its own page list and P.  The caller checks the device
 * values; a page entry outside [0, n_pages) reads zeros.  Strides as aria_attention_prefill_paged_prefix's.  No workspace. */
int aria_attention_prefill_paged_varlen(const void* q, const void* k, const void* v, const void* k_pool, const void* v_pool,
                                        const int32_t* page_table, int64_t page_table_stride, int32_t n_pages,
                                        const int32_t* prefix_lens, const int32_t* cu_seqlens, void* out, int32_t n_seg, int32_t H,
                                        int32_t S_tot, int64_t q_stride_h, int64_t kv_stride_h, int64_t page_stride,
                                        int64_t pool_stride_h, float scale, aria_stream_t stream);
/* aria_kv_pages_store for packed segments: packed row t of segment b (cu_seqlens, prefix_lens and page_table as
 * aria_attention_prefill_paged_varlen's, max_pages columns per table row) is position p = prefix_lens[b] + t - cu_seqlens[b] of
 * its request and goes to row p % 256 of page page_table[b, p / 256].  Nothing is written for p past 256 * max_pages, a table
 * entry outside [0, n_pages), or the null page 0.  Each segment's pages are bit-identical to aria_kv_pages_store on it alone. */
int aria_kv_pages_store_varlen(const void* k, const void* v, int64_t src_stride_h, int32_t S_tot, void* k_pool, void* v_pool,
                               int64_t page_stride, int64_t pool_stride_h, const int32_t* page_table, int64_t page_table_stride,
                               int32_t max_pages, int32_t n_pages, const int32_t* prefix_lens, const int32_t* cu_seqlens,
                               int32_t n_seg, int32_t H, aria_stream_t stream);
/* fp8 KV pages: e4m3 code pools k_pool / v_pool [n_pages, H, 256, 128] and fp32 scale pools k_scale / v_scale [n_pages, H, 256]
 * (strides as aria_attention_decode_paged_fp8's), with the quantiser and dequantiser of aria_kv_store_fp8 / aria_kv_load_fp8.
 * aria_kv_append_paged_fp8: aria_kv_append_paged that quantises: row r of k_new / v_new goes to row write_pos[r] % 256 of page
 *   block_table[r, write_pos[r] / 256] with the codes and scale aria_kv_append_fp8 gives it.  Nothing is written for a negative
 *   write_pos, one at or past 256 * max_pages, a table entry outside [0, n_pages), or the null page 0. */
int aria_kv_append_paged_fp8(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_pool,
                             void* v_pool, float* k_scale, float* v_scale, int64_t page_stride, int64_t pool_stride_h,
                             int64_t scale_page_stride, int64_t scale_stride_h, const int32_t* block_table,
                             int64_t block_table_stride, int32_t max_pages, int32_t n_pages, const int32_t* write_pos, int32_t R,
                             int32_t H, aria_stream_t stream);
/* aria_kv_pages_store_varlen that quantises: packed row t of segment b (k / v [1, H, >= S_tot, 128] bf16, head stride
 * src_stride_h) goes to the page row aria_kv_pages_store_varlen gives it, as codes and a scale, and bf16(code * scale) is written
 * back over the source row in place (every row), so attention over k / v then reads what the pages hold.  Never writes the null
 * page 0 nor a page that is not listed. */
int aria_kv_pages_store_varlen_fp8(void* k, void* v, int64_t src_stride_h, int32_t S_tot, void* k_pool, void* v_pool, float* k_scale,
                                   float* v_scale, int64_t page_stride, int64_t pool_stride_h, int64_t scale_page_stride,
                                   int64_t scale_stride_h, const int32_t* page_table, int64_t page_table_stride, int32_t max_pages,
                                   int32_t n_pages, const int32_t* prefix_lens, const int32_t* cu_seqlens, int32_t n_seg, int32_t H,
                                   aria_stream_t stream);
/* Dequantise pages pages[i] (DEVICE int32 [n_list]) of the fp8 pools into page i of bf16 pools k_out / v_out [n_list, H, 256, 128]
 * (strides out_page_stride / out_stride_h, multiples of 8): bf16(code * scale), aria_kv_load_fp8's values.  An entry outside
 * [0, n_pages) gives zeros. */
int aria_kv_pages_load_fp8(const void* k_pool, const void* v_pool, const float* k_scale, const float* v_scale, int64_t page_stride,
                           int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h, const int32_t* pages,
                           int32_t n_list, int32_t n_pages, void* k_out, void* v_out, int64_t out_page_stride,
                           int64_t out_stride_h, int32_t H, aria_stream_t stream);
/* aria_sample_tokens_rows with every sampling parameter per row, from DEVICE arrays [R]: temperature (0 = greedy), top_k, top_p,
 * seed (uint64), noise row and offset.  Row r is bit-identical to aria_sample_tokens run alone on that row with its scalars at
 * rng_offset = offsets[r] as row noise_rows[r].  The caller checks the parameters as aria_sample_tokens does; out-of-range
 * entries are brought into range (a non-positive or non-finite temperature is greedy, top_k is clamped to [0, 1024], and top_p
 * is 1 without a top_k) rather than read past the kernel's buffers.  R <= 2^20, V <= 2^24. */
int aria_sample_tokens_slots(const void* logits, int64_t logits_stride, int64_t* next_ids, int32_t R, int32_t V,
                             const float* temperature, const int32_t* top_k, const float* top_p, const uint64_t* seed,
                             const int32_t* noise_rows, const uint64_t* offsets, aria_stream_t stream);
/* aria_sample_tokens_slots behind Hugging Face's logits processors (transformers' GenerationMixin order), every parameter per
 * row from DEVICE arrays [R]: temperature, top_k, top_p and seed as there, min_p (fp32, 0 = off), repetition_penalty (fp32,
 * 1 = off) and min_new_tokens (int32).  Row r's scores are the fp32 values of its bf16 logits where
 *   - an id set in its presence bitmap (DEVICE uint32 [R, ceil(V / 32)], bit i of word i / 32; aria_presence_set) becomes
 *     x < 0 ? x * penalty : x / penalty, IEEE-rounded (RepetitionPenaltyLogitsProcessor);
 *   - while the row has emitted fewer than min_new_tokens tokens, every EOS id (HOST array of n_eos <= 8 ids, copied at the
 *     call) becomes -inf (MinNewTokensLengthLogitsProcessor);
 * then greedy takes their argmax (ties to the lowest id), and sampling runs temperature -> top-k -> top-p as aria_sample_tokens
 * does, then min-p: a survivor with p < min_p * max p, p the softmax over the survivors, is removed (MinPLogitsWarper; the
 * largest always stays).  min_p also applies with top_k = 0.  probs_out [R, V] or NULL: the final distribution, renormalised
 * over what min-p keeps.  Row r draws the noise of row noise_rows[r] (DEVICE int32 [R], or NULL for row r) at offset
 * rng_offset[r] (offset_per_row) or rng_offset[0] (DEVICE uint64); n_emitted (DEVICE int32) is likewise per row or one value.
 * A row whose processors are off (penalty 1, min_p 0, min_new_tokens 0) gets aria_sample_tokens_slots' token and
 * aria_sample_tokens' probs_out bit for bit.  Out-of-range entries are brought into range as there (a non-positive or
 * non-finite penalty is 1, a min_p outside (0, 1] is 0).  R <= 2^20, V <= 2^18 (the bitmap is staged in shared memory). */
int aria_sample_tokens_processed(const void* logits, int64_t logits_stride, int64_t* next_ids, float* probs_out, int32_t R,
                                 int32_t V, const float* temperature, const int32_t* top_k, const float* top_p, const float* min_p,
                                 const uint64_t* seed, const float* repetition_penalty, const int32_t* min_new_tokens,
                                 const uint32_t* presence, const int32_t* noise_rows, const uint64_t* rng_offset,
                                 int32_t offset_per_row, const int32_t* n_emitted, int32_t emitted_per_row, const int64_t* eos_ids,
                                 int32_t n_eos, aria_stream_t stream);
/* Token-presence bitmaps for aria_sample_tokens_processed: for each row r < R, bitmap row r (uint32 [R, ceil(V / 32)]) is
 * cleared first when `clear`, then bit id is set for each of the row's first n ids, ids + r * ids_stride (DEVICE int64),
 * n = lengths[r] clamped to [0, T] (DEVICE int32 [R]) or T when lengths is NULL.  Ids outside [0, V) are skipped.
 * R <= 2^20, V <= 2^18, one CTA per row. */
int aria_presence_set(const int64_t* ids, int64_t ids_stride, int32_t R, int32_t T, const int32_t* lengths, int32_t clear,
                      uint32_t* bitmap, int32_t V, aria_stream_t stream);
/* Token log-probabilities of bf16 logits [R, V] (row r at logits + r * logits_stride, contiguous within a row), one CTA per row,
 * under the row's raw distribution: lp(t) = (x_t - m) - log(sum_i exp(x_i - m)), m = max_i x_i, in fp32 summed in a fixed order.
 * Row r writes output entry o = r * cols + c: logprobs[o] = lp(tokens[r]) (NaN for a token outside [0, V)), and its n largest
 * logits by (value desc, id asc) to top_ids[o * n_max + j] / top_logprobs[o * n_max + j], j < n; entries n .. n_max - 1 (also
 * those past V) get id -1 and logprob -inf.  n = n_row[r] (DEVICE int32 [R], -1 skips the row; clamped to n_max) or n_max when
 * n_row is NULL; 0 <= n_max <= 20.  Column c: col NULL -> 0; else col[r] (col_per_row) or col[0], taken mod ring when ring > 0;
 * a column outside [0, cols) skips the row.  finished (DEVICE uint8 [R] or NULL): a finished row gets the filler (logprob 0,
 * ids -1, logprobs -inf) when finished_fill, else is left untouched.  A row's result depends only on its logits, token and n.
 * R <= 2^20, V <= 2^24. */
int aria_token_logprobs(const void* logits, int64_t logits_stride, const int64_t* tokens, int32_t R, int32_t V, int32_t n_max,
                        const int32_t* n_row, const int32_t* col, int32_t col_per_row, int32_t ring, const uint8_t* finished,
                        int32_t finished_fill, float* logprobs, int32_t* top_ids, float* top_logprobs, int32_t cols,
                        aria_stream_t stream);
/* Decode-state advance after the sampler, per row (generate() and continuous batching).  For each row r < R that is not
 * finished: its token next_ids[r] is stored at out_tokens[r, n_out[r]] ([R, out_stride] int32) and n_out[r] + 1; the row
 * finishes when the token is one of the n_eos <= 8 EOS ids (HOST array, copied into the launch) or n_out reaches max_new[r];
 * ids_in[r] <- the token (pad_token_id once finished); rope_pos, write_pos, kv_len and rng_offset[r] (uint64) + 1.  A finished
 * row (idle slots are finished) changes nothing.  R <= 1024, one launch. */
int aria_decode_advance_slots(const int64_t* next_ids, int64_t* ids_in, int32_t* out_tokens, int64_t out_stride, int32_t* n_out,
                              const int32_t* max_new, int32_t* rope_pos, int32_t* write_pos, int32_t* kv_len, uint64_t* rng_offset,
                              uint8_t* finished, const int64_t* eos_ids, int32_t n_eos, int64_t pad_token_id, int32_t R,
                              aria_stream_t stream);
/* Drafts from each row's history hist [B, hist_stride] int64 (its first hist_len[b] entries: the prompt after its left padding,
 * then the tokens emitted so far), Hugging Face's PromptLookupCandidateGenerator.get_candidates per row: for n = min(M, len - 1)
 * down to 1, the earliest occurrence of the last n tokens that has a non-empty continuation; the continuation, at most K tokens
 * and not past the history, cut before its first EOS (HOST array of n_eos <= 8 ids); no match: no draft.  The draft is then cut
 * to max_new - 1 - n_out[b] tokens (what a step can still emit after the row's next token), and a finished row has none.
 * Writes drafts [B, K] (row stride draft_stride; entries past a draft repeat the row's last token), draft_len [B], and sets
 * *any_draft = 1 when a row has a draft (it is never cleared here).  K in [1, 15], M in [1, 16].  One CTA per row. */
int aria_ngram_draft(const int64_t* hist, int64_t hist_stride, const int32_t* hist_len, const uint8_t* finished, const int32_t* n_out,
                     int32_t max_new, int64_t* drafts, int64_t draft_stride, int32_t* draft_len, int32_t* any_draft, int32_t B,
                     int32_t K, int32_t M, const int64_t* eos_ids, int32_t n_eos, aria_stream_t stream);
/* After aria_sample_tokens_rows on a step of width Q (1, or Kp1 = K + 1 with step_ids [B, Q] = the last token, then the drafts of
 * draft_len [B]), per row b that is neither finished nor at max_new tokens: a = the number of leading drafts equal to the target
 * before them (targets [B * Q]); emits targets t_0 .. t_a to out_tokens[b, n_out[b] ...] ([B, max_new]) and to the history,
 * stopping after the first EOS id (finished[b] = 1) and at max_new tokens; then n_out, hist_len, rope_pos, write_pos and kv_len
 * move on by the count emitted.  Every row then gets the next step's inputs: ids1[b] and idsk[b * Kp1] = its last token,
 * pos_k / lens_k [B * Kp1] = rope_pos + i / kv_len + i, off1[b] = n_out[b], offk[b * Kp1 + i] = n_out[b] + i.
 * status[0] = every row finished or at max_new, status[1] = 0 (aria_ngram_draft sets it); counters[0] += drafts verified,
 * counters[1] += drafts accepted.  Out tokens are not written past a row's end: the caller fills them with pad first.
 * B <= 1024, one launch. */
int aria_lookup_accept_advance(const int64_t* targets, const int64_t* step_ids, const int32_t* draft_len, int32_t Q, int64_t* ids1,
                               int64_t* idsk, int32_t Kp1, int32_t* pos_k, int32_t* lens_k, uint64_t* off1, uint64_t* offk,
                               int64_t* out_tokens, int32_t max_new, int64_t* hist, int64_t hist_stride, int32_t* hist_len,
                               int32_t* n_out, uint8_t* finished, int32_t* rope_pos, int32_t* write_pos, int32_t* kv_len,
                               int32_t* status, uint64_t* counters, const int64_t* eos_ids, int32_t n_eos, int32_t B,
                               aria_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Stop strings (Hugging Face's StopStringCriteria), checked after the decode advance
 * ------------------------------------------------------------------------------------------------ */
/* The vocabulary table: token id i's cleaned string is vocab_bytes[vocab_offsets[i], vocab_offsets[i + 1]) (UTF-8), for
 * 0 <= i < V; ids outside [0, V) match nothing.  A stop set is up to 16 strings of stop_bytes [16, 512] (UTF-8) with byte
 * lengths stop_lens [16] (0 = unused), and *lookback: the tokens HF looks at, the characters of the longest string (<= 128).
 * Every array is DEVICE memory.  A row stops after its final token when that token completes a string: some byte prefix of
 * it ends with the string's last bytes (or holds the whole string), and the tokens before it, walking back within the
 * lookback window, cover the rest of the string, the earliest one allowed to run off its start.  One warp per row. */
/* R <= 1024 rows, row r with its own stop set (stop_bytes [R, 16, 512], stop_lens [R, 16], lookback [R]; lookback 0 = no
 * strings) and its own stop ids (stop_ids [R, 8] int64, the first n_stop_ids[r] of them).  Its history is its last
 * tail_len[r] <= 128 prompt ids, right-aligned in prompt_tail [R, 128] int64, then out_tokens[r, 0 .. n_out[r]) ([R, out_stride]
 * int32).  A row that is not finished and whose final token is one of its stop ids or completes one of its strings gets
 * finished[r] = 1 and ids_in[r] = pad_token_id. */
int aria_stop_check_slots(const uint8_t* vocab_bytes, const int32_t* vocab_offsets, int32_t V, const uint8_t* stop_bytes,
                          const int32_t* stop_lens, const int32_t* lookback, const int64_t* stop_ids, const int32_t* n_stop_ids,
                          const int64_t* prompt_tail, const int32_t* tail_len, const int32_t* out_tokens, int64_t out_stride,
                          const int32_t* n_out, uint8_t* finished, int64_t* ids_in, int64_t pad_token_id, int32_t R,
                          aria_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ARIA_B200_H */
