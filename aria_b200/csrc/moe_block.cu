// aria_moe_block_fwd: the whole MoELayer.forward (aria/model/moe_lm.py:548-577) behind ONE C-ABI call.
//
//   router GEMM + top-k + softmax + histogram (moe_lm.py:190-201, 261-269)  -> aria_router_topk
//   stable counting sort by expert            (moe_lm.py:313-334)           -> aria_build_permutation, aria_permute_rows
//   fc1 grouped GEMM + glu, fc2 grouped GEMM  (moe_lm.py:467-525)           -> grouped_gemm x 2 (device-resident offsets: no
//                                                                              tokens_per_expert.cpu() sync, moe_lm.py:478)
//   shared experts                            (moe_lm.py:368-395)           -> aria_gemm x 2 on `side_stream` when given: the
//                                                                              branch is independent until the final add
//   unpermute + score-weighted sum + `+= shared` (moe_lm.py:336-365, 575-576) -> aria_unpermute_combine
//
// Host-side driver only (SURVEY.md §8b "moe_block_fwd (fused driver)"): it owns the launch ORDER, the workspace carve-up and
// the fork/join of the shared-expert branch, so that the reference-side binding is one call per layer instead of nine; the
// kernels are the same ones the individual entries launch.  No allocation, no host sync, graph-capturable.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/aria_b200.h"
#include "common.cuh"

namespace {

constexpr int64_t kAlign = 256;
inline int64_t al(int64_t n) { return (n + kAlign - 1) / kAlign * kAlign; }

struct BlockWs {
  int64_t idx, scores, counts, offsets, dest, src, logits, permuted, h, y, hs, shared, total;
  int64_t sxq, sxs, shq, shs;  // shared_fp8: e4m3 rows and row scales of x and of h for the W8A8 shared experts
};

// shared_fp8 appends the shared branch's quantised rows after the regions of the other modes, which keep their offsets and
// total.  They are the branch's own: it runs on the side stream, concurrently with everything of the routed branch.
BlockWs carve(int64_t T, int32_t d, int32_t E, int32_t k, int32_t I, int32_t Is, bool shared_fp8 = false) {
  BlockWs w{};
  int64_t o = 0;
  const int64_t R = T * k;
  w.idx = o;      o += al(R * 4);
  w.scores = o;   o += al(R * 2);
  w.counts = o;   o += al(static_cast<int64_t>(E) * 4);
  w.offsets = o;  o += al(static_cast<int64_t>(E + 1) * 4);
  w.dest = o;     o += al(R * 4);
  w.src = o;      o += al(R * 4);
  w.logits = o;   o += al(T * E * 2);
  w.permuted = o; o += al(R * d * 2);
  w.h = o;        o += al(R * I * 2);
  w.y = o;        o += al(R * d * 2);
  w.hs = o;       o += al(T * Is * 2);
  w.shared = o;   o += al(T * d * 2);
  if (shared_fp8) {
    w.sxq = o;    o += al(T * d);
    w.sxs = o;    o += al(T * 4);
    w.shq = o;    o += al(T * Is);
    w.shs = o;    o += al(T * 4);
  }
  w.total = o;
  return w;
}

// fork / join events of the shared-expert branch, one pair per device (created once; recording an event is legal during
// stream capture and becomes a dependency edge of the graph)
cudaEvent_t* branch_events() {
  static cudaEvent_t ev[aria::kMaxDevices][2] = {};
  static bool made[aria::kMaxDevices] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= aria::kMaxDevices) return nullptr;
  if (!made[dev]) {
    if (cudaEventCreateWithFlags(&ev[dev][0], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&ev[dev][1], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    made[dev] = true;
  }
  return ev[dev];
}

// W8A8 keeps the workspace of the other modes: the e4m3 rows and scales of fc1's input go to the `permuted` region (R d 2
// bytes), those of h to the same region once fc1 has consumed the first ones (R I bytes, hence I <= 2 d), and h's row
// scales to the `src` region, dead after the gather (R 4 bytes: at I = 2 d the rows of h fill `permuted`).
struct W8a8Ws {
  int64_t xq, xs, hq, hs;
};
inline int64_t al16(int64_t n) { return (n + 15) / 16 * 16; }
bool w8a8_fits(int64_t R, int32_t d, int32_t I, const BlockWs& ws, W8a8Ws& o) {
  o.xq = ws.permuted;
  o.xs = ws.permuted + al16(R * d);
  o.hq = ws.permuted;
  o.hs = ws.src;
  const int64_t permuted_bytes = ws.h - ws.permuted, src_bytes = ws.logits - ws.src;
  return al16(R * d) + R * 4 <= permuted_bytes && R * I <= permuted_bytes && R * 4 <= src_bytes;
}

// The e4m3 shared-expert weights' column scales (SharedScales::gate == NULL: bf16 shared experts)
struct SharedScales {
  const float* gate;
  const float* up;
  const float* down;
};

// The whole block.  fc1_scale / fc2_scale NULL: bf16 expert weights; given: fc1_w / fc2_w are e4m3 with per-(expert, column)
// fp32 scales and the two expert GEMMs run the fp8-weight grouped GEMM, or with w8a8 aria_grouped_gemm_w8a8 on K-major weights
// ([E, 2I, d] / [E, d, I]) and row-quantised activations.  With shared scales, the shared experts are W8A8 (aria_gemm_w8a8 on
// row-quantised x and h).  Every other launch is the same.
int moe_block_run(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w, const float* fc1_scale,
                  const float* fc2_scale, bool w8a8, const void* gate_w, const void* up_w, const void* down_w, void* out, int64_t T,
                  int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared, const int32_t* forced_top_idx, void* workspace,
                  int64_t workspace_bytes, aria_stream_t stream, aria_stream_t side_stream,
                  const SharedScales& ss = SharedScales{nullptr, nullptr, nullptr}) {
  if (!x || !w_router || !fc1_w || !fc2_w || !out || !workspace) return ARIA_ERR_BAD_ARG;
  if (T <= 0 || d <= 0 || E <= 0 || E > 64 || k <= 0 || k > 8 || k > E || I <= 0 || I_shared < 0) return ARIA_ERR_BAD_ARG;
  if (I_shared > 0 && (!gate_w || !up_w || !down_w)) return ARIA_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(workspace) & 15) != 0) return ARIA_ERR_BAD_ARG;
  const bool shared_fp8 = ss.gate != nullptr;
  const BlockWs ws = carve(T, d, E, k, I, I_shared, shared_fp8);
  if (workspace_bytes < ws.total) return ARIA_ERR_BAD_ARG;
  W8a8Ws q{};
  if (w8a8 && !w8a8_fits(T * k, d, I, ws, q)) return ARIA_ERR_BAD_ARG;
  uint8_t* base = static_cast<uint8_t*>(workspace);
  auto at = [&](int64_t off) { return static_cast<void*>(base + off); };
  int32_t* idx = static_cast<int32_t*>(at(ws.idx));
  int32_t* counts = static_cast<int32_t*>(at(ws.counts));
  int32_t* offsets = static_cast<int32_t*>(at(ws.offsets));
  int32_t* dest = static_cast<int32_t*>(at(ws.dest));
  int32_t* src = static_cast<int32_t*>(at(ws.src));
  const int64_t R = T * k;
  cudaStream_t s_main = reinterpret_cast<cudaStream_t>(stream);
  cudaStream_t s_side = reinterpret_cast<cudaStream_t>(side_stream);
  int rc;

  // ---- shared experts: an independent branch (its own stream when the caller provides one)
  const bool fork = I_shared > 0 && s_side != nullptr && s_side != s_main;
  cudaEvent_t* ev = nullptr;
  auto shared_branch = [&](aria_stream_t st) -> int {
    if (shared_fp8) {
      // x -> e4m3 rows -> W8A8 SwiGLU (gate | up) -> h -> e4m3 rows -> W8A8 down
      float* xs = static_cast<float*>(at(ws.sxs));
      float* hs = static_cast<float*>(at(ws.shs));
      int r = aria_permute_quantize_fp8_rows(x, nullptr, at(ws.sxq), xs, T, d, st);
      if (r) return r;
      aria_gemm_desc_t g;
      memset(&g, 0, sizeof(g));
      g.a = at(ws.sxq); g.lda = d; g.m = T; g.n = I_shared; g.k = d;
      g.b[0] = gate_w; g.b[1] = up_w; g.n_seg = 2; g.b_layout = ARIA_B_NK; g.num_groups = 1;
      g.epilogue = ARIA_EPI_SWIGLU;
      g.out[0] = at(ws.hs); g.ldo = I_shared;
      const float* gu_scale[3] = {ss.gate, ss.up, nullptr};
      if ((r = aria_gemm_w8a8(&g, xs, gu_scale, st))) return r;
      if ((r = aria_permute_quantize_fp8_rows(at(ws.hs), nullptr, at(ws.shq), hs, T, I_shared, st))) return r;
      memset(&g, 0, sizeof(g));
      g.a = at(ws.shq); g.lda = I_shared; g.m = T; g.n = d; g.k = I_shared;
      g.b[0] = down_w; g.n_seg = 1; g.b_layout = ARIA_B_NK; g.num_groups = 1;
      g.epilogue = ARIA_EPI_LINEAR;
      g.out[0] = at(ws.shared); g.ldo = d;
      const float* d_scale[3] = {ss.down, nullptr, nullptr};
      return aria_gemm_w8a8(&g, hs, d_scale, st);
    }
    aria_gemm_desc_t g;
    memset(&g, 0, sizeof(g));
    g.a = x; g.lda = d; g.m = T; g.n = I_shared; g.k = d;
    g.b[0] = gate_w; g.b[1] = up_w; g.n_seg = 2; g.b_layout = ARIA_B_NK; g.num_groups = 1;
    g.epilogue = ARIA_EPI_SWIGLU;
    g.out[0] = at(ws.hs); g.ldo = I_shared;
    int r = aria_gemm(&g, st);
    if (r) return r;
    memset(&g, 0, sizeof(g));
    g.a = at(ws.hs); g.lda = I_shared; g.m = T; g.n = d; g.k = I_shared;
    g.b[0] = down_w; g.n_seg = 1; g.b_layout = ARIA_B_NK; g.num_groups = 1;
    g.epilogue = ARIA_EPI_LINEAR;
    g.out[0] = at(ws.shared); g.ldo = d;
    return aria_gemm(&g, st);
  };
  if (fork) {
    ev = branch_events();
    if (!ev) return ARIA_ERR_CUDA;
    if (cudaEventRecord(ev[0], s_main) != cudaSuccess) return ARIA_ERR_CUDA;
    if (cudaStreamWaitEvent(s_side, ev[0], 0) != cudaSuccess) return ARIA_ERR_CUDA;
    if ((rc = shared_branch(side_stream))) return rc;
    if (cudaEventRecord(ev[1], s_side) != cudaSuccess) return ARIA_ERR_CUDA;
  }

  // ---- routed experts
  if (forced_top_idx) {  // parity / replay hook: expert choice given, scores = softmax over the logits at those ids
    if ((rc = aria_router_topk(x, w_router, at(ws.logits), idx, at(ws.scores), counts, T, d, E, k, stream))) return rc;
    if ((rc = aria_route_given_indices(at(ws.logits), forced_top_idx, at(ws.scores), counts, T, E, k, stream))) return rc;
    idx = const_cast<int32_t*>(forced_top_idx);
  } else {
    // (aria_router_topk always materialises the bf16 logits: top-k runs on the ROUNDED values, moe_lm.py:200,261)
    if ((rc = aria_router_topk(x, w_router, at(ws.logits), idx, at(ws.scores), counts, T, d, E, k, stream))) return rc;
  }
  if ((rc = aria_build_permutation(idx, counts, offsets, dest, src, T, E, k, 1, stream))) return rc;
  if (w8a8) {
    float* xs = static_cast<float*>(at(q.xs));
    float* hs = static_cast<float*>(at(q.hs));
    if ((rc = aria_permute_quantize_fp8_rows(x, src, at(q.xq), xs, R, d, stream))) return rc;
    if ((rc = aria_grouped_gemm_w8a8(at(q.xq), xs, fc1_w, fc1_scale, at(ws.h), offsets, R, d, I, E, ARIA_EPI_SWIGLU, stream))) return rc;
    if ((rc = aria_permute_quantize_fp8_rows(at(ws.h), nullptr, at(q.hq), hs, R, I, stream))) return rc;
    if ((rc = aria_grouped_gemm_w8a8(at(q.hq), hs, fc2_w, fc2_scale, at(ws.y), offsets, R, I, d, E, ARIA_EPI_LINEAR, stream))) return rc;
  } else {  // bf16 weights, or e4m3 ones with their scales
    if ((rc = aria_permute_rows(x, src, at(ws.permuted), R, d, stream))) return rc;
    if ((rc = aria::grouped_gemm(at(ws.permuted), fc1_w, fc1_scale, at(ws.h), offsets, R, d, I, E, ARIA_EPI_SWIGLU, s_main)))
      return rc;
    if ((rc = aria::grouped_gemm(at(ws.h), fc2_w, fc2_scale, at(ws.y), offsets, R, I, d, E, ARIA_EPI_LINEAR, s_main))) return rc;
  }

  // ---- join + combine (+ shared)
  const void* shared = nullptr;
  if (I_shared > 0) {
    if (fork) {
      if (cudaStreamWaitEvent(s_main, ev[1], 0) != cudaSuccess) return ARIA_ERR_CUDA;
    } else if ((rc = shared_branch(stream))) {
      return rc;
    }
    shared = at(ws.shared);
  }
  return aria_unpermute_combine(at(ws.y), dest, at(ws.scores), shared, out, T, d, k, stream);
}

}  // namespace

extern "C" int64_t aria_moe_block_fwd_workspace_bytes(int64_t T, int32_t d, int32_t E, int32_t k, int32_t I, int32_t I_shared) {
  if (T <= 0 || d <= 0 || E <= 0 || k <= 0 || I <= 0 || I_shared < 0) return ARIA_ERR_BAD_ARG;
  return carve(T, d, E, k, I, I_shared).total;
}

extern "C" int aria_moe_block_fwd(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w, const void* gate_w,
                                  const void* up_w, const void* down_w, void* out, int64_t T, int32_t d, int32_t E, int32_t k,
                                  int32_t I, int32_t I_shared, const int32_t* forced_top_idx, void* workspace,
                                  int64_t workspace_bytes, aria_stream_t stream, aria_stream_t side_stream) {
  return moe_block_run(x, w_router, fc1_w, fc2_w, nullptr, nullptr, false, gate_w, up_w, down_w, out, T, d, E, k, I, I_shared,
                       forced_top_idx, workspace, workspace_bytes, stream, side_stream);
}

namespace {

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The expert GEMMs' constraints of the fp8-weight and W8A8 modes, checked by the entries so that nothing is launched for a
// block that would fail half-way
bool fp8_experts_ok(int32_t d, int32_t I, const void* fc1_w, const void* fc2_w, const float* fc1_scale, const float* fc2_scale) {
  if (!fc1_scale || !fc2_scale) return false;
  if (d <= 0 || I <= 0 || d % 64 != 0 || I % 64 != 0) return false;
  return al16(fc1_w) && al16(fc2_w) && al16(fc1_scale) && al16(fc2_scale);
}

// ... and of the quantiser in front of them
bool w8a8_experts_ok(int32_t d, int32_t I, const void* fc1_w_nk, const void* fc2_w_nk, const float* fc1_scale,
                     const float* fc2_scale) {
  if (!fc1_scale || !fc2_scale) return false;
  if (d <= 0 || I <= 0 || d % 128 != 0 || I % 128 != 0 || d > 4096 || I > 4096 || I > 2 * d) return false;
  return al16(fc1_w_nk) && al16(fc2_w_nk) && al16(fc1_scale) && al16(fc2_scale);
}

}  // namespace

extern "C" int aria_moe_block_fwd_fp8(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w,
                                      const float* fc1_scale, const float* fc2_scale, const void* gate_w, const void* up_w,
                                      const void* down_w, void* out, int64_t T, int32_t d, int32_t E, int32_t k, int32_t I,
                                      int32_t I_shared, const int32_t* forced_top_idx, void* workspace, int64_t workspace_bytes,
                                      aria_stream_t stream, aria_stream_t side_stream) {
  if (!fp8_experts_ok(d, I, fc1_w, fc2_w, fc1_scale, fc2_scale)) return ARIA_ERR_BAD_ARG;
  return moe_block_run(x, w_router, fc1_w, fc2_w, fc1_scale, fc2_scale, false, gate_w, up_w, down_w, out, T, d, E, k, I, I_shared,
                       forced_top_idx, workspace, workspace_bytes, stream, side_stream);
}

extern "C" int aria_moe_block_fwd_w8a8(const void* x, const void* w_router, const void* fc1_w_nk, const void* fc2_w_nk,
                                       const float* fc1_scale, const float* fc2_scale, const void* gate_w, const void* up_w,
                                       const void* down_w, void* out, int64_t T, int32_t d, int32_t E, int32_t k, int32_t I,
                                       int32_t I_shared, const int32_t* forced_top_idx, void* workspace, int64_t workspace_bytes,
                                       aria_stream_t stream, aria_stream_t side_stream) {
  if (!w8a8_experts_ok(d, I, fc1_w_nk, fc2_w_nk, fc1_scale, fc2_scale)) return ARIA_ERR_BAD_ARG;
  return moe_block_run(x, w_router, fc1_w_nk, fc2_w_nk, fc1_scale, fc2_scale, true, gate_w, up_w, down_w, out, T, d, E, k, I,
                       I_shared, forced_top_idx, workspace, workspace_bytes, stream, side_stream);
}

extern "C" int64_t aria_moe_block_fwd_shared_fp8_workspace_bytes(int64_t T, int32_t d, int32_t E, int32_t k, int32_t I,
                                                                 int32_t I_shared) {
  if (T <= 0 || d <= 0 || E <= 0 || k <= 0 || I <= 0 || I_shared <= 0) return ARIA_ERR_BAD_ARG;
  return carve(T, d, E, k, I, I_shared, true).total;
}

extern "C" int aria_moe_block_fwd_shared_fp8(const void* x, const void* w_router, const void* fc1_w, const void* fc2_w,
                                             const float* fc1_scale, const float* fc2_scale, int32_t expert_mode,
                                             const void* gate_w, const void* up_w, const void* down_w, const float* gate_scale,
                                             const float* up_scale, const float* down_scale, void* out, int64_t T, int32_t d,
                                             int32_t E, int32_t k, int32_t I, int32_t I_shared, const int32_t* forced_top_idx,
                                             void* workspace, int64_t workspace_bytes, aria_stream_t stream,
                                             aria_stream_t side_stream) {
  // the shared GEMMs' and quantisers' constraints (aria_gemm_w8a8: K % 128, N % 64; the row quantiser: d <= 4096)
  if (!gate_w || !up_w || !down_w || !gate_scale || !up_scale || !down_scale) return ARIA_ERR_BAD_ARG;
  if (I_shared <= 0 || d <= 0 || d % 128 != 0 || I_shared % 128 != 0 || d > 4096 || I_shared > 4096) return ARIA_ERR_BAD_ARG;
  if (!al16(gate_w) || !al16(up_w) || !al16(down_w) || !al16(gate_scale) || !al16(up_scale) || !al16(down_scale))
    return ARIA_ERR_BAD_ARG;
  if (T >= (int64_t(1) << 31)) return ARIA_ERR_BAD_ARG;
  const SharedScales ss{gate_scale, up_scale, down_scale};
  switch (expert_mode) {
    case ARIA_MOE_EXPERTS_BF16:
      if (fc1_scale || fc2_scale) return ARIA_ERR_BAD_ARG;
      return moe_block_run(x, w_router, fc1_w, fc2_w, nullptr, nullptr, false, gate_w, up_w, down_w, out, T, d, E, k, I, I_shared,
                           forced_top_idx, workspace, workspace_bytes, stream, side_stream, ss);
    case ARIA_MOE_EXPERTS_FP8:
      if (!fp8_experts_ok(d, I, fc1_w, fc2_w, fc1_scale, fc2_scale)) return ARIA_ERR_BAD_ARG;
      return moe_block_run(x, w_router, fc1_w, fc2_w, fc1_scale, fc2_scale, false, gate_w, up_w, down_w, out, T, d, E, k, I,
                           I_shared, forced_top_idx, workspace, workspace_bytes, stream, side_stream, ss);
    case ARIA_MOE_EXPERTS_W8A8:
      if (!w8a8_experts_ok(d, I, fc1_w, fc2_w, fc1_scale, fc2_scale)) return ARIA_ERR_BAD_ARG;
      return moe_block_run(x, w_router, fc1_w, fc2_w, fc1_scale, fc2_scale, true, gate_w, up_w, down_w, out, T, d, E, k, I,
                           I_shared, forced_top_idx, workspace, workspace_bytes, stream, side_stream, ss);
    default:
      return ARIA_ERR_BAD_ARG;
  }
}
