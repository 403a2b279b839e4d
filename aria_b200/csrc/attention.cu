// Attention for sm_90a.
//
// aria_attention_fwd: flash-style forward with both contractions on wgmma tensor cores:
//     S = Q K^T   (A = Q tile, B = K tile, both K-major SW128 in shared memory, S accumulates in registers)
//     O += P V    (A = P, bf16, straight from the registers that held S; B = V tile consumed MN-major — V is [keys, d] with d
//                  contiguous, exactly the HF cache layout — O accumulates in registers)
//   warpgroup 0: TMA producer (Q once, K/V through a two-stage ring); warpgroups 1-2: 64 query rows each, fp32 online
//   softmax on the fragments (four threads share a row: max / sum over two shuffles) and the final normalise + store.
//   One CTA per (batch, head, 128 queries); causal launches visit the heaviest query tiles first.
// Replaces flash_attn_func / SDPA behind LLAMA_ATTENTION_CLASSES (aria/model/moe_lm.py:594) and the
// Idefics2 / nn.MultiheadAttention attention of the ViT + projector (vision_encoder.py:120, projector.py:93), whose
// 72-wide heads live in 128-wide rows: QK contracts HD = 80 columns (5 k-steps), PV produces all 128 and only out_hd are stored.
// Scores and softmax statistics stay fp32.  The running row max is raised lazily, only when it grows by more than 2^8: P then
// lies in [0, 256] and is rounded to bf16 at that scale, which measured closer to transformers' eager attention (the reference
// of the ViT path) than rounding P relative to the exact running max, and it skips most rescales of O.
//
// aria_attention_decode: single-query attention against the KV cache; HBM-bound, CUDA cores, split-KV.
#include "common.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int AT_BM = 128;   // queries per CTA
constexpr int AT_BN = 128;   // keys per step
constexpr int AT_D = 128;    // head dim (row width of q / k / v)
constexpr int AT_TILE = AT_BM * AT_D * 2;  // 32 KB
constexpr int AT_HALF = AT_TILE / 2;       // one SW128 column chunk: [128 rows][64 bf16]
constexpr int AT_STAGES = 2;
constexpr int AT_THREADS = 384;            // producer warpgroup + two consumer warpgroups
constexpr int AT_SMEM = 1024 + AT_TILE /*Q*/ + AT_STAGES * 2 * AT_TILE /*K, V*/ + 256;

struct AttnParams {
  int B, H, Tq, Tk;
  int out_hd;
  float scale_log2;
  const uint8_t* key_mask;  // [B, Tk] 1 = masked out
  __nv_bfloat16* out;       // [B, Tq, H*out_hd]
  float* lse;               // [B, H, Tq] natural-log logsumexp of scale * q.k (LSE instantiations only)
  int n_q_tiles;
};

// HD = head dim contracted by QK^T (80 for the 72-wide ViT heads, 128 for the LM); LSE: also store the row logsumexp
// (what the backward needs to recompute P)
template <int HD, bool CAUSAL, bool LSE>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                            // [2 chunks][128 rows][64]
  uint8_t* sK = sQ + AT_TILE;                    // [STAGES][32 KB]
  uint8_t* sV = sK + AT_STAGES * AT_TILE;        // [STAGES][32 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + AT_STAGES * AT_TILE);
  uint64_t* q_full = bars;                       // [1]
  uint64_t* k_full = bars + 1;                   // [STAGES]
  uint64_t* v_full = k_full + AT_STAGES;         // [STAGES]
  uint64_t* kv_empty = v_full + AT_STAGES;       // [STAGES], one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int BH = p.B * p.H;
  const int bh = blockIdx.x % BH;
  const int q_tile = p.n_q_tiles - 1 - blockIdx.x / BH;  // heaviest (latest rows) first
  const int b = bh / p.H, h = bh % p.H;
  const int q0 = q_tile * AT_BM;
  const int pos_off = p.Tk - p.Tq;
  int n_kv = (p.Tk + AT_BN - 1) / AT_BN;
  if (CAUSAL) n_kv = min(n_kv, (pos_off + min(q0 + AT_BM, p.Tq) - 1) / AT_BN + 1);

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < AT_STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);
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
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % AT_STAGES;
        mbar_wait(&kv_empty[s], ((j / AT_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&k_full[s], AT_TILE);
        tma_load_4d(sK + s * AT_TILE, &tmK, &k_full[s], 0, j * AT_BN, h, b);
        tma_load_4d(sK + s * AT_TILE + AT_HALF, &tmK, &k_full[s], 64, j * AT_BN, h, b);
        mbar_arrive_expect_tx(&v_full[s], AT_TILE);
        tma_load_4d(sV + s * AT_TILE, &tmV, &v_full[s], 0, j * AT_BN, h, b);
        tma_load_4d(sV + s * AT_TILE + AT_HALF, &tmV, &v_full[s], 64, j * AT_BN, h, b);
      }
    }
    return;
  }

  // =========================== consumer warpgroup cw: query rows [q0 + 64 cw, +64) ===========================
  setmaxnreg_inc<240>();
  const int cw = wg - 1;
  const int r_lo = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's two rows: r_lo and r_lo + 8
  const int qpos_lo = pos_off + r_lo, qpos_hi = qpos_lo + 8;
  const int kq = 2 * (lane & 3);                                  // key / column offset of this thread in an 8-wide block
  const uint8_t* km = p.key_mask ? p.key_mask + static_cast<int64_t>(b) * p.Tk : nullptr;
  const uint32_t sQa = smem_u32(sQ) + cw * 64 * 128, sKa = smem_u32(sK), sVa = smem_u32(sV);
  // K-major k-step kk (16 columns of the head): chunk kk / 4, +32 B per step inside the chunk
  auto kmaj_off = [](int kk) { return static_cast<uint32_t>((kk >> 2) * AT_HALF + (kk & 3) * 32); };
  // V MN-major: LBO = 16 KB between the two 64-column chunks, SBO = 1024 (8 keys), +2048 B per 16 keys
  const uint64_t dV0 = make_smem_desc(sVa, AT_HALF, 1024);

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_kv; ++j) {
    const int s = j % AT_STAGES;
    const uint32_t ph = (j / AT_STAGES) & 1;
    float sc[64];
    mbar_wait(&k_full[s], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_m64n128_ss<0, 0>(sc, make_smem_desc(sQa + kmaj_off(kk), 16, 1024),
                             make_smem_desc(sKa + s * AT_TILE + kmaj_off(kk), 16, 1024), kk ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sc);

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
    if (__any_sync(0xffffffffu, up_lo || up_hi)) {
      const float f_lo = !up_lo ? 1.f : (m_lo == -INFINITY ? 0.f : fast_ex2(m_lo - mc_lo));
      const float f_hi = !up_hi ? 1.f : (m_hi == -INFINITY ? 0.f : fast_ex2(m_hi - mc_hi));
      if (up_lo) m_lo = mc_lo;
      if (up_hi) m_hi = mc_hi;
      l_lo *= f_lo;
      l_hi *= f_hi;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        o[4 * jj] *= f_lo;
        o[4 * jj + 1] *= f_lo;
        o[4 * jj + 2] *= f_hi;
        o[4 * jj + 3] *= f_hi;
      }
    }
    const float neg_lo = (m_lo == -INFINITY) ? 0.f : -m_lo, neg_hi = (m_hi == -INFINITY) ? 0.f : -m_hi;
    // P as the A operand of the PV product: k-step kk (keys 16 kk..) = {row lo keys +0/+1, row hi, row lo keys +8/+9, row hi}
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const bool hi = r & 1;
        const float x0 = fast_ex2(fmaf(sc[8 * kk + 2 * r], p.scale_log2, hi ? neg_hi : neg_lo));
        const float x1 = fast_ex2(fmaf(sc[8 * kk + 2 * r + 1], p.scale_log2, hi ? neg_hi : neg_lo));
        if (hi) l_hi += x0 + x1; else l_lo += x0 + x1;
        pa[kk][r] = pack_bf16(x0, x1);
      }
    }
    mbar_wait(&v_full[s], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_m64n128_rs<1>(o, pa[kk], dV0 + ((s * AT_TILE + kk * 2048) >> 4));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
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
    if (q >= p.Tq) continue;
    const float l = hrow ? l_hi : l_lo;
    const float inv_l = l > 0.f ? 1.0f / l : 0.f;
    __nv_bfloat16* orow = p.out + (static_cast<int64_t>(b) * p.Tq + q) * ld + h * p.out_hd;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      if (8 * jj < p.out_hd)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + kq) = pack_bf16(o[4 * jj + 2 * hrow] * inv_l, o[4 * jj + 2 * hrow + 1] * inv_l);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Decode: one query per (b,h); block = 4 warps over a contiguous chunk of keys; each lane owns 4 dims.
// Partial (m, l, acc[128]) per (b,h,split) -> workspace; a second kernel merges the splits.
constexpr int DEC_SPLIT_KEYS = 256;

__global__ void __launch_bounds__(128) attn_decode_partial(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kc,
                                                           const __nv_bfloat16* __restrict__ vc, const uint8_t* __restrict__ key_mask,
                                                           float* __restrict__ ws, int H, int Tk,
                                                           int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b,
                                                           int64_t kv_stride_h, float scale_log2, int splits) {
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / H, h = bh % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k_begin = split * DEC_SPLIT_KEYS, k_end = min(Tk, k_begin + DEC_SPLIT_KEYS);
  const __nv_bfloat16* kbase = kc + b * kv_stride_b + h * kv_stride_h;
  const __nv_bfloat16* vbase = vc + b * kv_stride_b + h * kv_stride_h;
  const uint8_t* km = key_mask ? key_mask + static_cast<int64_t>(b) * Tk : nullptr;
  const uint2 qv = *reinterpret_cast<const uint2*>(q + b * q_stride_b + h * q_stride_h + lane * 4);
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

__global__ void __launch_bounds__(128) attn_decode_merge(const float* __restrict__ ws, __nv_bfloat16* __restrict__ out, int splits) {
  const int bh = blockIdx.x, d = threadIdx.x;
  const float* base = ws + static_cast<int64_t>(bh) * splits * (AT_D + 2);
  float M = -INFINITY;
  for (int s = 0; s < splits; ++s) M = fmaxf(M, base[s * (AT_D + 2) + AT_D]);
  float L = 0.f, A = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float ms = base[s * (AT_D + 2) + AT_D];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
    L += base[s * (AT_D + 2) + AT_D + 1] * f;
    A += base[s * (AT_D + 2) + d] * f;
  }
  out[static_cast<int64_t>(bh) * AT_D + d] = __float2bfloat16_rn(L > 0.f ? A / L : 0.f);
}

static int make_tmap_heads(CUtensorMap* tm, const void* ptr, int T, int H, int B, int64_t stride_b, int64_t stride_h) {
  uint64_t dims[4] = {static_cast<uint64_t>(AT_D), static_cast<uint64_t>(T), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
  uint64_t str[3] = {static_cast<uint64_t>(AT_D) * 2, static_cast<uint64_t>(stride_h) * 2, static_cast<uint64_t>(stride_b) * 2};
  uint32_t box[4] = {64, 128, 1, 1};
  return make_tmap_bf16(tm, ptr, 4, dims, str, box);
}

template <int HD, bool CAUSAL, bool LSE>
static int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const AttnParams& p, int64_t grid,
                       cudaStream_t stream) {
  auto kern = attn_fwd_kernel<HD, CAUSAL, LSE>;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, kern, AT_SMEM) != cudaSuccess) return ARIA_ERR_CUDA;
  kern<<<static_cast<int>(grid), AT_THREADS, AT_SMEM, stream>>>(tmQ, tmK, tmV, p);
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
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_heads(&tmQ, q, Tq, H, B, q_stride_b, q_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmK, k, Tk, H, B, kv_stride_b, kv_stride_h);
  if (rc) return rc;
  rc = make_tmap_heads(&tmV, v, Tk, H, B, kv_stride_b, kv_stride_h);
  if (rc) return rc;
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
  if (lse) {
    if (out_hd <= 80) return causal ? launch_attn<80, true, true>(tmQ, tmK, tmV, p, grid, stream) : launch_attn<80, false, true>(tmQ, tmK, tmV, p, grid, stream);
    return causal ? launch_attn<128, true, true>(tmQ, tmK, tmV, p, grid, stream) : launch_attn<128, false, true>(tmQ, tmK, tmV, p, grid, stream);
  }
  if (out_hd <= 80) return causal ? launch_attn<80, true, false>(tmQ, tmK, tmV, p, grid, stream) : launch_attn<80, false, false>(tmQ, tmK, tmV, p, grid, stream);
  return causal ? launch_attn<128, true, false>(tmQ, tmK, tmV, p, grid, stream) : launch_attn<128, false, false>(tmQ, tmK, tmV, p, grid, stream);
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
  attn_decode_partial<<<grid, 128, 0, stream>>>(static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
                                                static_cast<const __nv_bfloat16*>(v), key_mask, static_cast<float*>(workspace), H, Tk,
                                                q_stride_b, q_stride_h, kv_stride_b, kv_stride_h, scale * 1.4426950408889634f, splits);
  int rc = check_launch("attn_decode_partial");
  if (rc) return rc;
  attn_decode_merge<<<B * H, 128, 0, stream>>>(static_cast<const float*>(workspace), static_cast<__nv_bfloat16*>(out), splits);
  return check_launch("attn_decode_merge");
}
