// Attention backward for sm_90a: the LM's causal attention (head dim 128), FlashAttention-2 style.
//
// aria_attention_bwd runs three kernels:
//   attn_bwd_pre   D = rowsum(dO * O) (fp32), lse * log2 e (+inf for a row that sees no key, so its P is exactly 0), and zeroes
//                  the fp32 dQ accumulator.
//   attn_bwd_kernel one CTA per (batch, head, 128 keys); causal launches visit the heaviest key tiles (the earliest) first.
//                  Two warpgroups, 64 keys each; dK and dV accumulate in registers (fp32) over all query tiles, which with the
//                  score fragments needs ~250 registers a thread: so no producer warpgroup (its 128 threads would cap the
//                  register file at 168 a thread).  One thread issues the TMA loads instead: K and V once, then [64 x 128] Q and
//                  dO tiles through a three-stage ring, two tiles ahead.  Per query tile:
//                      S^T  = K Q^T                          (wgmma, A = K rows K-major, B = Q K-major)
//                      P^T  = exp2(S^T * scale * log2 e - lse * log2 e), masked as in the forward
//                      dV  += P^T dO                         (A = P^T from registers, B = dO consumed MN-major)
//                      dP^T = V dO^T                         (A = V rows K-major, B = dO K-major)
//                      dS^T = P^T o (dP^T - D)
//                      dK  += dS^T Q                         (A = dS^T from registers, B = Q consumed MN-major)
//                      dQ  += dS K                           (A = dS^T in shared memory read MN-major, B = K consumed MN-major)
//                  the two warpgroups split dQ by head-dim halves (64 columns each over all 128 keys) and add it to the fp32
//                  accumulator with float2 atomicAdd.  dK (times scale) and dV are stored once, as bf16.
//   attn_bwd_post  dQ = bf16(scale * accumulator).
// dK and dV are each produced by exactly one CTA in a fixed order: bit-reproducible.  dQ sums the key tiles' contributions with
// fp32 atomics, so its low bits depend on their arrival order.
//
// aria_attention_bwd_varlen: the same three kernels over n_seg causal segments packed along one row axis (B = 1), segment s =
// rows [cu[s], cu[s+1]).  attn_bwd_varlen_tiles first lists the segments' 128-key tiles, each aligned at its segment's start,
// heaviest (most query rows) first; attn_bwd_kernel<true, true> takes one tile per CTA and walks 64-row query steps from the
// tile's first row to the segment's end.  Query rows at or past the segment's end get P = 0 (and so add exact zeros to dQ);
// keys past it are masked by causality for the segment's own queries, and their dK / dV rows are not stored.  Per segment the
// tiles, the query steps and their order are those of aria_attention_bwd on the segment alone, so dK and dV are bit-identical
// to it.  The statistics and the dQ accumulator carry one extra 64-row step past N (lse2 = +inf), so a step that starts at an
// unaligned row never leaves them.
#include "common.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int AB_BN = 128;                  // keys per CTA (64 per consumer warpgroup)
constexpr int AB_BM = 64;                   // queries per step
constexpr int AB_D = 128;                   // head dim
constexpr int AB_KV = AB_BN * AB_D * 2;     // 32 KB: K or V tile = two SW128 column chunks [128 rows][64]
constexpr int AB_KV_HALF = AB_KV / 2;
constexpr int AB_QT = AB_BM * AB_D * 2;     // 16 KB: Q or dO tile = two chunks [64 rows][64]
constexpr int AB_QT_HALF = AB_QT / 2;
constexpr int AB_DS = AB_BN * AB_BM * 2;    // 16 KB: dS^T [128 keys][64 queries], one SW128 chunk
constexpr int AB_STAGES = 3;
constexpr int AB_THREADS = 256;
constexpr int AB_SMEM = 1024 + 2 * AB_KV + AB_STAGES * 2 * AB_QT + 2 * AB_DS + 256;

// workspace: dq_acc [B*H][Tq_pad][128] fp32, then lse2 and delta [B*H][Tq_pad] fp32 (query rows padded to the 64-row step, so
// the main kernel reads statistics and adds dQ without bounds checks: pad rows carry lse2 = +inf, i.e. P = 0)
static int64_t bwd_tq_pad(int32_t Tq) { return (static_cast<int64_t>(Tq) + AB_BM - 1) / AB_BM * AB_BM; }
// varlen: query steps start at any row, so one more step of padding; and at most ceil(N / 128) + n_seg key tiles
static int64_t bwd_varlen_pad(int32_t N) { return bwd_tq_pad(N) + AB_BM; }
static int64_t bwd_varlen_slots(int32_t n_seg, int32_t N) { return (static_cast<int64_t>(N) + AB_BN - 1) / AB_BN + n_seg; }

struct AttnBwdParams {
  int B, H, Tq, Tk, Tq_pad;
  float scale, scale_log2;
  const uint8_t* key_mask;  // [B, Tk] 1 = masked out
  const float* lse2;        // [B*H][Tq_pad]
  const float* delta;       // [B*H][Tq_pad]
  float* dq_acc;            // [B*H][Tq_pad][128]
  __nv_bfloat16* dk;        // head-major, kv strides
  __nv_bfloat16* dv;
  int64_t kv_stride_b, kv_stride_h;
  const int2* tiles;        // varlen: [slots] {first key row, segment end} per key tile, heaviest first; {-1, 0} = idle slot
};

// Varlen key-tile list (one block): tile t of segment s is {cu[s] + 128 t, cu[s+1]}; a counting sort on the number of 64-row
// query steps it walks puts the heaviest first (as the batched launch's tile order does), then the unused slots are idled.
// Boundaries are clamped to [0, N] and at most `slots` tiles are listed, so malformed boundaries (not nondecreasing from 0 to
// N) give wrong gradients but never a read or write outside q / k / v, dq / dk / dv or the workspace.
constexpr int AB_WEIGHTS = 1024;  // sort classes: query steps, capped (longer tiles are all "heaviest")
__global__ void __launch_bounds__(1024) attn_bwd_varlen_tiles(const int32_t* __restrict__ cu, int n_seg, int N, int slots,
                                                                int2* __restrict__ tiles) {
  __shared__ int slot[AB_WEIGHTS];
  __shared__ int total;
  auto weight = [](int rows) { return min((rows + AB_BM - 1) / AB_BM, AB_WEIGHTS - 1); };
  for (int w = threadIdx.x; w < AB_WEIGHTS; w += blockDim.x) slot[w] = 0;
  __syncthreads();
  auto start = [&](int s) { return min(max(cu[s], 0), N); };
  auto end = [&](int s) { return min(max(cu[s + 1], 0), N); };
  for (int s = threadIdx.x; s < n_seg; s += blockDim.x)
    for (int k0 = start(s), e = end(s); k0 < e; k0 += AB_BN) atomicAdd(&slot[weight(e - k0)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {  // first slot of each class, heaviest class first
    int run = 0;
    for (int w = AB_WEIGHTS - 1; w >= 0; --w) {
      const int n = slot[w];
      slot[w] = run;
      run += n;
    }
    total = min(run, slots);
  }
  __syncthreads();
  for (int s = threadIdx.x; s < n_seg; s += blockDim.x)
    for (int k0 = start(s), e = end(s); k0 < e; k0 += AB_BN) {
      const int i = atomicAdd(&slot[weight(e - k0)], 1);
      if (i < slots) tiles[i] = make_int2(k0, e);
    }
  for (int i = total + threadIdx.x; i < slots; i += blockDim.x) tiles[i] = make_int2(-1, 0);
}

// one warp per (b, h, padded query row)
__global__ void __launch_bounds__(256) attn_bwd_pre(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                                                    const float* __restrict__ lse, float* __restrict__ dq_acc, float* __restrict__ lse2,
                                                    float* __restrict__ delta, int H, int Tq, int Tq_pad, int64_t rows) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int64_t bh = row / Tq_pad;
  const int q = static_cast<int>(row % Tq_pad);
  *reinterpret_cast<float4*>(dq_acc + row * AB_D + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
  if (q >= Tq) {
    if (lane == 0) {
      lse2[row] = INFINITY;
      delta[row] = 0.f;
    }
    return;
  }
  const int64_t b = bh / H, h = bh % H;
  const int64_t tok = ((b * Tq + q) * H + h) * AB_D + lane * 4;
  const uint2 o = *reinterpret_cast<const uint2*>(out + tok);
  const uint2 g = *reinterpret_cast<const uint2*>(dout + tok);
  float d = bf16_lo(o.x) * bf16_lo(g.x) + bf16_hi(o.x) * bf16_hi(g.x) + bf16_lo(o.y) * bf16_lo(g.y) + bf16_hi(o.y) * bf16_hi(g.y);
#pragma unroll
  for (int s = 16; s; s >>= 1) d += __shfl_xor_sync(0xffffffffu, d, s);
  if (lane == 0) {
    const float l = lse[bh * Tq + q];
    lse2[row] = l == -INFINITY ? INFINITY : l * 1.4426950408889634f;
    delta[row] = d;
  }
}

// VARLEN (causal, B = 1): the CTA's key tile and its segment's end come from p.tiles; see the header
template <bool CAUSAL, bool VARLEN>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, const AttnBwdParams p) {
  static_assert(!VARLEN || CAUSAL, "packed segments are causal");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;                             // [2 chunks][128 keys][64]
  uint8_t* sV = sK + AB_KV;
  uint8_t* sQ = sV + AB_KV;                       // [STAGES][2 chunks][64 queries][64]
  uint8_t* sdO = sQ + AB_STAGES * AB_QT;
  uint8_t* sdS = sdO + AB_STAGES * AB_QT;         // [2 buffers][128 keys][64 queries]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sdS + 2 * AB_DS);
  uint64_t* kv_full = bars;                       // [1]
  uint64_t* qd_full = bars + 1;                   // [STAGES]: Q and dO tiles

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int BH = p.B * p.H;
  const int bh = blockIdx.x % BH;
  const int k_tile = blockIdx.x / BH;             // causal: the earliest keys are seen by the most queries
  const int b = bh / p.H, h = bh % p.H;
  int k0 = k_tile * AB_BN;
  const int pos_off = p.Tk - p.Tq;
  int n_m = (p.Tq + AB_BM - 1) / AB_BM;
  int m_begin = CAUSAL ? max(0, k0 - pos_off) / AB_BM : 0;  // earlier query tiles see none of these keys
  int m_base = 0;                                 // row of query step 0 (varlen: the key tile's first row)
  int seg_end = p.Tk;                             // keys and query rows at or past it are dead
  if constexpr (VARLEN) {
    const int2 t = p.tiles[k_tile];
    if (t.x < 0) return;                          // idle slot: the grid is an upper bound on the tile count
    k0 = m_base = t.x;
    seg_end = t.y;
    m_begin = 0;
    n_m = (seg_end - k0 + AB_BM - 1) / AB_BM;
  }

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    prefetch_tmap(&tmdO);
    mbar_init(kv_full, 1);
    for (int i = 0; i < AB_STAGES; ++i) mbar_init(&qd_full[i], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // Q and dO tiles of query tile i into ring stage s
  auto load_qd = [&](int i, int s) {
    mbar_arrive_expect_tx(&qd_full[s], 2 * AB_QT);
    const int m0 = m_base + i * AB_BM;
    tma_load_4d(sQ + s * AB_QT, &tmQ, &qd_full[s], 0, m0, h, b);
    tma_load_4d(sQ + s * AB_QT + AB_QT_HALF, &tmQ, &qd_full[s], 64, m0, h, b);
    tma_load_3d(sdO + s * AB_QT, &tmdO, &qd_full[s], h * AB_D, m0, b);
    tma_load_3d(sdO + s * AB_QT + AB_QT_HALF, &tmdO, &qd_full[s], h * AB_D + 64, m0, b);
  };
  const bool loader = threadIdx.x == 0;
  if (loader) {
    mbar_arrive_expect_tx(kv_full, 2 * AB_KV);
    tma_load_4d(sK, &tmK, kv_full, 0, k0, h, b);
    tma_load_4d(sK + AB_KV_HALF, &tmK, kv_full, 64, k0, h, b);
    tma_load_4d(sV, &tmV, kv_full, 0, k0, h, b);
    tma_load_4d(sV + AB_KV_HALF, &tmV, kv_full, 64, k0, h, b);
    for (int i = m_begin; i < min(n_m, m_begin + AB_STAGES - 1); ++i) load_qd(i, i - m_begin);
  }

  // =========================== warpgroup cw: keys [k0 + 64 cw, +64) ===========================
  const int cw = wg;
  const int kr = (warp & 3) * 16 + (lane >> 2);   // this thread's fragment rows: kr and kr + 8
  const int key_lo = k0 + cw * 64 + kr, key_hi = key_lo + 8;
  const int kq = 2 * (lane & 3);                  // column offset of this thread in an 8-wide block
  const uint8_t* km = p.key_mask ? p.key_mask + static_cast<int64_t>(b) * p.Tk : nullptr;
  const bool dead_lo = key_lo >= seg_end || (km && km[key_lo]);
  const bool dead_hi = key_hi >= seg_end || (km && km[key_hi]);
  const uint32_t sKa = smem_u32(sK), sVa = smem_u32(sV), sQa = smem_u32(sQ), sdOa = smem_u32(sdO), sdSa = smem_u32(sdS);
  // K-major k-step kk (16 head dims): chunk kk / 4, +32 B per step inside the chunk
  auto kv_kmaj = [](int kk) { return static_cast<uint32_t>((kk >> 2) * AB_KV_HALF + (kk & 3) * 32); };
  auto qt_kmaj = [](int kk) { return static_cast<uint32_t>((kk >> 2) * AB_QT_HALF + (kk & 3) * 32); };
  const float* lse2 = p.lse2 + static_cast<int64_t>(bh) * p.Tq_pad;
  const float* delta = p.delta + static_cast<int64_t>(bh) * p.Tq_pad;

  float dk[64], dv[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    dk[i] = 0.f;
    dv[i] = 0.f;
  }
  mbar_wait(kv_full, 0);

  for (int i = m_begin; i < n_m; ++i) {
    const int it = i - m_begin, s = it % AB_STAGES;
    const int m0 = m_base + i * AB_BM;
    const uint32_t sQs = sQa + s * AB_QT, sdOs = sdOa + s * AB_QT;
    float st[32], dp[32];
    mbar_wait(&qd_full[s], (it / AB_STAGES) & 1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_D / 16; ++kk)
      wgmma_m64n64_ss<0, 0>(st, make_smem_desc(sKa + cw * 64 * 128 + kv_kmaj(kk), 16, 1024), make_smem_desc(sQs + qt_kmaj(kk), 16, 1024),
                            kk ? 1u : 0u);
    wgmma_commit();
#pragma unroll
    for (int kk = 0; kk < AB_D / 16; ++kk)
      wgmma_m64n64_ss<0, 0>(dp, make_smem_desc(sVa + cw * 64 * 128 + kv_kmaj(kk), 16, 1024), make_smem_desc(sdOs + qt_kmaj(kk), 16, 1024),
                            kk ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    fence_regs(st);

    // P^T: row = key, column = query m0 + 8 jj + kq + e
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      // varlen steps start at any row: two 4-byte loads where the pair may be 8-byte misaligned
      const float2 l2 = VARLEN ? make_float2(lse2[m0 + 8 * jj + kq], lse2[m0 + 8 * jj + kq + 1])
                               : *reinterpret_cast<const float2*>(lse2 + m0 + 8 * jj + kq);
      st[4 * jj] = fast_ex2(fmaf(st[4 * jj], p.scale_log2, -l2.x));
      st[4 * jj + 1] = fast_ex2(fmaf(st[4 * jj + 1], p.scale_log2, -l2.y));
      st[4 * jj + 2] = fast_ex2(fmaf(st[4 * jj + 2], p.scale_log2, -l2.x));
      st[4 * jj + 3] = fast_ex2(fmaf(st[4 * jj + 3], p.scale_log2, -l2.y));
    }
    const bool need_mask = km != nullptr || k0 + AB_BN > seg_end || (CAUSAL && k0 + cw * 64 + 63 > pos_off + m0) ||
                           (VARLEN && m0 + AB_BM > seg_end);
    if (need_mask) {  // diagonal / key tail / padded keys / (varlen) query rows past the segment
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qpos = pos_off + m0 + 8 * jj + kq + e;
          const bool qdead = VARLEN && qpos >= seg_end;
          if (dead_lo || qdead || (CAUSAL && key_lo > qpos)) st[4 * jj + e] = 0.f;
          if (dead_hi || qdead || (CAUSAL && key_hi > qpos)) st[4 * jj + 2 + e] = 0.f;
        }
      }
    }
    // A-operand fragments, k-step kk (queries 16 kk..) = {row lo +0/+1, row hi, row lo +8/+9, row hi}
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_bf16(st[8 * kk + 2 * r], st[8 * kk + 2 * r + 1]);
    wgmma_fence();
    // dO MN-major: LBO = 8 KB between the two 64-column chunks, SBO = 1024 (8 queries), +2048 B per 16 queries
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n128_rs<1>(dv, pa[kk], make_smem_desc(sdOs + kk * 2048, AB_QT_HALF, 1024));
    wgmma_commit();
    wgmma_wait<1>();
    fence_regs(dp);

#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 dd = VARLEN ? make_float2(delta[m0 + 8 * jj + kq], delta[m0 + 8 * jj + kq + 1])
                               : *reinterpret_cast<const float2*>(delta + m0 + 8 * jj + kq);
      dp[4 * jj] = st[4 * jj] * (dp[4 * jj] - dd.x);
      dp[4 * jj + 1] = st[4 * jj + 1] * (dp[4 * jj + 1] - dd.y);
      dp[4 * jj + 2] = st[4 * jj + 2] * (dp[4 * jj + 2] - dd.x);
      dp[4 * jj + 3] = st[4 * jj + 3] * (dp[4 * jj + 3] - dd.y);
    }
    uint32_t ds[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) ds[kk][r] = pack_bf16(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n128_rs<1>(dk, ds[kk], make_smem_desc(sQs + kk * 2048, AB_QT_HALF, 1024));
    wgmma_commit();

    // dS^T -> shared memory (SW128 rows of 64 queries) for dQ; double-buffered, so one barrier per step suffices
    uint8_t* buf = sdS + (it & 1) * AB_DS;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = cw * 64 + kr + (r & 1) * 8, jj = 2 * kk + (r >> 1);
        *reinterpret_cast<uint32_t*>(buf + row * 128 + ((jj ^ (row & 7)) << 4) + kq * 2) = ds[kk][r];
      }
    fence_proxy_async_smem();
    named_bar_sync(1, 256);
    // both warpgroups are past step it - 1, so its ring stage is free: refill it with query tile i + 2
    if (loader && i + AB_STAGES - 1 < n_m) load_qd(i + AB_STAGES - 1, (it + AB_STAGES - 1) % AB_STAGES);
    // dQ[:, 64 cw .. +64] = dS K[:, 64 cw .. +64]: A = dS^T buffer as MN-major [keys][queries], B = K chunk cw as MN-major
    float dq[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_BN / 16; ++kk)
      wgmma_m64n64_ss<1, 1>(dq, make_smem_desc(sdSa + (it & 1) * AB_DS + kk * 2048, AB_DS, 1024),
                            make_smem_desc(sKa + cw * AB_KV_HALF + kk * 2048, AB_KV_HALF, 1024), kk ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dq);
    fence_regs(dk);
    fence_regs(dv);

    // dQ fragment: row = query m0 + kr (+8), column = head dim 64 cw + 8 jj + kq (+1)
    float* dqa = p.dq_acc + (static_cast<int64_t>(bh) * p.Tq_pad + m0 + kr) * AB_D + cw * 64 + kq;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      atomicAdd(reinterpret_cast<float2*>(dqa + 8 * jj), make_float2(dq[4 * jj], dq[4 * jj + 1]));
      atomicAdd(reinterpret_cast<float2*>(dqa + 8 * AB_D + 8 * jj), make_float2(dq[4 * jj + 2], dq[4 * jj + 3]));
    }
  }

  // dK = scale * dS^T Q, dV = P^T dO: rows key_lo / key_hi, columns 8 jj + kq (+1)
  const int64_t base = static_cast<int64_t>(b) * p.kv_stride_b + static_cast<int64_t>(h) * p.kv_stride_h;
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int key = hrow ? key_hi : key_lo;
    if (key >= seg_end) continue;
    __nv_bfloat16* dkr = p.dk + base + static_cast<int64_t>(key) * AB_D;
    __nv_bfloat16* dvr = p.dv + base + static_cast<int64_t>(key) * AB_D;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      *reinterpret_cast<uint32_t*>(dkr + 8 * jj + kq) = pack_bf16(dk[4 * jj + 2 * hrow] * p.scale, dk[4 * jj + 2 * hrow + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(dvr + 8 * jj + kq) = pack_bf16(dv[4 * jj + 2 * hrow], dv[4 * jj + 2 * hrow + 1]);
    }
  }
}

// dq[b, h, q, :] = bf16(scale * dq_acc); one thread per 4 head dims
__global__ void __launch_bounds__(256) attn_bwd_post(const float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dq, int H, int Tq,
                                                     int Tq_pad, int64_t q_stride_b, int64_t q_stride_h, float scale, int64_t n) {
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int d4 = static_cast<int>(t & 31);
  const int64_t row = t >> 5;                       // (b*H + h)*Tq + q
  const int64_t bh = row / Tq;
  const int q = static_cast<int>(row % Tq);
  const int64_t b = bh / H, h = bh % H;
  const float4 a = *reinterpret_cast<const float4*>(dq_acc + (bh * Tq_pad + q) * AB_D + d4 * 4);
  uint2 o;
  o.x = pack_bf16(a.x * scale, a.y * scale);
  o.y = pack_bf16(a.z * scale, a.w * scale);
  *reinterpret_cast<uint2*>(dq + b * q_stride_b + h * q_stride_h + static_cast<int64_t>(q) * AB_D + d4 * 4) = o;
}

static int make_tmap_heads_box(CUtensorMap* tm, const void* ptr, int T, int H, int B, int64_t stride_b, int64_t stride_h, uint32_t rows) {
  uint64_t dims[4] = {static_cast<uint64_t>(AB_D), static_cast<uint64_t>(T), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
  uint64_t str[3] = {static_cast<uint64_t>(AB_D) * 2, static_cast<uint64_t>(stride_h) * 2, static_cast<uint64_t>(stride_b) * 2};
  uint32_t box[4] = {64, rows, 1, 1};
  return make_tmap_bf16(tm, ptr, 4, dims, str, box);
}

template <bool CAUSAL, bool VARLEN = false>
static int launch_attn_bwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const CUtensorMap& tmdO,
                           const AttnBwdParams& p, int64_t grid, cudaStream_t stream) {
  auto kern = attn_bwd_kernel<CAUSAL, VARLEN>;
  static bool attr_set[kMaxDevices] = {};
  if (ensure_dynamic_smem(attr_set, kern, AB_SMEM) != cudaSuccess) return ARIA_ERR_CUDA;
  kern<<<static_cast<int>(grid), AB_THREADS, AB_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, p);
  return check_launch("attn_bwd_kernel");
}

}  // namespace aria

using namespace aria;

extern "C" int64_t aria_attention_bwd_workspace_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk, int32_t causal) {
  (void)Tk; (void)causal;
  if (B <= 0 || H <= 0 || Tq <= 0) return 0;
  return static_cast<int64_t>(B) * H * bwd_tq_pad(Tq) * (AB_D + 2) * static_cast<int64_t>(sizeof(float));
}

extern "C" int aria_attention_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
                                  void* dq, void* dk, void* dv, const uint8_t* key_mask, int32_t B, int32_t H, int32_t Tq, int32_t Tk,
                                  int64_t q_stride_b, int64_t q_stride_h, int64_t kv_stride_b, int64_t kv_stride_h, float scale,
                                  int32_t causal, void* workspace, int64_t workspace_bytes, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k && v && out && dout && lse && dq && dk && dv && workspace);
  ARIA_CHECK_ARG(B > 0 && H > 0 && Tq > 0 && Tk > 0 && Tk >= (causal ? Tq : 0));
  ARIA_CHECK_ARG(q_stride_b % 8 == 0 && q_stride_h % 8 == 0 && kv_stride_b % 8 == 0 && kv_stride_h % 8 == 0);
  ARIA_CHECK_ARG(q_stride_b >= 0 && q_stride_h >= 0 && kv_stride_b >= 0 && kv_stride_h >= 0);
  auto aligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  ARIA_CHECK_ARG(aligned(q) && aligned(k) && aligned(v) && aligned(out) && aligned(dout) && aligned(dq) && aligned(dk) && aligned(dv) &&
                 aligned(workspace) && (reinterpret_cast<uintptr_t>(lse) & 3) == 0);
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_bwd_workspace_bytes(B, H, Tq, Tk, causal));
  const int64_t Tq_pad = bwd_tq_pad(Tq);
  const int64_t n_k_tiles = (Tk + AB_BN - 1) / AB_BN;
  const int64_t grid = static_cast<int64_t>(B) * H * n_k_tiles;
  const int64_t pre_rows = static_cast<int64_t>(B) * H * Tq_pad;
  const int64_t post_n = static_cast<int64_t>(B) * H * Tq * 32;
  ARIA_CHECK_ARG(grid < (1ll << 31) && (pre_rows + 7) / 8 < (1ll << 31) && (post_n + 255) / 256 < (1ll << 31));
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * AB_D * 2 * Tq * B < (1ll << 40));

  CUtensorMap tmQ, tmK, tmV, tmdO;
  int rc = make_tmap_heads_box(&tmQ, q, Tq, H, B, q_stride_b, q_stride_h, AB_BM);
  if (rc) return rc;
  rc = make_tmap_heads_box(&tmK, k, Tk, H, B, kv_stride_b, kv_stride_h, AB_BN);
  if (rc) return rc;
  rc = make_tmap_heads_box(&tmV, v, Tk, H, B, kv_stride_b, kv_stride_h, AB_BN);
  if (rc) return rc;
  {  // dO is token-major [B, Tq, H*128]: a head's tile is columns [128 h, +128) of its rows
    uint64_t dims[3] = {static_cast<uint64_t>(H) * AB_D, static_cast<uint64_t>(Tq), static_cast<uint64_t>(B)};
    uint64_t str[2] = {static_cast<uint64_t>(H) * AB_D * 2, static_cast<uint64_t>(H) * AB_D * 2 * Tq};
    uint32_t box[3] = {64, AB_BM, 1};
    rc = make_tmap_bf16(&tmdO, dout, 3, dims, str, box);
    if (rc) return rc;
  }

  float* ws = static_cast<float*>(workspace);
  AttnBwdParams p{};
  p.B = B;
  p.H = H;
  p.Tq = Tq;
  p.Tk = Tk;
  p.Tq_pad = static_cast<int>(Tq_pad);
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.key_mask = key_mask;
  p.dq_acc = ws;
  p.lse2 = ws + pre_rows * AB_D;
  p.delta = p.lse2 + pre_rows;
  p.dk = static_cast<__nv_bfloat16*>(dk);
  p.dv = static_cast<__nv_bfloat16*>(dv);
  p.kv_stride_b = kv_stride_b;
  p.kv_stride_h = kv_stride_h;

  attn_bwd_pre<<<static_cast<int>((pre_rows + 7) / 8), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), lse, ws, ws + pre_rows * AB_D,
      ws + pre_rows * AB_D + pre_rows, H, Tq, static_cast<int>(Tq_pad), pre_rows);
  rc = check_launch("attn_bwd_pre");
  if (rc) return rc;
  rc = causal ? launch_attn_bwd<true>(tmQ, tmK, tmV, tmdO, p, grid, stream) : launch_attn_bwd<false>(tmQ, tmK, tmV, tmdO, p, grid, stream);
  if (rc) return rc;
  attn_bwd_post<<<static_cast<int>((post_n + 255) / 256), 256, 0, stream>>>(ws, static_cast<__nv_bfloat16*>(dq), H, Tq,
                                                                            static_cast<int>(Tq_pad), q_stride_b, q_stride_h, scale, post_n);
  return check_launch("attn_bwd_post");
}

extern "C" int64_t aria_attention_bwd_varlen_workspace_bytes(int32_t n_seg, int32_t H, int32_t N) {
  if (n_seg <= 0 || H <= 0 || N < n_seg) return 0;
  const int64_t slots = (bwd_varlen_slots(n_seg, N) * static_cast<int64_t>(sizeof(int2)) + 15) / 16 * 16;
  return static_cast<int64_t>(H) * bwd_varlen_pad(N) * (AB_D + 2) * static_cast<int64_t>(sizeof(float)) + slots;
}

extern "C" int aria_attention_bwd_varlen(const void* q, const void* k, const void* v, const void* out, const void* dout, const float* lse,
                                         void* dq, void* dk, void* dv, const int32_t* cu_seqlens, int32_t n_seg, int32_t H, int32_t N,
                                         int64_t q_stride_h, int64_t kv_stride_h, float scale, void* workspace, int64_t workspace_bytes,
                                         aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(q && k && v && out && dout && lse && dq && dk && dv && cu_seqlens && workspace);
  ARIA_CHECK_ARG(n_seg > 0 && H > 0 && N >= n_seg);
  ARIA_CHECK_ARG(q_stride_h >= static_cast<int64_t>(N) * AB_D && kv_stride_h >= static_cast<int64_t>(N) * AB_D);
  ARIA_CHECK_ARG(q_stride_h % 8 == 0 && kv_stride_h % 8 == 0);
  auto aligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  ARIA_CHECK_ARG(aligned(q) && aligned(k) && aligned(v) && aligned(out) && aligned(dout) && aligned(dq) && aligned(dk) && aligned(dv) &&
                 aligned(workspace) && (reinterpret_cast<uintptr_t>(lse) & 3) == 0 && (reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0);
  ARIA_CHECK_ARG(workspace_bytes >= aria_attention_bwd_varlen_workspace_bytes(n_seg, H, N));
  const int64_t pad = bwd_varlen_pad(N);
  const int64_t slots = bwd_varlen_slots(n_seg, N);
  const int64_t grid = static_cast<int64_t>(H) * slots;
  const int64_t pre_rows = static_cast<int64_t>(H) * pad;
  const int64_t post_n = static_cast<int64_t>(H) * N * 32;
  ARIA_CHECK_ARG(grid < (1ll << 31) && (pre_rows + 7) / 8 < (1ll << 31) && (post_n + 255) / 256 < (1ll << 31));
  ARIA_CHECK_ARG(static_cast<int64_t>(H) * AB_D * 2 * N < (1ll << 40));

  // one batch row: its stride is never stepped
  CUtensorMap tmQ, tmK, tmV, tmdO;
  int rc = make_tmap_heads_box(&tmQ, q, N, H, 1, q_stride_h * H, q_stride_h, AB_BM);
  if (rc) return rc;
  rc = make_tmap_heads_box(&tmK, k, N, H, 1, kv_stride_h * H, kv_stride_h, AB_BN);
  if (rc) return rc;
  rc = make_tmap_heads_box(&tmV, v, N, H, 1, kv_stride_h * H, kv_stride_h, AB_BN);
  if (rc) return rc;
  {  // dO is token-major [N, H*128]
    uint64_t dims[3] = {static_cast<uint64_t>(H) * AB_D, static_cast<uint64_t>(N), 1};
    uint64_t str[2] = {static_cast<uint64_t>(H) * AB_D * 2, static_cast<uint64_t>(H) * AB_D * 2 * N};
    uint32_t box[3] = {64, AB_BM, 1};
    rc = make_tmap_bf16(&tmdO, dout, 3, dims, str, box);
    if (rc) return rc;
  }

  float* ws = static_cast<float*>(workspace);
  AttnBwdParams p{};
  p.B = 1;
  p.H = H;
  p.Tq = N;
  p.Tk = N;
  p.Tq_pad = static_cast<int>(pad);
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.dq_acc = ws;
  p.lse2 = ws + pre_rows * AB_D;
  p.delta = p.lse2 + pre_rows;
  p.dk = static_cast<__nv_bfloat16*>(dk);
  p.dv = static_cast<__nv_bfloat16*>(dv);
  p.kv_stride_b = static_cast<int64_t>(H) * kv_stride_h;
  p.kv_stride_h = kv_stride_h;
  int2* tiles = reinterpret_cast<int2*>(ws + pre_rows * (AB_D + 2));
  p.tiles = tiles;

  attn_bwd_varlen_tiles<<<1, 1024, 0, stream>>>(cu_seqlens, n_seg, N, static_cast<int>(slots), tiles);
  rc = check_launch("attn_bwd_varlen_tiles");
  if (rc) return rc;
  attn_bwd_pre<<<static_cast<int>((pre_rows + 7) / 8), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), lse, ws, ws + pre_rows * AB_D,
      ws + pre_rows * AB_D + pre_rows, H, N, static_cast<int>(pad), pre_rows);
  rc = check_launch("attn_bwd_pre");
  if (rc) return rc;
  rc = launch_attn_bwd<true, true>(tmQ, tmK, tmV, tmdO, p, grid, stream);
  if (rc) return rc;
  attn_bwd_post<<<static_cast<int>((post_n + 255) / 256), 256, 0, stream>>>(ws, static_cast<__nv_bfloat16*>(dq), H, N,
                                                                            static_cast<int>(pad), 0, q_stride_h, scale, post_n);
  return check_launch("attn_bwd_post");
}
