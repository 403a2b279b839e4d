// Persistent wgmma GEMM (M=128 x N=BN tiles, two consumer warpgroups of 64 rows each).  See gemm_common.cuh for the design.
#include <cuda_fp8.h>

#include "gemm_common.cuh"

namespace aria {

// four k-blocks in flight: the ring takes what the fp32 staging tile of the epilogue leaves of the 227 KB per block
constexpr int GEMM_STAGES = 4;
// gemm_kernel with the hand-off epilogue (HANDOFF): no staging tile, so up to six 32 KB stages fit beside the 32 KB bf16
// output tile.  Six measured faster for the dense launches (nn.Linear weights: the LM's q/k/v, the shared gate/up), four for
// the grouped expert launches ([E, K, N] weights), whose 196,608-row launches ran 2-3 % slower with six (DESIGN §6).
constexpr int handoff_stages(bool b_mn) { return b_mn ? 4 : 6; }
// fp8 B (B_FP8): TMA lands the e4m3 boxes in a ring of their own, the producer warpgroup's three idle warps widen them to bf16
// in the SW128 layout of the bf16 ring, and the wgmma sequence is unchanged.  Three landing slots fit beside the four bf16
// stages and the fp32 staging tile (DESIGN §3); a fourth would not.
constexpr int FP8_LAND_STAGES = 3;
constexpr int FP8_CONVERT_WARPS = 3;
// Fewest rows of a dense LINEAR GEMM that runs as CTA pairs (gemm_run)
constexpr int PAIR_MIN_ROWS = 2048;
// Shortest reduction of a wide LINEAR GEMM that runs as CTA pairs (gemm_run)
constexpr int WIDE_PAIR_MIN_K = 2048;
// HANDOFF_RING: the ring's stages of a hand-off launch (handoff_stages), 0 for the staged epilogue (a CTA pair takes what
// one CTA takes)
template <int BN, bool B_FP8 = false, bool PAIR = false, int HANDOFF_RING = 0>
constexpr int gemm_smem_bytes() {
  return 1024 /*align*/ + (HANDOFF_RING ? HANDOFF_RING : GEMM_STAGES) * (A_STAGE_BYTES + BN * BK * 2) +
         (HANDOFF_RING ? 2 * 2 * OUT_BOX_BYTES : BM * acc_ld(BN) * 4) + 256 /*barriers*/ +
         (B_FP8 ? FP8_LAND_STAGES * BN * BK : 0);
}
static_assert(gemm_smem_bytes<128, true>() <= 232448, "fp8 landing ring must fit the opt-in shared memory of a block");
static_assert(gemm_smem_bytes<128, false, false, handoff_stages(false)>() <= 232448,
              "hand-off ring must fit the opt-in shared memory of a block");

// 16 e4m3 values (one 16-byte landing chunk, columns in address order) -> 16 bf16 in two 16-byte chunks; every e4m3 value,
// subnormals and -0 included, is exact in fp16, fp32 and bf16
ARIA_DEVICE void e4m3x16_to_bf16(const uint4 v, uint4& lo, uint4& hi) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t o[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w[i] >> (16 * h)), __NV_E4M3);
      const float2 f = __half22float2(__half2(hr));
      o[2 * i + h] = pack_bf16(f.x, f.y);
    }
  }
  lo = make_uint4(o[0], o[1], o[2], o[3]);
  hi = make_uint4(o[4], o[5], o[6], o[7]);
}

// The epilogue warps' part of gemm_kernel's hand-off (HANDOFF): half h of a 128-wide tile, which holds what epilogue_tile
// rounds first — bf16(x + bias) (LINEAR; HEADS without RoPE), bf16(gate) | bf16(up) in the two 64-column boxes (SWIGLU),
// bf16(x) (HEADS, a RoPE segment) — is finished with epilogue_tile's arithmetic and stored, consecutive threads on
// consecutive 16-byte chunks of a row so that each warp store covers whole row segments.  The row checks are
// epilogue_tile's: no row at or past the group's end (it belongs to the next group), per-group destinations, head-major
// rows in their own batch.  Ends with the one arrival on out_free.
template <int EPI>
ARIA_DEVICE void handoff_finish_half(const GemmParams& p, uint32_t half, uint64_t* out_free, int et, int h, int grp,
                                     int m_idx, int n_idx, int row0, int rows, int n_out_total) {
  const int r_base = m_idx * BM + 64 * h;  // row of the group at row 0 of the half
  if constexpr (EPI == ARIA_EPI_SWIGLU) {
    // out = bf16(bf16(silu(g)) * u) into 64 output columns: 8 chunks per row, 12 rows per step
    constexpr int CH = 8, ROW_STEP = EPI_THREADS / CH;
    const int c = (et % CH) * 8, col = n_idx * (BM / 2) + c;
    if (col + 8 <= p.N) {
      __nv_bfloat16* out = p.out[0] + col;
#pragma unroll 1
      for (int r = et / CH; r < 64 && r_base + r < rows; r += ROW_STEP) {
        const uint4 gv = ld_shared_v4(half + out_half_offset(r, c)), uv = ld_shared_v4(half + out_half_offset(r, 64 + c));
        const uint32_t g[4] = {gv.x, gv.y, gv.z, gv.w}, u[4] = {uv.x, uv.y, uv.z, uv.w};
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float s0 = fast_silu(bf16_lo(g[e])), s1 = fast_silu(bf16_hi(g[e]));
          bf16r2(s0, s1);
          o[e] = pack_bf16(s0 * bf16_lo(u[e]), s1 * bf16_hi(u[e]));
        }
        st_global_v4(out + static_cast<int64_t>(row0 + r_base + r) * p.ldo, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  } else if constexpr (EPI == ARIA_EPI_LINEAR) {
    // the activation, then the store: 16 chunks per row, 6 rows per step
    constexpr int CH = 16, ROW_STEP = EPI_THREADS / CH;
    const int c = (et % CH) * 8, col = n_idx * BM + c;
    if (col + 8 <= n_out_total) {
#pragma unroll 1
      for (int r = et / CH; r < 64 && r_base + r < rows; r += ROW_STEP) {
        const int r_in_grp = r_base + r;
        uint4 v = ld_shared_v4(half + out_half_offset(r, c));
        if (p.act == ARIA_ACT_GELU_TANH) act_bf16x8<ARIA_ACT_GELU_TANH>(v);
        else if (p.act == ARIA_ACT_GELU_NEW) act_bf16x8<ARIA_ACT_GELU_NEW>(v);
        // per-group destination: possibly a peer GPU's memory, the stores then travel over NVLink
        __nv_bfloat16* orow = p.out_group_base ? reinterpret_cast<__nv_bfloat16*>(p.out_group_base[grp]) +
                                                     static_cast<int64_t>(p.out_group_row0[grp] + r_in_grp) * p.ldo
                                               : p.out[0] + static_cast<int64_t>(row0 + r_in_grp) * p.ldo;
        st_global_v4(orow + col, v);
      }
    }
  } else {
    const int col0 = n_idx * BM, seg = col0 / p.N, cseg0 = col0 - seg * p.N;
    if ((p.rope_mask >> seg) & 1) {
      // the tile is one whole head (head_dim 128): rotate-half RoPE with op-by-op bf16 rounding,
      // out = bf16(bf16(x*cos) + bf16(rotate_half(x)*sin)); a thread takes a chunk of the low 64 columns and its partner 64
      // further on, 12 rows per step
      constexpr int CH = 8, ROW_STEP = EPI_THREADS / CH;
      const int c = (et % CH) * 8;
      __nv_bfloat16* head = p.out[seg] + (cseg0 / p.head_dim) * p.stride_h + c;
#pragma unroll 1
      for (int r = et / CH; r < 64 && r_base + r < rows; r += ROW_STEP) {
        const int grow = row0 + r_base + r;
        const int b = grow / p.rows_per_batch, tok = grow - b * p.rows_per_batch;
        const int pos = p.position_ids ? p.position_ids[grow] : p.pos0 + tok;
        const __nv_bfloat16* cs = p.rope_cos + static_cast<int64_t>(pos) * p.head_dim + c;
        const __nv_bfloat16* sn = p.rope_sin + static_cast<int64_t>(pos) * p.head_dim + c;
        const uint4 xlv = ld_shared_v4(half + out_half_offset(r, c)), xhv = ld_shared_v4(half + out_half_offset(r, 64 + c));
        const uint32_t xl[4] = {xlv.x, xlv.y, xlv.z, xlv.w}, xh[4] = {xhv.x, xhv.y, xhv.z, xhv.w};
        __nv_bfloat16* dst = head + b * p.stride_b + static_cast<int64_t>(p.pos0 + tok) * p.head_ld;
        // the low columns, x_lo cos_lo - x_hi sin_lo, then the high ones, x_hi cos_hi + x_lo sin_hi: one pair of table
        // vectors live at a time
#pragma unroll
        for (int part = 0; part < 2; ++part) {
          const uint4 cv = __ldg(reinterpret_cast<const uint4*>(cs + 64 * part));
          const uint4 sv = __ldg(reinterpret_cast<const uint4*>(sn + 64 * part));
          const uint32_t cw4[4] = {cv.x, cv.y, cv.z, cv.w}, sw4[4] = {sv.x, sv.y, sv.z, sv.w};
          const uint32_t* x0 = part ? xh : xl;  // times cos
          const uint32_t* x1 = part ? xl : xh;  // times sin, negated for the low columns
          uint32_t o[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float a0 = bf16_lo(x0[e]) * bf16_lo(cw4[e]), b0 = bf16_hi(x0[e]) * bf16_hi(cw4[e]);
            float a1 = (part ? bf16_lo(x1[e]) : -bf16_lo(x1[e])) * bf16_lo(sw4[e]);
            float b1 = (part ? bf16_hi(x1[e]) : -bf16_hi(x1[e])) * bf16_hi(sw4[e]);
            bf16r2(a0, a1);
            bf16r2(b0, b1);
            o[e] = pack_bf16(a0 + a1, b0 + b1);
          }
          st_global_v4(dst + 64 * part, make_uint4(o[0], o[1], o[2], o[3]));
        }
      }
    } else {
      // heads_store_tile's scatter of bf16(x + bias): 16 chunks per row, 6 rows per step
      constexpr int CH = 16, ROW_STEP = EPI_THREADS / CH;
      const int c = (et % CH) * 8, cs = cseg0 + c;
      if (cs + 8 <= p.N) {
        const int hd = cs / p.head_dim;
        __nv_bfloat16* col_base = p.out[seg] + hd * p.stride_h + (cs - hd * p.head_dim);
#pragma unroll 1
        for (int r = et / CH; r < 64 && r_base + r < rows; r += ROW_STEP) {
          const int grow = row0 + r_base + r;
          const int b = grow / p.rows_per_batch, tok = grow - b * p.rows_per_batch;
          st_global_v4(col_base + b * p.stride_b + static_cast<int64_t>(p.pos0 + tok) * p.head_ld,
                       ld_shared_v4(half + out_half_offset(r, c)));
        }
      }
    }
  }
  named_bar_sync(EPI_BAR, EPI_THREADS);  // every chunk of the half has been read
  if (et == 0) mbar_arrive(out_free);
}

template <int BN, bool B_MN>
ARIA_DEVICE void wgmma_tile_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 128) wgmma_m64n128_ss<0, B_MN ? 1 : 0>(acc, da, db, 1u);
  else wgmma_m64n144_ss<0, B_MN ? 1 : 0>(acc, da, db, 1u);
}

// PAIR: the kernel runs as clusters of two CTAs that take n-tiles 2 j and 2 j + 1 of the same m-tile (pair j).  Each CTA loads
// one 64-row half of the shared A tile and multicasts it into both CTAs' ring; each loads its own B.  Per CTA and k-block that
// is (64 + BN) x 64 instead of (128 + BN) x 64 elements from L2.  Protocol (DESIGN §3):
//   * full[s] of each CTA expects the whole stage, its own B and both A halves; its producer's expect_tx is the one arrival
//     (the peer's half may land first).
//   * empty[s] of each CTA counts the consumer warps of BOTH CTAs: no producer multicasts into a slot its peer still reads.
//   * with an odd n-tile count the last pair's second tile is a phantom: its CTA loads and multicasts its A half, waits for
//     and releases every stage like the others, and loads no B, issues no MMA and stores nothing.
//   * cluster barriers after the barrier init (before any remote access) and before exit (no CTA leaves while its peer can
//     still write its shared memory or arrive on its barriers).
// HANDOFF (gemm_handoff_kernel; gemm_run: grouped launches without a residual, SwiGLU, HEADS with RoPE; bf16 B, one CTA):
// the hand-off protocol of gemm_common.cuh in place of stage_and_epilogue.  The consumers write their fragment into a
// 64 x 128 bf16 half (what epilogue_tile rounds first, so the stored bits are unchanged) and start the next tile's k-loop;
// the epilogue warps finish the half (handoff_finish_half).  A warpgroup with no row of the tile in its half sits out, on
// both sides.  Without the 64 KB fp32 staging tile the ring has up to six stages (handoff_stages).
template <int BN, bool B_MN, int EPI, bool B_FP8, bool PAIR, bool HANDOFF>
ARIA_DEVICE void gemm_body(const CUtensorMap* tmA, const CUtensorMap* tmA_min, const CUtensorMap* tmB0,
                           const CUtensorMap* tmB1, const CUtensorMap* tmB2, const GemmParams& p) {
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  constexpr int STAGES = HANDOFF ? handoff_stages(B_MN) : GEMM_STAGES;
  constexpr int ACC_LD = acc_ld(BN);
  constexpr int OUT_BN = (EPI == ARIA_EPI_SWIGLU) ? BN / 2 : BN;  // output columns per tile
  constexpr int HALF_BYTES = 2 * OUT_BOX_BYTES;                   // HANDOFF: a consumer warpgroup's 64 x 128 bf16 half
  static_assert(BN == 128 || BN == 144, "tile widths with a wgmma wrapper");
  static_assert(!B_FP8 || (B_MN && BN == 128 && EPI != ARIA_EPI_HEADS), "fp8 B: grouped [G, K, N] weights, 128-wide tiles");
  static_assert(!PAIR || (!B_MN && !B_FP8), "CTA pairs: dense K-major bf16 B");
  static_assert(!HANDOFF || (BN == 128 && !B_FP8 && !PAIR), "hand-off: one-CTA bf16 launches, 128-wide tiles");
  constexpr int LAND_BYTES = BN * BK;  // one k-block of fp8 B: BN/64 boxes of 64 k-rows x 64 bytes, unswizzled

  uint8_t* smem = smem_1024();
  // HANDOFF: the bf16 output tile, [2 warpgroups][2 boxes][64 rows][128 B]; otherwise the fp32 accumulator staging tile,
  // [BM][ACC_LD]
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  const uint32_t out_tile = smem_u32(stg);
  const BarrierRing<STAGES> bar(smem + STAGES * STAGE_BYTES + (HANDOFF ? 2 * HALF_BYTES : BM * ACC_LD * 4));
  const HandoffBars hb(bar.empty + STAGES);  // HANDOFF
  // B_FP8: e4m3 landing ring after the barrier block; its full barriers complete on the TMA bytes, its empty ones once per
  // converter warp
  const BarrierRing<FP8_LAND_STAGES> land_bar(bar.empty + STAGES);
  uint8_t* land = reinterpret_cast<uint8_t*>(bar.full) + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(tmA);
    if (p.group_offsets) prefetch_tmap(tmA_min);
    prefetch_tmap(tmB0);
    if (p.n_seg > 1 || EPI == ARIA_EPI_SWIGLU) prefetch_tmap(tmB1);
    if (p.n_seg > 2) prefetch_tmap(tmB2);
    // B_FP8: a stage is full once A has landed AND every converter warp has written its share of B
    bar.init(B_FP8 ? 1 + FP8_CONVERT_WARPS : 1, PAIR ? 2 * CONSUMER_WARPS : CONSUMER_WARPS);
    if constexpr (B_FP8) land_bar.init(1, FP8_CONVERT_WARPS);
    if constexpr (HANDOFF) hb.init();
    fence_mbar_init();
  }
  if constexpr (PAIR) cluster_sync();
  else __syncthreads();

  const int n_out_total = p.N * (EPI == ARIA_EPI_SWIGLU ? 1 : p.n_seg);  // output columns overall
  const int n_tiles = (n_out_total + OUT_BN - 1) / OUT_BN;
  const int k_blocks = (p.K + BK - 1) / BK;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full0 = smem_u32(bar.full), empty0 = smem_u32(bar.empty);
  // grouped launch: A tiles are loaded and computed only as far as the group's rows reach (tma_load_a_rows)
  const bool grouped = !PAIR && p.group_offsets != nullptr;

  if (wg == 0) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<HANDOFF ? 80 : 40>();  // the epilogue warps: HEADS (RoPE) spilled at 56 to 72; 128 x 80 + 256 x 208 <= 64 K
    if (warp == 0 && elect_one()) {
      const uint32_t rank = PAIR ? cluster_ctarank() : 0;
      TileSched sched;
      sched.init(p, pair_sched_n<PAIR>(n_tiles));
      RingPos<STAGES> rp;
      RingPos<FP8_LAND_STAGES> lp;  // B_FP8 landing ring
      for (int t = first_tile<PAIR>();; t += tile_step<PAIR>()) {
        int grp, m_idx, n_idx, row0, rows;
        if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
        if constexpr (PAIR) n_idx = 2 * n_idx + rank;
        const bool phantom = PAIR && n_idx >= n_tiles;
        const int a_row = row0 + m_idx * BM;
        const int a_rows = grouped ? tile_a_rows(rows, m_idx) : BM;
        // PAIR: this CTA's half of the A tile; a half wholly past the last row is never read back, so the box is moved onto
        // the first half rather than issued out of bounds
        const int a_half_row = a_row + (m_idx * BM + static_cast<int>(rank) * (BM / 2) < rows ? rank * (BM / 2) : 0);
        const int bgrp = weight_block(p, grp);
        // B coordinates of this tile (k-invariant part)
        int b_c0 = 0, b_c1 = 0;          // K-major: row (n) coordinate of the two boxes; MN-major: base k row
        const CUtensorMap* tb0 = tmB0;
        const CUtensorMap* tb1 = tmB1;
        if constexpr (B_MN) {
          b_c0 = bgrp * p.K;
        } else if constexpr (EPI == ARIA_EPI_SWIGLU) {
          b_c0 = b_c1 = n_idx * OUT_BN;
        } else {
          const int col = n_idx * BN;
          const int seg = col / p.N;
          tb0 = seg == 0 ? tmB0 : (seg == 1 ? tmB1 : tmB2);
          b_c0 = col - seg * p.N + bgrp * p.b_group_rows;
        }
        for (int kb = 0; kb < k_blocks; ++kb) {
          const uint32_t fb = full0 + rp.stage * 8;
          const uint32_t sa = smem_base + rp.stage * STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          mbar_wait_addr(empty0 + rp.stage * 8, rp.phase ^ 1);
          if constexpr (PAIR) {
            mbar_arrive_expect_tx_addr(fb, phantom ? A_STAGE_BYTES : STAGE_BYTES);
            tma_load_2d_multicast_addr(sa + rank * (A_STAGE_BYTES / 2), tmA, fb, kb * BK, a_half_row, 0b11);
            if (phantom) {
              rp.next();
              continue;
            }
          } else {
            mbar_arrive_expect_tx_addr(fb, a_rows * (BK * 2) + (B_FP8 ? 0 : B_STAGE_BYTES));
            tma_load_a_rows(sa, tmA, tmA_min, fb, kb * BK, a_row, a_rows);
          }
          if constexpr (B_MN) {
            // B = [G*K, Ncols] rows k, N contiguous; one box = 64 k-rows x 64 n, BN/64 boxes per stage
            uint32_t dst = sb, box_bytes = 64 * BK * 2, bar_addr = fb;
            if constexpr (B_FP8) {
              // the e4m3 boxes go to the landing ring; the converters widen them into this stage's B slot.  That slot is
              // free: the converters see this k-block only after the empty-barrier wait above.
              bar_addr = smem_u32(land_bar.full) + lp.stage * 8;
              mbar_wait_addr(smem_u32(land_bar.empty) + lp.stage * 8, lp.phase ^ 1);
              mbar_arrive_expect_tx_addr(bar_addr, LAND_BYTES);
              dst = smem_u32(land) + lp.stage * LAND_BYTES;
              box_bytes = 64 * BK;
            }
            const int krow = b_c0 + kb * BK;
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              tma_load_2d_addr(dst + c * box_bytes, tmB0, bar_addr, tile_b_col<BN, EPI>(c * 64, n_idx, p.N), krow);
            if constexpr (B_FP8) lp.next();
          } else if constexpr (EPI == ARIA_EPI_SWIGLU) {
            tma_load_2d_addr(sb, tb0, fb, kb * BK, b_c0);
            tma_load_2d_addr(sb + (BN / 2) * BK * 2, tb1, fb, kb * BK, b_c1);
          } else {
            tma_load_2d_addr(sb, tb0, fb, kb * BK, b_c0);
          }
          rp.next();
        }
      }
    } else if constexpr (B_FP8) {
      if (warp > 0) {
        // ============ converters (warps 1-3): e4m3 landing slot -> bf16 B slot of the same k-block, SW128 MN-major ============
        // Chunk i of a landing slot is 16 fp8 columns: box i / 256, k-row (i / 4) % 64, columns 16 (i % 4) +[0, 16).  Widened,
        // they are the 16-byte chunks 2 (i % 4) and 2 (i % 4) + 1 of that 128-byte bf16 row, stored at chunk j ^ (row % 8)
        // as TMA's 128-byte swizzle would have placed them.
        const int ct = threadIdx.x - 32;
        TileSched sched;
        sched.init(p, n_tiles);
        RingPos<STAGES> rp;
        RingPos<FP8_LAND_STAGES> lp;
        for (int t = blockIdx.x;; t += gridDim.x) {
          int grp, m_idx, n_idx, row0, rows;
          if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
          for (int kb = 0; kb < k_blocks; ++kb) {
            mbar_wait_addr(smem_u32(land_bar.full) + lp.stage * 8, lp.phase);
            const uint8_t* src = land + lp.stage * LAND_BYTES;
            uint8_t* dst = smem + rp.stage * STAGE_BYTES + A_STAGE_BYTES;
#pragma unroll 1
            for (int i = ct; i < LAND_BYTES / 16; i += FP8_CONVERT_WARPS * 32) {
              const uint4 v = *reinterpret_cast<const uint4*>(src + i * 16);
              uint4 lo, hi;
              e4m3x16_to_bf16(v, lo, hi);
              const int r = (i >> 2) & 63, j = 2 * (i & 3);
              uint8_t* row = dst + (i >> 8) * (64 * BK * 2) + r * 128;
              *reinterpret_cast<uint4*>(row + ((j ^ (r & 7)) << 4)) = lo;
              *reinterpret_cast<uint4*>(row + (((j + 1) ^ (r & 7)) << 4)) = hi;
            }
            fence_proxy_async_smem();  // generic-proxy stores -> visible to the wgmma (async proxy) reads
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(&bar.full[rp.stage]);
              mbar_arrive(&land_bar.empty[lp.stage]);
            }
            rp.next();
            lp.next();
          }
        }
      }
    } else if constexpr (HANDOFF) {
      if (warp > 0) {
        // ================ epilogue warps (1-3): finish and store each half the consumers hand off ================
        const int et = threadIdx.x - 32;
        handoff_walk<false>(p, n_tiles, hb, [&](int h, int grp, int m_idx, int n_idx, int row0, int rows) {
          handoff_finish_half<EPI>(p, out_tile + h * HALF_BYTES, &hb.out_free[h], et, h, grp, m_idx, n_idx, row0, rows,
                                   n_out_total);
        });
      }
    }
  } else {
    // =========================== consumers: MMA + epilogue of rows [64 cw, +64) of each tile ===========================
    setmaxnreg_inc<HANDOFF ? 208 : 232>();
    const int cw = wg - 1;
    constexpr uint32_t b_lbo = B_MN ? 64 * BK * 2 : 16;
    constexpr uint32_t b_sbo = 1024;
    constexpr uint32_t b_kadv = (B_MN ? 16 * 128 : 32) >> 4;
    // descriptors of stage 0 / k-step 0; the start-address field is (addr >> 4) in the low 14 bits and shared-memory
    // addresses stay below 2^18, so adding (byte offset >> 4) never carries into the next field
    const uint64_t da0 = make_smem_desc(smem_base + cw * 64 * 128, 16, 1024);
    const uint64_t db0 = make_smem_desc(smem_base + A_STAGE_BYTES, b_lbo, b_sbo);
    const ConsumerThread ct = consumer_thread(cw, lane);
    const uint32_t rank = PAIR ? cluster_ctarank() : 0;
    TileSched sched;
    sched.init(p, pair_sched_n<PAIR>(n_tiles));
    RingPos<STAGES> rp;
    uint32_t free_phase = 0;  // HANDOFF: the phase of out_free[cw] to wait for, inverted
    const uint32_t half = out_tile + cw * HALF_BYTES;
    const int fr = ct.frag_row - 64 * cw;  // fragment rows fr and fr + 8 of the warpgroup's half
    // a stage is released to this CTA's producer and, PAIR, to the peer's, whose A half also lands in it
    auto release = [&](int s) {
      if (lane == 0) {
        mbar_arrive(&bar.empty[s]);
        if constexpr (PAIR) mbar_arrive_cluster(&bar.empty[s], rank ^ 1);
      }
    };
    // a tile this warpgroup computes nothing of: it waits for and releases every stage, so the barrier counts hold
    auto pass_tile = [&] {
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
        release(rp.stage);
        rp.next();
      }
    };
    for (int t = first_tile<PAIR>();; t += tile_step<PAIR>()) {
      int grp, m_idx, n_idx, row0, rows;
      if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
      if constexpr (PAIR) {
        n_idx = 2 * n_idx + rank;
        if (n_idx >= n_tiles) {  // phantom tile: the stages the peer's multicast fills
          pass_tile();
          continue;
        }
      }
      // grouped: no row of the group in rows [64, 128) of the tile, which are then not loaded either.  A whole warpgroup sits
      // out, so the named barrier of its stage_and_epilogue stays consistent.  HANDOFF: no row of the launch or group in
      // the warpgroup's half, as the epilogue warps' walk (handoff_walk) assumes.
      if (sits_out(HANDOFF ? m_idx * BM + 64 * cw >= rows : grouped && cw == 1 && rows - m_idx * BM <= BM / 2)) {
        pass_tile();
        continue;
      }
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      float2 bsc[BN / 8];
      if constexpr (B_FP8) load_col_scales<BN, EPI>(p, grp, n_idx, ct.frag_col, bsc);
      // HANDOFF, LINEAR and HEADS: bias pairs of this thread's columns (8 j + frag_col, +1), fetched while the k-loop runs; a
      // tile lies in one segment, columns past N get 0 and are never stored.  SwiGLU and RoPE segments have no bias.
      uint32_t bias2[BN / 8];
      bool has_bias = false;  // no bias: nothing is added, so a -0 stays -0 as in epilogue_tile
      if constexpr (HANDOFF && EPI != ARIA_EPI_SWIGLU) {
        const int col0 = n_idx * BN, seg = col0 / p.N, cseg0 = col0 - seg * p.N;
        const __nv_bfloat16* bias = p.bias[seg];
        has_bias = bias != nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = cseg0 + 8 * j + ct.frag_col;
          bias2[j] = (bias && c < p.N) ? __ldg(reinterpret_cast<const uint32_t*>(bias + c)) : 0u;
        }
      }
      // one k-block's wgmma group stays in flight while the next one is issued; a stage is released once its group retired
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
        const uint64_t da = da0 + rp.stage * (STAGE_BYTES >> 4);
        const uint64_t db = db0 + rp.stage * (STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_tile_k16<BN, B_MN>(acc, da + k * 2, db + k * b_kadv);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = static_cast<int>(rp.stage);
        rp.next();
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) release(prev);
      if constexpr (HANDOFF) {
        // the epilogue warps have finished this warpgroup's previous tile and left its half
        mbar_wait(&hb.out_free[cw], free_phase ^ 1);
        free_phase ^= 1;
        // what epilogue_tile rounds first: bf16(x + bias) (LINEAR, HEADS; SwiGLU: bf16(gate) | bf16(up), RoPE: bf16(x))
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {  // rows fr and fr + 8
            float x0 = acc[4 * j + 2 * i], x1 = acc[4 * j + 2 * i + 1];
            if (has_bias) {
              x0 += bf16_lo(bias2[j]);
              x1 += bf16_hi(bias2[j]);
            }
            st_shared_u32(half + out_half_offset(fr + 8 * i, 8 * j + ct.frag_col), pack_bf16(x0, x1));
          }
        }
        mbar_arrive(&hb.out_full[cw]);
        continue;
      }
      stage_and_epilogue<BN, EPI, B_FP8 ? AccScale::COL : AccScale::NONE>(p, stg, ct, acc, bsc, 1.f, 1.f, n_out_total, grp,
                                                                           m_idx, n_idx, row0, rows);
    }
  }
  if constexpr (PAIR) cluster_sync();
}

template <int BN, bool B_MN, int EPI, bool B_FP8 = false, bool PAIR = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA_min,
            const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
            const __grid_constant__ CUtensorMap tmB2, const GemmParams p) {
  gemm_body<BN, B_MN, EPI, B_FP8, PAIR, false>(&tmA, &tmA_min, &tmB0, &tmB1, &tmB2, p);
}

// gemm_kernel with the hand-off epilogue (HANDOFF above): 128-wide tiles, bf16 B, one CTA
template <bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_handoff_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA_min,
                    const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
                    const __grid_constant__ CUtensorMap tmB2, const GemmParams p) {
  gemm_body<128, B_MN, EPI, false, false, true>(&tmA, &tmA_min, &tmB0, &tmB1, &tmB2, p);
}

// Wide dense GEMM for the 4,900-row ViT and projector launches (gemm_run): bf16, nn.Linear weights, LINEAR or HEADS without
// RoPE.  128 x 192 tiles (1152 = 6 x 192), each consumer warpgroup one wgmma m64n192k16 per k16 step on its 64 rows.  The
// epilogue starts on the accumulator registers: each thread adds the bias to its fragment and rounds it exactly as
// epilogue_tile / heads_store_tile do and writes it as bf16 into its warpgroup's 64 x 192 half of an output tile in shared
// memory (three 64 x 64 SW128 boxes, 24 KB).  Without the fp32 staging tile of gemm_kernel the ring keeps four 40 KB stages.
//   * LINEAR without a residual, and HEADS (hand-off): the consumers write bias + rounding only, arrive on out_full[cw] and
//     go on to the next tile's k-loop; before writing the next tile's half they wait on out_free[cw].  The producer
//     warpgroup's idle warps 1-3 (the epilogue warps) walk the same tiles: per half they wait on out_full, apply the
//     activation in place (LINEAR; it sees bf16(x + bias) either way, so the bits are those of epilogue_tile), then one of
//     them TMA-stores the half, waits for the store to have read it and arrives on out_free.  HEADS: they read the half back
//     in 16-byte chunks and scatter them head-major with heads_store_tile's mapping (a 192-wide tile spans 2 2/3 heads of
//     72, so TMA cannot store it), then arrive on out_free.  The tensor cores no longer idle through those epilogues.
//   * LINEAR with a residual: one thread per warpgroup stores the half with TMA and does not wait for it; it waits for the
//     store to have read the half during the next tile's first k-block.  The producer TMA-loads the tile's residual rows
//     into the half once that wait is over (out_free), on a barrier of its own (res_full), and the consumers add them at
//     their fragment positions: out = bf16(x + res).  These launches' time is their mainloop (DESIGN §6).
// HANDOFF selects the first protocol, per launch (gemm_run: no residual), so the residual instantiations carry no hand-off
// code.  A half with no row of the launch is neither computed nor stored.  PAIR: the A-multicast CTA pairs of gemm_kernel
// (same protocol, same phantom tile).
constexpr int WIDE_BN = 192;
constexpr int WIDE_STAGE_BYTES = A_STAGE_BYTES + WIDE_BN * BK * 2;  // 16 + 24 KB
constexpr int WIDE_HALF_BYTES = 3 * OUT_BOX_BYTES;  // a consumer warpgroup's 64 output rows: three boxes
constexpr int gemm_wide_smem_bytes() {
  return 1024 /*align*/ + GEMM_STAGES * WIDE_STAGE_BYTES + 2 * WIDE_HALF_BYTES + 256 /*barriers*/;
}
static_assert(gemm_wide_smem_bytes() <= 232448, "wide GEMM must fit the opt-in shared memory of a block");

template <int EPI, bool PAIR, bool HANDOFF>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
                 const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2,
                 const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes, const GemmParams p) {
  constexpr int BN = WIDE_BN;
  constexpr int STAGES = GEMM_STAGES;
  static_assert(EPI == ARIA_EPI_LINEAR || EPI == ARIA_EPI_HEADS, "wide GEMM epilogues");
  static_assert(HANDOFF || EPI == ARIA_EPI_LINEAR, "HEADS launches hand off");

  uint8_t* smem = smem_1024();
  uint8_t* out_tile = smem + STAGES * WIDE_STAGE_BYTES;  // [2 warpgroups][3 boxes][64 rows][128 B]
  const BarrierRing<STAGES> bar(out_tile + 2 * WIDE_HALF_BYTES);
  // out_free[2]: a warpgroup's previous tile has left its half (stored or scattered); out_full[2]: hand-off only
  const HandoffBars hb(bar.empty + STAGES);
  uint64_t* out_free = hb.out_free;
  uint64_t* res_full = out_free + 2;  // [2]: the residual rows of a warpgroup's half have landed in it

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  constexpr bool handoff = HANDOFF;
  constexpr bool res = !HANDOFF;  // LINEAR with a residual

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB0);
    if (p.n_seg > 1) prefetch_tmap(&tmB1);
    if (p.n_seg > 2) prefetch_tmap(&tmB2);
    if (EPI == ARIA_EPI_LINEAR) prefetch_tmap(&tmOut);
    if (res) prefetch_tmap(&tmRes);
    bar.init(1, PAIR ? 2 * CONSUMER_WARPS : CONSUMER_WARPS);
    hb.init();
    for (int h = 0; h < 2; ++h) mbar_init(&res_full[h], 1);
    fence_mbar_init();
  }
  if constexpr (PAIR) cluster_sync();
  else __syncthreads();

  const int n_out_total = p.N * p.n_seg;
  const int n_tiles = (n_out_total + BN - 1) / BN;
  const int k_blocks = (p.K + BK - 1) / BK;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full0 = smem_u32(bar.full), empty0 = smem_u32(bar.empty);
  // output boxes of a tile that hold a column of the launch (fc1's 80-column tail tile: 2)
  auto tile_boxes = [&](int col0) { return min(3, (n_out_total - col0 + 63) / 64); };

  if (wg == 0) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<56>();  // the residual loads and the pair rank need more than 40
    if (warp == 0 && elect_one()) {
      const uint32_t rank = PAIR ? cluster_ctarank() : 0;
      TileSched sched;
      sched.init(p, pair_sched_n<PAIR>(n_tiles));
      RingPos<STAGES> rp;
      uint32_t out_phase = 0;  // bit h: the phase of out_free[h] to wait for
      for (int t = first_tile<PAIR>();; t += tile_step<PAIR>()) {
        int grp, m_idx, n_idx, row0, rows;
        if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
        if constexpr (PAIR) n_idx = 2 * n_idx + rank;
        const bool phantom = PAIR && n_idx >= n_tiles;
        const int a_row = m_idx * BM;
        // PAIR: this CTA's half of the A tile, moved onto the first half when it lies wholly past the last row (gemm_kernel)
        const int a_half_row = a_row + (a_row + static_cast<int>(rank) * (BM / 2) < rows ? rank * (BM / 2) : 0);
        const int col0 = n_idx * BN;
        const int seg = col0 / p.N;
        const CUtensorMap* tb = seg == 0 ? &tmB0 : (seg == 1 ? &tmB1 : &tmB2);
        const int b_row = col0 - seg * p.N;
        // the residual goes in once the ring is full: by then the consumers are at this tile's first k-block, where they
        // release the output tile
        const int res_kb = min(STAGES - 1, k_blocks - 1);
        for (int kb = 0; kb < k_blocks; ++kb) {
          const uint32_t fb = full0 + rp.stage * 8;
          const uint32_t sa = smem_base + rp.stage * WIDE_STAGE_BYTES;
          mbar_wait_addr(empty0 + rp.stage * 8, rp.phase ^ 1);
          if constexpr (PAIR) {
            mbar_arrive_expect_tx_addr(fb, phantom ? A_STAGE_BYTES : WIDE_STAGE_BYTES);
            tma_load_2d_multicast_addr(sa + rank * (A_STAGE_BYTES / 2), &tmA, fb, kb * BK, a_half_row, 0b11);
            if (phantom) {
              rp.next();
              continue;
            }
          } else {
            mbar_arrive_expect_tx_addr(fb, WIDE_STAGE_BYTES);
            tma_load_2d_addr(sa, &tmA, fb, kb * BK, a_row);
          }
          tma_load_2d_addr(sa + A_STAGE_BYTES, tb, fb, kb * BK, b_row);
          rp.next();
          if (res && kb == res_kb) {
            const int nbox = tile_boxes(col0);
            for (int h = 0; h < 2; ++h) {
              if (a_row + 64 * h >= rows) continue;  // a half past the last row: no consumer waits for it
              mbar_wait(&out_free[h], (out_phase >> h) & 1);
              out_phase ^= 1u << h;
              mbar_arrive_expect_tx(&res_full[h], nbox * OUT_BOX_BYTES);
              for (int c = 0; c < nbox; ++c)
                tma_load_2d(out_tile + h * WIDE_HALF_BYTES + c * OUT_BOX_BYTES, &tmRes, &res_full[h], col0 + 64 * c,
                            a_row + 64 * h);
            }
          }
        }
      }
    } else if (warp > 0 && handoff) {
      // ================ epilogue warps (1-3): activation and store of each half the consumers hand off ================
      const int et = threadIdx.x - 32;
      handoff_walk<PAIR>(p, n_tiles, hb, [&](int h, int grp, int m_idx, int n_idx, int row0, int rows) {
        const int col0 = n_idx * BN;
        const int seg = col0 / p.N;
        const int cseg0 = col0 - seg * p.N;
        const uint32_t half = smem_u32(out_tile) + h * WIDE_HALF_BYTES;
        if constexpr (EPI == ARIA_EPI_LINEAR) {
          const int nbox = tile_boxes(col0);
          if (p.act == ARIA_ACT_GELU_TANH || p.act == ARIA_ACT_GELU_NEW) {
            const int n_chunks = nbox * (OUT_BOX_BYTES / 16);
            if (p.act == ARIA_ACT_GELU_TANH) act_inplace<ARIA_ACT_GELU_TANH>(half, n_chunks, et);
            else act_inplace<ARIA_ACT_GELU_NEW>(half, n_chunks, et);
            fence_proxy_async_smem();
          }
          named_bar_sync(EPI_BAR, EPI_THREADS);
          if (et == 0) {
            fence_proxy_async_smem();
            for (int c = 0; c < nbox; ++c)
              tma_store_2d_addr(&tmOut, half + c * OUT_BOX_BYTES, col0 + 64 * c, m_idx * BM + 64 * h);
            bulk_commit_group();
            bulk_wait_group_read<0>();
            mbar_arrive(&out_free[h]);
          }
        } else {
          // heads_store_tile's mapping, consecutive threads on consecutive 8-column chunks of a row.  96 threads are 4 rows
          // of 24 chunks, so a thread keeps its column chunk (head, d) and steps 4 rows at a time.
          constexpr int CH = BN / 8;
          constexpr int ROW_STEP = EPI_THREADS / CH;
          static_assert(EPI_THREADS % CH == 0, "a thread keeps its column chunk");
          const int c = (et % CH) * 8, cs = cseg0 + c;
          if (cs + 8 <= p.N) {
            const int head = cs / p.head_dim, d = cs - head * p.head_dim;
            __nv_bfloat16* col_base = p.out[seg] + head * p.stride_h + d;
            int r = et / CH, r_in_grp = m_idx * BM + 64 * h + r;
            int b = r_in_grp / p.rows_per_batch, tok = r_in_grp - b * p.rows_per_batch;
#pragma unroll 1
            for (; r < 64 && r_in_grp < rows; r += ROW_STEP, r_in_grp += ROW_STEP) {
              st_global_v4(col_base + b * p.stride_b + static_cast<int64_t>(p.pos0 + tok) * p.head_ld,
                           ld_shared_v4(half + out_half_offset(r, c)));
              for (tok += ROW_STEP; tok >= p.rows_per_batch; tok -= p.rows_per_batch) ++b;
            }
          }
          named_bar_sync(EPI_BAR, EPI_THREADS);  // every chunk of the half has been read
          if (et == 0) mbar_arrive(&out_free[h]);
        }
      });
    }
  } else {
    // =========================== consumers: MMA + epilogue of rows [64 cw, +64) of each tile ===========================
    setmaxnreg_inc<224>();
    const int cw = wg - 1;
    const uint64_t da0 = make_smem_desc(smem_base + cw * 64 * 128, 16, 1024);
    const uint64_t db0 = make_smem_desc(smem_base + A_STAGE_BYTES, 16, 1024);
    const ConsumerThread ct = consumer_thread(cw, lane);
    const int fr = ct.frag_row - 64 * cw;  // fragment rows fr and fr + 8 of the warpgroup's half
    const bool leader = (threadIdx.x & 127) == 0;
    uint8_t* half = out_tile + cw * WIDE_HALF_BYTES;
    const uint32_t half_s = smem_u32(half);
    const uint32_t rank = PAIR ? cluster_ctarank() : 0;
    TileSched sched;
    sched.init(p, pair_sched_n<PAIR>(n_tiles));
    RingPos<STAGES> rp;
    uint32_t res_phase = 0, free_phase = 0;
    auto release = [&](int s) {
      if (lane == 0) {
        mbar_arrive(&bar.empty[s]);
        if constexpr (PAIR) mbar_arrive_cluster(&bar.empty[s], rank ^ 1);
      }
    };
    auto pass_tile = [&] {
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
        release(rp.stage);
        rp.next();
      }
    };
    for (int t = first_tile<PAIR>();; t += tile_step<PAIR>()) {
      int grp, m_idx, n_idx, row0, rows;
      if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
      if constexpr (PAIR) n_idx = 2 * n_idx + rank;
      // a phantom tile, or no row of the launch in this warpgroup's half (the 36-row last m-tile of 4,900)
      if (sits_out((PAIR && n_idx >= n_tiles) || m_idx * BM + 64 * cw >= rows)) {
        pass_tile();
        continue;
      }
      const int col0 = n_idx * BN;
      const int seg = col0 / p.N;
      const int cseg0 = col0 - seg * p.N;
      const __nv_bfloat16* bias = p.bias[seg];
      // bias pairs of this thread's columns (8 j + frag_col, +1), fetched while the k-loop runs; columns past N get 0
      uint32_t bias2[BN / 8];
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = cseg0 + 8 * j + ct.frag_col;
        bias2[j] = (bias && c < p.N) ? __ldg(reinterpret_cast<const uint32_t*>(bias + c)) : 0u;
      }
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
        const uint64_t da = da0 + rp.stage * (WIDE_STAGE_BYTES >> 4);
        const uint64_t db = db0 + rp.stage * (WIDE_STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_m64n192_ss<0, 0>(acc, da + k * 2, db + k * 2, 1u);
        wgmma_commit();
        if (res && kb == 0 && leader) {
          // the previous tile's store has read this half; the producer may now load this tile's residual
          bulk_wait_group_read<0>();
          mbar_arrive(&out_free[cw]);
        }
        wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = static_cast<int>(rp.stage);
        rp.next();
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) release(prev);
      if (handoff) {
        // the epilogue warps have stored or scattered this warpgroup's previous tile and left its half
        mbar_wait(&out_free[cw], free_phase ^ 1);
        free_phase ^= 1;
        // bias and rounding only, in a loop of its own: the residual loop below, with its per-element branches on the
        // activation, unrolls to ~9k instructions, and fc1 measured 113-115 us through it, 89-94 us with this loop (DESIGN §6)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {  // rows fr and fr + 8
            float x0 = acc[4 * j + 2 * i], x1 = acc[4 * j + 2 * i + 1];
            if (bias) {
              x0 += bf16_lo(bias2[j]);
              x1 += bf16_hi(bias2[j]);
            }
            st_shared_u32(half_s + out_half_offset(fr + 8 * i, 8 * j + ct.frag_col), pack_bf16(x0, x1));
          }
        }
        if constexpr (EPI == ARIA_EPI_LINEAR) fence_proxy_async_smem();  // the epilogue warps' TMA store reads the half
        mbar_arrive(&hb.out_full[cw]);
        continue;
      }
      if constexpr (EPI == ARIA_EPI_LINEAR) {  // with a residual
        mbar_wait(&res_full[cw], res_phase);
        res_phase ^= 1;
        named_bar_sync(1 + cw, 128);  // the leader has seen the previous store read the half
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + ct.frag_col;
#pragma unroll
          for (int i = 0; i < 2; ++i) {  // rows fr and fr + 8
            uint32_t* dst = reinterpret_cast<uint32_t*>(half + out_half_offset(fr + 8 * i, c));
            float x0 = acc[4 * j + 2 * i], x1 = acc[4 * j + 2 * i + 1];
            if (bias) {
              x0 += bf16_lo(bias2[j]);
              x1 += bf16_hi(bias2[j]);
            }
            x0 = bf16r(x0);
            x1 = bf16r(x1);
            if (p.act != ARIA_ACT_NONE) {
              x0 = bf16r(act_apply(x0, p.act));
              x1 = bf16r(act_apply(x1, p.act));
            }
            const uint32_t r = *dst;
            x0 += bf16_lo(r);
            x1 += bf16_hi(r);
            *dst = pack_bf16(x0, x1);
          }
          // one 64-column box at a time: hoisting all 48 residual loads ahead of the arithmetic spilled registers
          if (j % 8 == 7) asm volatile("" ::: "memory");
        }
        fence_proxy_async_smem();
        named_bar_sync(1 + cw, 128);
        if (leader) {
          const int nbox = tile_boxes(col0);
          for (int c = 0; c < nbox; ++c)
            tma_store_2d_addr(&tmOut, smem_u32(half + c * OUT_BOX_BYTES), col0 + 64 * c, m_idx * BM + 64 * cw);
          bulk_commit_group();
        }
      }
    }
    if (leader) bulk_wait_group_read<0>();  // no CTA leaves while a store still reads its shared memory
  }
  if constexpr (PAIR) cluster_sync();
}

// W8A8 grouped GEMM: e4m3 A [rows, K] with one fp32 scale per row, e4m3 B [G * N_b, K] (K-major: fp8 wgmma has no transpose)
// with one per (group, column).  The pipeline, tile scheduler and epilogues are gemm_kernel's; a k-block is 128 fp8 elements,
// one 128-byte SW128 row, so the A and B stages keep their 16 KB and the K-major descriptors are the bf16 ones.  The tensor
// core's fp8 accumulation keeps ~14 bits, so each k-block is accumulated on its own (`part`) and promoted into the fp32
// accumulator before the next one starts; the other consumer warpgroup keeps the tensor cores busy during that wait.
constexpr int W8_BK = 128;
static_assert(BM * W8_BK == A_STAGE_BYTES, "W8A8 A stage = bf16 A stage");

// Dense nn.Linear weights (gemm_w8a8_dense_kernel): one [N, K] e4m3 weight and one fp32 scale per output column for each
// segment s < n_seg (q / k / v, or gate / up for SwiGLU), each behind its own tensor map, so the weights stay separate tensors
struct W8a8DenseScales {
  const float* b[3];
};

// The column scales of this thread's accumulator columns in tile n_idx of a dense launch (load_col_scales of the grouped
// kernel, per segment): LINEAR / HEADS tiles lie in one segment (n_seg > 1: N % 128 == 0); a SwiGLU tile holds BN/2 gate
// columns, then the matching up columns.  Columns past N get 0.
template <int BN, int EPI>
ARIA_DEVICE void load_dense_col_scales(const GemmParams& p, const W8a8DenseScales& sc, int n_idx, int frag_col,
                                       float2 (&bsc)[BN / 8]) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    int col, seg;
    if constexpr (EPI == ARIA_EPI_SWIGLU) {
      seg = 8 * j < BN / 2 ? 0 : 1;
      col = n_idx * (BN / 2) + 8 * j - seg * (BN / 2) + frag_col;
    } else {
      seg = n_idx * BN / p.N;
      col = n_idx * BN - seg * p.N + 8 * j + frag_col;
    }
    const float* srow = seg == 0 ? sc.b[0] : (seg == 1 ? sc.b[1] : sc.b[2]);  // no dynamic index: keeps sc out of local memory
    bsc[j] = col < p.N ? __ldg(reinterpret_cast<const float2*>(srow + col)) : make_float2(0.f, 0.f);
  }
}

// The W8A8 pipeline.  Grouped (DENSE = false): one B map over the [G * N_b, K] expert weights; A is loaded as far as the
// group's rows reach and warpgroup 2 sits out tiles it has no row in, as in gemm_kernel's grouped launches (tmA_min:
// tma_load_a_rows).  DENSE: up to three [N, K]
// weights (tmB0..2, one per segment), a single group of p.M rows, and every epilogue of gemm_kernel (LINEAR with residual,
// SWIGLU from separate gate and up weights, HEADS with RoPE).  The k-loop, the tile and the promotion are the same.
template <int EPI, bool DENSE>
ARIA_DEVICE void w8a8_body(const CUtensorMap* tmA, const CUtensorMap* tmA_min, const CUtensorMap* tmB0, const CUtensorMap* tmB1,
                           const CUtensorMap* tmB2, const GemmParams& p, const float* __restrict__ a_scale,
                           const W8a8DenseScales& dsc) {
  constexpr int BN = 128;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * W8_BK;
  constexpr int STAGES = GEMM_STAGES;
  constexpr int ACC_LD = acc_ld(BN);
  constexpr int OUT_BN = (EPI == ARIA_EPI_SWIGLU) ? BN / 2 : BN;
  static_assert(DENSE || EPI == ARIA_EPI_LINEAR || EPI == ARIA_EPI_SWIGLU, "W8A8 grouped: expert GEMM epilogues");

  uint8_t* smem = smem_1024();
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  const BarrierRing<STAGES> bar(stg + BM * ACC_LD);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(tmA);
    if constexpr (!DENSE) prefetch_tmap(tmA_min);
    prefetch_tmap(tmB0);
    if constexpr (DENSE) {
      if (p.n_seg > 1 || EPI == ARIA_EPI_SWIGLU) prefetch_tmap(tmB1);
      if (p.n_seg > 2) prefetch_tmap(tmB2);
    }
    bar.init(1, CONSUMER_WARPS);
    fence_mbar_init();
  }
  __syncthreads();

  // output columns overall: dense LINEAR / HEADS launches have n_seg segments of N columns
  const int n_out_total = DENSE ? p.N * (EPI == ARIA_EPI_SWIGLU ? 1 : p.n_seg) : p.N;
  const int n_tiles = (n_out_total + OUT_BN - 1) / OUT_BN;
  const int k_blocks = p.K / W8_BK;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full0 = smem_u32(bar.full), empty0 = smem_u32(bar.empty);

  if (wg == 0) {
    // =========================== TMA producer ===========================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      TileSched sched;
      sched.init(p, n_tiles);
      RingPos<STAGES> rp;
      for (int t = blockIdx.x;; t += gridDim.x) {
        int grp, m_idx, n_idx, row0, rows;
        if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
        const int a_row = row0 + m_idx * BM;
        const int a_rows = DENSE ? BM : tile_a_rows(rows, m_idx);  // rows of W8_BK e4m3 = 128 bytes, as the bf16 k-block's
        // B rows of the two 64-row boxes: (group, column c) is row group * N_b + c; SwiGLU takes the gate and the up box
        int b_r0, b_r1;
        const CUtensorMap* tb0 = tmB0;
        const CUtensorMap* tb1 = tmB0;
        if constexpr (DENSE) {
          if constexpr (EPI == ARIA_EPI_SWIGLU) {
            b_r0 = b_r1 = n_idx * OUT_BN;
            tb1 = tmB1;
          } else {
            const int col = n_idx * BN;
            const int seg = col / p.N;
            tb0 = tb1 = seg == 0 ? tmB0 : (seg == 1 ? tmB1 : tmB2);
            b_r0 = col - seg * p.N;
            b_r1 = b_r0 + 64;
          }
        } else if constexpr (EPI == ARIA_EPI_SWIGLU) {
          b_r0 = weight_block(p, grp) * 2 * p.N + n_idx * OUT_BN;
          b_r1 = b_r0 + p.N;
        } else {
          b_r0 = weight_block(p, grp) * p.N + n_idx * BN;
          b_r1 = b_r0 + 64;
        }
        for (int kb = 0; kb < k_blocks; ++kb) {
          const uint32_t fb = full0 + rp.stage * 8;
          const uint32_t sa = smem_base + rp.stage * STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          mbar_wait_addr(empty0 + rp.stage * 8, rp.phase ^ 1);
          mbar_arrive_expect_tx_addr(fb, a_rows * W8_BK + BN * W8_BK);
          tma_load_a_rows(sa, tmA, tmA_min, fb, kb * W8_BK, a_row, a_rows);
          tma_load_2d_addr(sb, tb0, fb, kb * W8_BK, b_r0);
          tma_load_2d_addr(sb + 64 * W8_BK, tb1, fb, kb * W8_BK, b_r1);
          rp.next();
        }
      }
    }
  } else {
    // =========================== consumers: MMA + epilogue of rows [64 cw, +64) of each tile ===========================
    setmaxnreg_inc<232>();
    const int cw = wg - 1;
    const uint64_t da0 = make_smem_desc(smem_base + cw * 64 * 128, 16, 1024);
    const uint64_t db0 = make_smem_desc(smem_base + A_STAGE_BYTES, 16, 1024);
    const ConsumerThread ct = consumer_thread(cw, lane);
    TileSched sched;
    sched.init(p, n_tiles);
    RingPos<STAGES> rp;
    float part[BN / 2];  // one k-block's tensor-core sum (the first wgmma of a k-block overwrites it)
    for (int t = blockIdx.x;; t += gridDim.x) {
      int grp, m_idx, n_idx, row0, rows;
      if (!sched.decode(t, grp, m_idx, n_idx, row0, rows)) break;
      // grouped: no row of the group in rows [64, 128) of the tile (gemm_kernel): wait for and release every stage
      if (sits_out(!DENSE && cw == 1 && rows - m_idx * BM <= BM / 2)) {
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
          if (lane == 0) mbar_arrive(&bar.empty[rp.stage]);
          rp.next();
        }
        continue;
      }
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      float2 bsc[BN / 8];
      if constexpr (DENSE) load_dense_col_scales<BN, EPI>(p, dsc, n_idx, ct.frag_col, bsc);
      else load_col_scales<BN, EPI>(p, grp, n_idx, ct.frag_col, bsc);
      // row scales of the fragment's two rows (rows past the group's end are computed but never stored; the index is clamped
      // to the buffer)
      const int ar = row0 + m_idx * BM + ct.frag_row;
      const float as0 = __ldg(a_scale + min(ar, p.M - 1)), as1 = __ldg(a_scale + min(ar + 8, p.M - 1));
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait_addr(full0 + rp.stage * 8, rp.phase);
        const uint64_t da = da0 + rp.stage * (STAGE_BYTES >> 4);
        const uint64_t db = db0 + rp.stage * (STAGE_BYTES >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < W8_BK / 32; ++k) wgmma_m64n128k32_e4m3_ss(part, da + k * 2, db + k * 2, k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(part);
        if (lane == 0) mbar_arrive(&bar.empty[rp.stage]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        rp.next();
      }
      stage_and_epilogue<BN, EPI, AccScale::ROW_COL>(p, stg, ct, acc, bsc, as0, as1, n_out_total, grp, m_idx, n_idx, row0,
                                                     rows);
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_w8a8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA_min,
                 const __grid_constant__ CUtensorMap tmB, const GemmParams p, const float* __restrict__ a_scale) {
  w8a8_body<EPI, false>(&tmA, &tmA_min, &tmB, &tmB, &tmB, p, a_scale, W8a8DenseScales{});
}

template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_w8a8_dense_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
                       const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2, const GemmParams p,
                       const float* __restrict__ a_scale, const W8a8DenseScales b_scale) {
  w8a8_body<EPI, true>(&tmA, &tmA, &tmB0, &tmB1, &tmB2, p, a_scale, b_scale);
}

}  // namespace aria

using namespace aria;

static GemmParams gemm_params(const aria_gemm_desc_t* d, const float* b_scale) {
  const bool swiglu = d->epilogue == ARIA_EPI_SWIGLU;
  GemmParams p{};
  p.M = static_cast<int>(d->m);
  p.N = static_cast<int>(d->n);
  p.K = static_cast<int>(d->k);
  p.num_groups = d->num_groups;
  p.group_offsets = d->group_offsets;
  p.group_counts = d->group_counts;
  p.out_group_base = static_cast<const uint64_t*>(d->out_group_base);
  p.out_group_row0 = d->out_group_row0;
  p.group_mod = d->group_mod;
  p.b_group_rows = d->b_layout == ARIA_B_GNK ? static_cast<int>(d->n) : 0;
  p.n_seg = swiglu ? 1 : d->n_seg;
  p.act = d->act;
  for (int i = 0; i < 3; ++i) {
    p.bias[i] = static_cast<const __nv_bfloat16*>(d->bias[i]);
    p.out[i] = static_cast<__nv_bfloat16*>(d->out[i]);
  }
  p.residual = static_cast<const __nv_bfloat16*>(d->residual);
  p.ldr = d->ldr;
  p.ldo = d->ldo;
  p.head_dim = d->head_dim;
  p.head_ld = d->head_ld;
  p.rows_per_batch = d->rows_per_batch > 0 ? d->rows_per_batch : static_cast<int>(d->m);
  p.pos0 = d->pos0;
  p.stride_b = d->stride_b;
  p.stride_h = d->stride_h;
  p.rope_mask = d->rope_mask;
  p.rope_cos = static_cast<const __nv_bfloat16*>(d->rope_cos);
  p.rope_sin = static_cast<const __nv_bfloat16*>(d->rope_sin);
  p.position_ids = d->position_ids;
  p.b_scale = b_scale;
  return p;
}

// out[rows, n] = a[rows, k] x weight block g of b, for the rows of group g
static aria_gemm_desc_t grouped_desc(const void* a, const void* b, void* out, const int32_t* offsets, int64_t rows, int64_t k,
                                     int64_t n, int32_t groups, int32_t epilogue) {
  aria_gemm_desc_t d{};
  d.a = a;
  d.lda = k;
  d.m = rows;
  d.n = n;
  d.k = k;
  d.b[0] = b;
  d.n_seg = 1;
  d.b_layout = ARIA_B_GKN;
  d.num_groups = groups;
  d.group_offsets = offsets;
  d.epilogue = epilogue;
  d.out[0] = out;
  d.ldo = n;
  return d;
}

// Tiles of a launch at most: n-tiles x (m-tiles of all rows + one partial m-tile for each of `groups` groups)
static int64_t max_tiles(const aria_gemm_desc_t* d, int BN, int64_t groups) {
  const bool swiglu = d->epilogue == ARIA_EPI_SWIGLU;
  const int out_bn = swiglu ? BN / 2 : BN;
  const int64_t n_out_total = d->n * (swiglu ? 1 : d->n_seg);
  return (n_out_total + out_bn - 1) / out_bn * ((d->m + BM - 1) / BM + groups);
}

// aria_gemm, and grouped_gemm with b_scale != NULL (then d->b[0] is e4m3 and the GKN layout is the only one)
static int gemm_run(const aria_gemm_desc_t* d, const float* b_scale, cudaStream_t stream) {
  ARIA_CHECK_ARG(d != nullptr);
  ARIA_CHECK_ARG(d->a && d->b[0] && d->out[0]);
  ARIA_CHECK_ARG(d->m >= 0 && d->n > 0 && d->k > 0);
  ARIA_CHECK_ARG(d->n % 8 == 0 && d->k % 8 == 0 && d->lda % 8 == 0);
  ARIA_CHECK_ARG(d->n_seg >= 1 && d->n_seg <= 3);
  ARIA_CHECK_ARG(d->num_groups >= 1 && (d->group_mod >= 0 || d->num_groups % (-d->group_mod) == 0));
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(d->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->out[0]) & 15) == 0);
  if (d->m == 0) return ARIA_OK;
  const bool b_mn = d->b_layout == ARIA_B_GKN;
  const bool b_gnk = d->b_layout == ARIA_B_GNK;
  const bool swiglu = d->epilogue == ARIA_EPI_SWIGLU;
  if (b_mn) {
    ARIA_CHECK_ARG(d->n_seg == 1);
    // k-blocks must not straddle experts in the flattened [G*K, N] view (a single group has no neighbour: TMA zero-fills)
    ARIA_CHECK_ARG(d->k % BK == 0 || (d->num_groups == 1 && d->group_mod == 0));
    ARIA_CHECK_ARG(d->n % 64 == 0);
    ARIA_CHECK_ARG(d->epilogue != ARIA_EPI_HEADS);
  } else {
    ARIA_CHECK_ARG(d->num_groups == 1 || d->n_seg == 1);
    if (swiglu) ARIA_CHECK_ARG(d->n_seg == 2 && d->b[1]);
    if (b_gnk) ARIA_CHECK_ARG(d->n_seg == 1 && !swiglu && d->epilogue == ARIA_EPI_LINEAR && d->n % 128 == 0);
    else ARIA_CHECK_ARG(d->num_groups == 1);
  }
  if (d->num_groups > 1) ARIA_CHECK_ARG(d->group_offsets != nullptr);
  if (d->group_counts) ARIA_CHECK_ARG(d->group_offsets != nullptr);
  if (d->out_group_base) ARIA_CHECK_ARG(d->out_group_row0 != nullptr && d->epilogue == ARIA_EPI_LINEAR && d->group_offsets != nullptr);
  ARIA_CHECK_ARG(d->a_rows == 0 || d->a_rows >= d->m);

  // ---- tile shape selection: 128-wide tiles; the 72-dim ViT heads (n = 1152 = 8 x 144) take 144-wide tiles of whole heads
  int BN = 128;
  if (d->epilogue == ARIA_EPI_HEADS) {
    ARIA_CHECK_ARG(d->head_dim > 0 && d->head_dim % 8 == 0 && d->head_ld >= d->head_dim && d->n % d->head_dim == 0);
    if (d->rope_mask) ARIA_CHECK_ARG(d->head_dim == 128 && d->rope_cos && d->rope_sin);
    // the RoPE epilogue has no bias term: a rotated segment's bias would be dropped
    for (int s = 0; s < d->n_seg; ++s) ARIA_CHECK_ARG(!((d->rope_mask >> s) & 1) || !d->bias[s]);
    if (d->n % 128 != 0) {
      ARIA_CHECK_ARG(!d->rope_mask && d->n % 144 == 0);
      BN = 144;
    }
    for (int s = 0; s < d->n_seg; ++s) ARIA_CHECK_ARG(d->out[s] && d->b[s]);
  } else {
    if (swiglu) ARIA_CHECK_ARG(d->n % 64 == 0);
    if (d->n_seg > 1 && !swiglu) ARIA_CHECK_ARG(d->n % BN == 0);
  }

  // Dense bf16 GEMMs with nn.Linear weights and at least PAIR_MIN_ROWS rows, LINEAR or HEADS without RoPE (the ViT's four
  // GEMMs, the projector's 4,900-row k / v and in-projections) run on gemm_wide_kernel; tiles must not straddle two weights.
  // Measured on an H100 SXM at 700 W (DESIGN §6), µs before -> after: q/k/v heads 102.5 -> 83-85, o_proj 44.2 -> 34-36,
  // fc1 149-152 -> 127, fc2 122.5 -> 95-96; then with the hand-off epilogue q/k/v 83-85 -> 73-76 and fc1 124-125 -> 84-89.
  // Only fc2, whose 68 k-blocks make the mainloop the cost, gains from CTA pairs (95 against 105 µs); before the hand-off
  // o_proj, fc1 and the projector's k / v lost 10-25 % as pairs and q/k/v gained nothing, so pairs are selected for LINEAR
  // at K >= WIDE_PAIR_MIN_K only.  Other dense LINEAR launches of PAIR_MIN_ROWS rows and more (several
  // weights whose N is no multiple of 192) keep the 128-wide CTA pairs of gemm_kernel; the 768-row LM GEMMs lose 5-16 % as
  // pairs and keep the one-CTA kernel.
  const bool dense = !b_scale && d->b_layout == ARIA_B_NK && d->num_groups == 1 && !d->group_offsets;
  const bool wide = dense && d->m >= PAIR_MIN_ROWS && (d->n_seg == 1 || d->n % WIDE_BN == 0) &&
                    (d->epilogue == ARIA_EPI_HEADS ? !d->rope_mask : d->epilogue == ARIA_EPI_LINEAR);
  const bool wide_pair = wide && d->epilogue == ARIA_EPI_LINEAR && d->k >= WIDE_PAIR_MIN_K;
  const bool pair = !wide && dense && d->epilogue == ARIA_EPI_LINEAR && d->m >= PAIR_MIN_ROWS;
  const bool half_a = wide_pair || pair;

  CUtensorMap tmA, tmA_min, tmB[3];
  // a_rows: rows of the A buffer when groups live in fixed-capacity regions (m is then the EXPECTED row count that the
  // kernel-selection heuristics above use; the tensor map must cover the whole buffer).  Pairs: one box is a 64-row half.
  // Grouped launches also take the map with the small box (tma_load_a_rows).
  const uint64_t a_buf_rows = d->a_rows > 0 ? d->a_rows : d->m;
  int rc = make_tmap_2d(&tmA, d->a, d->k, a_buf_rows, d->lda * 2, BK, half_a ? BM / 2 : BM);
  if (rc) return rc;
  tmA_min = tmA;
  if (d->group_offsets) {
    rc = make_tmap_2d(&tmA_min, d->a, d->k, a_buf_rows, d->lda * 2, BK, A_BOX_MIN);
    if (rc) return rc;
  }
  if (b_mn) {
    const uint64_t ncols = swiglu ? 2 * d->n : d->n;
    const uint64_t n_weights = d->group_mod > 0 ? d->group_mod : (d->group_mod < 0 ? d->num_groups / (-d->group_mod) : d->num_groups);
    // fp8: byte map without swizzle, the 64-byte rows of a box land contiguously for the converters
    rc = b_scale ? make_tmap_2d(&tmB[0], d->b[0], ncols, n_weights * d->k, ncols, 64, BK, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_DATA_TYPE_UINT8)
                 : make_tmap_2d(&tmB[0], d->b[0], ncols, n_weights * d->k, ncols * 2, 64, BK);
    if (rc) return rc;
    tmB[1] = tmB[0];
    tmB[2] = tmB[0];
  } else {
    const int nb = swiglu ? 2 : d->n_seg;
    // rows of B staged per TMA box: the whole tile; SwiGLU splits gate | up
    const uint32_t box_rows = swiglu ? BN / 2 : (wide ? WIDE_BN : BN);
    for (int s = 0; s < 3; ++s) {
      const void* ptr = s < nb ? d->b[s] : d->b[0];
      const uint64_t b_rows = b_gnk ? static_cast<uint64_t>(d->group_mod > 0 ? d->group_mod : (d->group_mod < 0 ? d->num_groups / (-d->group_mod) : d->num_groups)) * d->n : d->n;
      rc = make_tmap_2d(&tmB[s], ptr, d->k, b_rows, d->k * 2, BK, box_rows);
      if (rc) return rc;
    }
  }

  const GemmParams p = gemm_params(d, b_scale);
  if (wide) {
    // out / residual: 64 x 64 boxes of the [m, n_seg n] row-major buffers
    CUtensorMap tmOut = tmA, tmRes = tmA;
    const uint64_t n_out = d->n * d->n_seg;
    if (d->epilogue == ARIA_EPI_LINEAR) {
      rc = make_tmap_2d(&tmOut, d->out[0], n_out, d->m, d->ldo * 2, 64, 64);
      if (rc) return rc;
      if (d->residual) {
        rc = make_tmap_2d(&tmRes, d->residual, n_out, d->m, d->ldr * 2, 64, 64);
        if (rc) return rc;
      }
    }
    const int64_t m_tiles = (d->m + BM - 1) / BM, n_tiles = (n_out + WIDE_BN - 1) / WIDE_BN;
    // the hand-off epilogue (gemm_wide_kernel's HANDOFF) for every launch without a residual
    if (wide_pair) {
      const int64_t pairs = (n_tiles + 1) / 2 * m_tiles;
      if (d->residual)
        return launch_persistent_pairs<gemm_wide_kernel<ARIA_EPI_LINEAR, true, false>>(
            "gemm_wide_kernel", GEMM_THREADS, gemm_wide_smem_bytes(), pairs, stream, tmA, tmB[0], tmB[1], tmB[2], tmOut, tmRes, p);
      return launch_persistent_pairs<gemm_wide_kernel<ARIA_EPI_LINEAR, true, true>>(
          "gemm_wide_kernel", GEMM_THREADS, gemm_wide_smem_bytes(), pairs, stream, tmA, tmB[0], tmB[1], tmB[2], tmOut, tmRes, p);
    }
#define ARIA_LAUNCH_WIDE(EPI_, HANDOFF_)                                                                                      \
  return launch_persistent<gemm_wide_kernel<EPI_, false, HANDOFF_>>("gemm_wide_kernel", GEMM_THREADS, gemm_wide_smem_bytes(), \
                                                                    n_tiles * m_tiles, stream, tmA, tmB[0], tmB[1], tmB[2],   \
                                                                    tmOut, tmRes, p)
    if (d->epilogue == ARIA_EPI_HEADS) ARIA_LAUNCH_WIDE(ARIA_EPI_HEADS, true);
    if (d->residual) ARIA_LAUNCH_WIDE(ARIA_EPI_LINEAR, false);
    ARIA_LAUNCH_WIDE(ARIA_EPI_LINEAR, true);
#undef ARIA_LAUNCH_WIDE
  }
  const int64_t tiles = max_tiles(d, BN, d->num_groups > 1 ? d->num_groups : 0);
  if (pair) {
    const int64_t m_tiles = (d->m + BM - 1) / BM, pairs = (tiles / m_tiles + 1) / 2 * m_tiles;
    return launch_persistent_pairs<gemm_kernel<128, false, ARIA_EPI_LINEAR, false, true>>(
        "gemm_kernel", GEMM_THREADS, gemm_smem_bytes<128>(), pairs, stream, tmA, tmA_min, tmB[0], tmB[1], tmB[2], p);
  }
#define ARIA_LAUNCH(BN_, MN_, EPI_, ...)                                                                                     \
  return launch_persistent<gemm_kernel<BN_, MN_, EPI_, ##__VA_ARGS__>>("gemm_kernel", GEMM_THREADS,                          \
                                                                       gemm_smem_bytes<BN_, ##__VA_ARGS__>(), tiles, stream, \
                                                                       tmA, tmA_min, tmB[0], tmB[1], tmB[2], p)
  if (b_scale) {
    if (swiglu) ARIA_LAUNCH(128, true, ARIA_EPI_SWIGLU, true);
    ARIA_LAUNCH(128, true, ARIA_EPI_LINEAR, true);
  }
  // the hand-off epilogue (gemm_kernel's HANDOFF) for the launches whose epilogue is long next to their tiles' mainloop: the
  // grouped expert GEMMs without a residual (fc1 + SwiGLU, fc2; expert-parallel regions and per-group destinations
  // included), dense SwiGLU (the shared experts' gate/up) and HEADS with RoPE (the LM's q/k/v).  Dense LINEAR launches and
  // the ViT / projector heads without RoPE below 2,048 rows keep the staged epilogue: their gain was not measured apart
  // from run-to-run noise (DESIGN §6).
#define ARIA_LAUNCH_HANDOFF(MN_, EPI_)                                                                                \
  return launch_persistent<gemm_handoff_kernel<MN_, EPI_>>("gemm_handoff_kernel", GEMM_THREADS,                      \
                                                           gemm_smem_bytes<128, false, false, handoff_stages(MN_)>(), \
                                                           tiles, stream, tmA, tmA_min, tmB[0], tmB[1], tmB[2], p)
  if (d->epilogue == ARIA_EPI_HEADS) {
    if (BN == 128 && d->rope_mask) ARIA_LAUNCH_HANDOFF(false, ARIA_EPI_HEADS);
    if (BN == 128) ARIA_LAUNCH(128, false, ARIA_EPI_HEADS);
    ARIA_LAUNCH(144, false, ARIA_EPI_HEADS);
  }
  if (swiglu) {
    if (b_mn) ARIA_LAUNCH_HANDOFF(true, ARIA_EPI_SWIGLU);
    ARIA_LAUNCH_HANDOFF(false, ARIA_EPI_SWIGLU);
  }
  if (d->group_offsets && !d->residual) {
    if (b_mn) ARIA_LAUNCH_HANDOFF(true, ARIA_EPI_LINEAR);
    ARIA_LAUNCH_HANDOFF(false, ARIA_EPI_LINEAR);
  }
  if (b_mn) ARIA_LAUNCH(128, true, ARIA_EPI_LINEAR);
  ARIA_LAUNCH(128, false, ARIA_EPI_LINEAR);
#undef ARIA_LAUNCH_HANDOFF
#undef ARIA_LAUNCH
}

extern "C" int aria_gemm(const aria_gemm_desc_t* d, aria_stream_t stream) {
  return gemm_run(d, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int aria::grouped_gemm(const void* a, const void* b, const float* b_scale, void* out, const int32_t* offsets, int64_t rows,
                       int64_t k, int64_t n, int32_t groups, int32_t epilogue, cudaStream_t stream) {
  const aria_gemm_desc_t d = grouped_desc(a, b, out, offsets, rows, k, n, groups, epilogue);
  return gemm_run(&d, b_scale, stream);
}

extern "C" int aria_grouped_gemm(const void* a, const void* b, void* out, const int32_t* group_offsets, int64_t rows,
                                 int64_t k, int64_t n, int32_t num_groups, aria_stream_t stream) {
  return grouped_gemm(a, b, nullptr, out, group_offsets, rows, k, n, num_groups, ARIA_EPI_LINEAR,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int aria_grouped_gemm_fp8(const void* a, const void* b_fp8, const float* b_scale, void* out,
                                     const int32_t* group_offsets, int64_t rows, int64_t k, int64_t n, int32_t num_groups,
                                     int32_t epilogue, aria_stream_t stream) {
  ARIA_CHECK_ARG(a && b_fp8 && b_scale && out && group_offsets);
  ARIA_CHECK_ARG(rows >= 0 && k > 0 && n > 0 && k % BK == 0 && n % 64 == 0 && num_groups >= 1);
  ARIA_CHECK_ARG(epilogue == ARIA_EPI_LINEAR || epilogue == ARIA_EPI_SWIGLU);
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(b_fp8) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(b_scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  return grouped_gemm(a, b_fp8, b_scale, out, group_offsets, rows, k, n, num_groups, epilogue,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int aria_grouped_gemm_w8a8(const void* a_fp8, const float* a_scale, const void* b_fp8_nk, const float* b_scale,
                                      void* out, const int32_t* group_offsets, int64_t rows, int64_t k, int64_t n,
                                      int32_t num_groups, int32_t epilogue, aria_stream_t stream_) {
  ARIA_CHECK_ARG(a_fp8 && a_scale && b_fp8_nk && b_scale && out && group_offsets);
  ARIA_CHECK_ARG(rows >= 0 && rows < (int64_t(1) << 31) && k > 0 && n > 0 && k % W8_BK == 0 && n % 64 == 0 && num_groups >= 1);
  ARIA_CHECK_ARG(k <= (1 << 30) && n <= (1 << 29) && static_cast<int64_t>(num_groups) * n * 2 < (int64_t(1) << 31));
  ARIA_CHECK_ARG(epilogue == ARIA_EPI_LINEAR || epilogue == ARIA_EPI_SWIGLU);
  ARIA_CHECK_ARG((reinterpret_cast<uintptr_t>(a_fp8) & 15) == 0 && (reinterpret_cast<uintptr_t>(b_fp8_nk) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(b_scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(a_scale) & 3) == 0);
  if (rows == 0) return ARIA_OK;
  const bool swiglu = epilogue == ARIA_EPI_SWIGLU;
  const aria_gemm_desc_t d = grouped_desc(a_fp8, b_fp8_nk, out, group_offsets, rows, k, n, num_groups, epilogue);
  const GemmParams p = gemm_params(&d, b_scale);

  // UINT8 maps, 128-byte swizzle: a box row is one 128-element k-block
  CUtensorMap tmA, tmA_min, tmB;  // A: the whole tile's box and the small one (tma_load_a_rows)
  int rc = make_tmap_2d(&tmA, a_fp8, k, rows, k, W8_BK, BM, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;
  rc = make_tmap_2d(&tmA_min, a_fp8, k, rows, k, W8_BK, A_BOX_MIN, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;
  rc = make_tmap_2d(&tmB, b_fp8_nk, k, num_groups * (swiglu ? 2 * n : n), k, W8_BK, 64, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;

  const int64_t tiles = max_tiles(&d, 128, num_groups);
  constexpr int SMEM = gemm_smem_bytes<128>();
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (swiglu)
    return launch_persistent<gemm_w8a8_kernel<ARIA_EPI_SWIGLU>>("gemm_w8a8_kernel", GEMM_THREADS, SMEM, tiles, stream, tmA,
                                                                 tmA_min, tmB, p, a_scale);
  return launch_persistent<gemm_w8a8_kernel<ARIA_EPI_LINEAR>>("gemm_w8a8_kernel", GEMM_THREADS, SMEM, tiles, stream, tmA,
                                                              tmA_min, tmB, p, a_scale);
}

extern "C" int aria_gemm_w8a8(const aria_gemm_desc_t* d, const float* a_scale, const float* const b_scale[3],
                              aria_stream_t stream_) {
  auto al = [](const void* ptr, uintptr_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) == 0; };
  ARIA_CHECK_ARG(d != nullptr && b_scale != nullptr);
  ARIA_CHECK_ARG(d->a && d->b[0] && d->out[0] && a_scale && b_scale[0]);
  ARIA_CHECK_ARG(d->b_layout == ARIA_B_NK && d->num_groups == 1 && d->group_mod == 0 && !d->group_offsets && !d->group_counts &&
                 !d->out_group_base && d->a_rows == 0);
  ARIA_CHECK_ARG(d->m >= 0 && d->m < (int64_t(1) << 31) && d->n > 0 && d->k > 0 && d->k <= (1 << 30) && d->n <= (1 << 29));
  ARIA_CHECK_ARG(d->k % W8_BK == 0 && d->n % 64 == 0 && d->lda >= d->k && d->lda % 16 == 0);
  ARIA_CHECK_ARG(d->n_seg >= 1 && d->n_seg <= 3);
  ARIA_CHECK_ARG(d->epilogue == ARIA_EPI_LINEAR || d->epilogue == ARIA_EPI_SWIGLU || d->epilogue == ARIA_EPI_HEADS);
  ARIA_CHECK_ARG(al(d->a, 16) && al(d->out[0], 16) && al(a_scale, 4));
  const bool swiglu = d->epilogue == ARIA_EPI_SWIGLU;
  const int nb = swiglu ? 2 : d->n_seg;  // weights (and scale vectors)
  if (swiglu) ARIA_CHECK_ARG(d->n_seg == 2);
  for (int s = 0; s < nb; ++s) ARIA_CHECK_ARG(d->b[s] && b_scale[s] && al(d->b[s], 16) && al(b_scale[s], 16));
  // LINEAR / HEADS tiles must not straddle two weights
  if (!swiglu && d->n_seg > 1) ARIA_CHECK_ARG(d->n % 128 == 0);
  if (d->epilogue == ARIA_EPI_HEADS) {
    ARIA_CHECK_ARG(d->n % 128 == 0 && d->head_dim > 0 && d->head_dim % 8 == 0 && d->head_ld >= d->head_dim &&
                   d->n % d->head_dim == 0);
    if (d->rope_mask) ARIA_CHECK_ARG(d->head_dim == 128 && d->rope_cos && d->rope_sin);
    for (int s = 0; s < d->n_seg; ++s) ARIA_CHECK_ARG(d->out[s] != nullptr && al(d->out[s], 16));
  } else {
    ARIA_CHECK_ARG(d->ldo % 8 == 0 && d->ldo >= (swiglu ? d->n : d->n * d->n_seg));
  }
  if (d->residual) ARIA_CHECK_ARG(d->epilogue == ARIA_EPI_LINEAR && al(d->residual, 16) && d->ldr % 8 == 0);
  if (d->m == 0) return ARIA_OK;

  // UINT8 maps, 128-byte swizzle: a box row is one 128-element k-block; each weight is its own [n, k] map
  CUtensorMap tmA, tmB[3];
  int rc = make_tmap_2d(&tmA, d->a, d->k, d->m, d->lda, W8_BK, BM, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
  if (rc) return rc;
  W8a8DenseScales sc{};
  for (int s = 0; s < 3; ++s) {
    const int src = s < nb ? s : 0;
    sc.b[s] = b_scale[src];
    rc = make_tmap_2d(&tmB[s], d->b[src], d->k, d->n, d->k, W8_BK, 64, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (rc) return rc;
  }
  const GemmParams p = gemm_params(d, nullptr);
  const int64_t tiles = max_tiles(d, 128, 0);
  constexpr int SMEM = gemm_smem_bytes<128>();
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
#define ARIA_LAUNCH(EPI_)                                                                                                      \
  return launch_persistent<gemm_w8a8_dense_kernel<EPI_>>("gemm_w8a8_dense_kernel", GEMM_THREADS, SMEM, tiles, stream, tmA, \
                                                          tmB[0], tmB[1], tmB[2], p, a_scale, sc)
  if (swiglu) ARIA_LAUNCH(ARIA_EPI_SWIGLU);
  if (d->epilogue == ARIA_EPI_HEADS) ARIA_LAUNCH(ARIA_EPI_HEADS);
  ARIA_LAUNCH(ARIA_EPI_LINEAR);
#undef ARIA_LAUNCH
}

extern "C" int aria_abi_version(void) { return 3; }
extern "C" const char* aria_build_arch(void) { return "sm_90a"; }
