// The fp8 KV cache (moe_lm.KVCache(dtype="fp8")): e4m3 codes [B, H, T_max, 128] with one fp32 scale per (row, head, token).
//
//   scale = max |x| / 448   (IEEE division; an all-zero row gets scale 1)
//   code  = e4m3(x / scale) (IEEE division, round to nearest even, saturating)
//
// bit for bit `(x.float() / scale[..., None]).to(torch.float8_e4m3fn)`, the rule of quant.cu's quantisers.
//
// aria_kv_store_fp8: quantises bf16 rows [0, n) of a source into cache rows [row0, row0 + n) (prefill, host positions).
// aria_kv_append_fp8: quantises one bf16 row per (b, h) into cache row pos[b] (device positions, the captured decode step).
// aria_kv_load_fp8: dequantises cache rows [0, n) into bf16, bf16(code * scale) (a multi-token continuation attends bf16 K/V).
// aria_kv_append_paged_fp8 / aria_kv_pages_store_varlen_fp8 / aria_kv_pages_load_fp8: the same quantiser and dequantiser over
// the page pools of serving.Engine's fp8 KV pages (codes [n_pages, H, 256, 128], scales [n_pages, H, 256]).
//
// One half-warp per 128-wide row, 8 values per lane; a block covers 4 rows of k and the same 4 rows of v.
#include <cuda_bf16.h>

#include "common.cuh"
#include "fp8.cuh"
#include "ptx.cuh"

namespace aria {

constexpr int KVQ_D = 128;
constexpr int KVQ_ROWS = 4;  // rows per 128-thread block: warp w takes row w, its low half-warp k and its high half-warp v

// The one quantiser of every entry: lane j (of 16) holds elements [8j, 8j + 8) of the row -> its 8 codes and the row's scale s
__device__ __forceinline__ uint2 quantize8_e4m3(const uint4 v, float& s) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) m = fmaxf(m, fmaxf(fabsf(__uint_as_float(u[i] << 16)), fabsf(__uint_as_float(u[i] & 0xFFFF0000u))));
  const unsigned half = 0xFFFFu << (threadIdx.x & 16);
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(half, m, o));
  s = m > 0.f ? __fdiv_rn(m, E4M3_MAX) : 1.f;
  return cast8_e4m3(v, s);
}

__device__ __forceinline__ void quantize_row_e4m3(const __nv_bfloat16* __restrict__ src, uint8_t* __restrict__ dst,
                                                  float* __restrict__ scale, int j) {
  float s;
  *reinterpret_cast<uint2*>(dst + 8 * j) = quantize8_e4m3(*reinterpret_cast<const uint4*>(src + 8 * j), s);
  if (j == 0) *scale = s;
}

// The one dequantiser: 8 codes of scale s -> 8 bf16 values bf16(code * s)
__device__ __forceinline__ uint4 dequantize8_e4m3(const uint2 c, float s) {
  const float4 lo = e4m3x4_to_float4(c.x), hi = e4m3x4_to_float4(c.y);
  uint4 o;
  o.x = pack_bf16(lo.x * s, lo.y * s);
  o.y = pack_bf16(lo.z * s, lo.w * s);
  o.z = pack_bf16(hi.x * s, hi.y * s);
  o.w = pack_bf16(hi.z * s, hi.w * s);
  return o;
}

// DEV_POS: cache row pos[b] of source row 0 (n = 1); otherwise cache row row0 + r of source row r
template <bool DEV_POS>
__global__ void __launch_bounds__(32 * KVQ_ROWS) kv_quant_kernel(const __nv_bfloat16* __restrict__ k_src,
                                                                 const __nv_bfloat16* __restrict__ v_src, int64_t s_sb, int64_t s_sh,
                                                                 uint8_t* __restrict__ kc, uint8_t* __restrict__ vc,
                                                                 float* __restrict__ ks, float* __restrict__ vs, int64_t c_sb,
                                                                 int64_t c_sh, int64_t sc_sb, int64_t sc_sh,
                                                                 const int32_t* __restrict__ pos, int row0, int n, int H, int T_max) {
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int r = blockIdx.y * KVQ_ROWS + (threadIdx.x >> 5);
  if (r >= n) return;
  const int t = DEV_POS ? pos[b] : row0 + r;
  if (t < 0 || t >= T_max) return;  // never past the cache
  const bool is_v = threadIdx.x & 16;
  const __nv_bfloat16* src = (is_v ? v_src : k_src) + b * s_sb + h * s_sh + static_cast<int64_t>(r) * KVQ_D;
  uint8_t* dst = (is_v ? vc : kc) + b * c_sb + h * c_sh + static_cast<int64_t>(t) * KVQ_D;
  float* sc = (is_v ? vs : ks) + b * sc_sb + h * sc_sh + t;
  quantize_row_e4m3(src, dst, sc, threadIdx.x & 15);
}

__global__ void __launch_bounds__(32 * KVQ_ROWS) kv_load_kernel(const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc,
                                                                const float* __restrict__ ks, const float* __restrict__ vs,
                                                                int64_t c_sb, int64_t c_sh, int64_t sc_sb, int64_t sc_sh,
                                                                __nv_bfloat16* __restrict__ k_out, __nv_bfloat16* __restrict__ v_out,
                                                                int64_t o_sb, int64_t o_sh, int n, int H) {
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int r = blockIdx.y * KVQ_ROWS + (threadIdx.x >> 5);
  if (r >= n) return;
  const bool is_v = threadIdx.x & 16;
  const int j = threadIdx.x & 15;
  const uint2 c = *reinterpret_cast<const uint2*>((is_v ? vc : kc) + b * c_sb + h * c_sh + static_cast<int64_t>(r) * KVQ_D + 8 * j);
  const float s = (is_v ? vs : ks)[b * sc_sb + h * sc_sh + r];
  *reinterpret_cast<uint4*>((is_v ? v_out : k_out) + b * o_sb + h * o_sh + static_cast<int64_t>(r) * KVQ_D + 8 * j) =
      dequantize8_e4m3(c, s);
}

// Paged fp8 pools (serving.Engine with kv_cache_dtype="fp8"): codes [n_pages, H, 256, 128] at (page_stride, pool_sh), scales
// [n_pages, H, 256] at (sc_page_stride, sc_sh).  One warp per (row t, head h) item, its low half-warp k and its high half v.
// VARLEN: item row t is packed row t of segment b, position prefix_lens[b] + t - cu[b] of its request (the varlen store); the
// dequantised values bf16(code * scale) are written back over every source row.  Otherwise (the append) row t is slot t, at
// position pos[t].  No page is written for an unmapped position, a table entry outside the pool, or the null page 0.
template <bool VARLEN>
__global__ void __launch_bounds__(32 * KVQ_ROWS) kv_quant_paged_kernel(
    __nv_bfloat16* __restrict__ k_src, __nv_bfloat16* __restrict__ v_src, int64_t s_sb, int64_t s_sh, uint8_t* __restrict__ kp,
    uint8_t* __restrict__ vp, float* __restrict__ ks, float* __restrict__ vs, int64_t page_stride, int64_t pool_sh,
    int64_t sc_page_stride, int64_t sc_sh, const int32_t* __restrict__ table, int64_t table_stride, int max_pages, int n_pages,
    const int32_t* __restrict__ pos, const int32_t* __restrict__ cu, int n_seg, int n_items, int H) {
  const int item = blockIdx.x * KVQ_ROWS + (threadIdx.x >> 5);
  if (item >= n_items) return;
  const int t = item / H, h = item % H;
  int row, p;
  if constexpr (VARLEN) {
    row = packed_segment(cu, n_seg, t);
    p = pos[row] + t - cu[row];
  } else {
    row = t;
    p = pos[t];
  }
  const int page = page_of(table + row * table_stride, max_pages, n_pages, p);
  if (!VARLEN && page <= 0) return;
  const bool is_v = threadIdx.x & 16;
  const int j = threadIdx.x & 15;
  __nv_bfloat16* src = (is_v ? v_src : k_src) + t * s_sb + h * s_sh + 8 * j;
  float s;
  const uint2 c = quantize8_e4m3(*reinterpret_cast<const uint4*>(src), s);
  if (page > 0) {  // not unmapped, outside the pool, or the null page
    const int r = p % PAGE_ROWS;
    *reinterpret_cast<uint2*>((is_v ? vp : kp) + page * page_stride + h * pool_sh + static_cast<int64_t>(r) * KVQ_D + 8 * j) = c;
    if (j == 0) (is_v ? vs : ks)[page * sc_page_stride + h * sc_sh + r] = s;
  }
  if constexpr (VARLEN) *reinterpret_cast<uint4*>(src) = dequantize8_e4m3(c, s);
}

// Page pages[i] of the fp8 pools -> page i of the bf16 pools out [n_list, H, 256, 128] (out_page_stride, out_sh), with the
// dequantiser of kv_load_kernel; an entry outside [0, n_pages) gives zeros.  Block (i * H + h, 4 rows).
__global__ void __launch_bounds__(32 * KVQ_ROWS) kv_pages_load_kernel(
    const uint8_t* __restrict__ kp, const uint8_t* __restrict__ vp, const float* __restrict__ ks, const float* __restrict__ vs,
    int64_t page_stride, int64_t pool_sh, int64_t sc_page_stride, int64_t sc_sh, const int32_t* __restrict__ pages, int n_pages,
    __nv_bfloat16* __restrict__ k_out, __nv_bfloat16* __restrict__ v_out, int64_t out_page_stride, int64_t out_sh, int H) {
  const int i = blockIdx.x / H, h = blockIdx.x % H;
  const int r = blockIdx.y * KVQ_ROWS + (threadIdx.x >> 5);
  const bool is_v = threadIdx.x & 16;
  const int j = threadIdx.x & 15;
  const int page = pages[i];
  uint4 o = make_uint4(0u, 0u, 0u, 0u);
  if (page >= 0 && page < n_pages) {
    const uint2 c = *reinterpret_cast<const uint2*>((is_v ? vp : kp) + page * page_stride + h * pool_sh +
                                                     static_cast<int64_t>(r) * KVQ_D + 8 * j);
    o = dequantize8_e4m3(c, (is_v ? vs : ks)[page * sc_page_stride + h * sc_sh + r]);
  }
  *reinterpret_cast<uint4*>((is_v ? v_out : k_out) + i * out_page_stride + h * out_sh + static_cast<int64_t>(r) * KVQ_D + 8 * j) = o;
}

// what all three entries require of the cache: e4m3 rows of 16-byte alignment and non-negative scale strides
static bool cache_args_ok(const void* kc, const void* vc, const float* ks, const float* vs, int64_t c_sb, int64_t c_sh,
                          int64_t sc_sb, int64_t sc_sh, int32_t B, int32_t H, int32_t T_max) {
  return kc && vc && ks && vs && c_sb % 16 == 0 && c_sh % 16 == 0 && sc_sb >= 0 && sc_sh >= 0 && B > 0 && H > 0 && T_max > 0 &&
         static_cast<int64_t>(B) * H < (1ll << 31);
}

// what the paged entries require of the pools: 16-byte code rows, pages that do not overlap, and scale strides to match
static bool pool_args_ok(const void* kp, const void* vp, const float* ks, const float* vs, int64_t page_stride, int64_t pool_sh,
                         int64_t sc_page_stride, int64_t sc_sh, int32_t n_pages, int32_t H) {
  return kp && vp && ks && vs && n_pages > 0 && H > 0 && page_stride % 16 == 0 && pool_sh % 16 == 0 &&
         pool_sh >= PAGE_ROWS * KVQ_D && page_stride >= pool_sh * H && sc_sh >= PAGE_ROWS && sc_page_stride >= sc_sh * H;
}

}  // namespace aria

using namespace aria;

extern "C" int aria_kv_store_fp8(const void* k_src, const void* v_src, int64_t src_stride_b, int64_t src_stride_h, void* k_cache,
                                 void* v_cache, float* k_scale, float* v_scale, int64_t cache_stride_b, int64_t cache_stride_h,
                                 int64_t scale_stride_b, int64_t scale_stride_h, int32_t row0, int32_t n_rows, int32_t B, int32_t H,
                                 int32_t T_max, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_src && v_src && src_stride_b % 8 == 0 && src_stride_h % 8 == 0);
  ARIA_CHECK_ARG(cache_args_ok(k_cache, v_cache, k_scale, v_scale, cache_stride_b, cache_stride_h, scale_stride_b, scale_stride_h, B,
                               H, T_max));
  ARIA_CHECK_ARG(row0 >= 0 && n_rows > 0 && n_rows <= T_max - row0);
  dim3 grid(B * H, (n_rows + KVQ_ROWS - 1) / KVQ_ROWS);
  ARIA_CHECK_ARG(grid.y <= 65535);
  kv_quant_kernel<false><<<grid, 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k_src), static_cast<const __nv_bfloat16*>(v_src), src_stride_b, src_stride_h,
      static_cast<uint8_t*>(k_cache), static_cast<uint8_t*>(v_cache), k_scale, v_scale, cache_stride_b, cache_stride_h,
      scale_stride_b, scale_stride_h, nullptr, row0, n_rows, H, T_max);
  return check_launch("kv_quant_kernel");
}

extern "C" int aria_kv_append_fp8(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h, void* k_cache,
                                  void* v_cache, float* k_scale, float* v_scale, int64_t cache_stride_b, int64_t cache_stride_h,
                                  int64_t scale_stride_b, int64_t scale_stride_h, const int32_t* pos, int32_t B, int32_t H,
                                  int32_t T_max, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_new && v_new && pos && new_stride_b % 8 == 0 && new_stride_h % 8 == 0);
  ARIA_CHECK_ARG(cache_args_ok(k_cache, v_cache, k_scale, v_scale, cache_stride_b, cache_stride_h, scale_stride_b, scale_stride_h, B,
                               H, T_max));
  kv_quant_kernel<true><<<dim3(B * H, 1), 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(k_new), static_cast<const __nv_bfloat16*>(v_new), new_stride_b, new_stride_h,
      static_cast<uint8_t*>(k_cache), static_cast<uint8_t*>(v_cache), k_scale, v_scale, cache_stride_b, cache_stride_h,
      scale_stride_b, scale_stride_h, pos, 0, 1, H, T_max);
  return check_launch("kv_quant_kernel");
}

extern "C" int aria_kv_load_fp8(const void* k_cache, const void* v_cache, const float* k_scale, const float* v_scale,
                                int64_t cache_stride_b, int64_t cache_stride_h, int64_t scale_stride_b, int64_t scale_stride_h,
                                void* k_out, void* v_out, int64_t out_stride_b, int64_t out_stride_h, int32_t n_rows, int32_t B,
                                int32_t H, int32_t T_max, aria_stream_t stream_) {
  ARIA_CHECK_ARG(cache_args_ok(k_cache, v_cache, k_scale, v_scale, cache_stride_b, cache_stride_h, scale_stride_b, scale_stride_h, B,
                               H, T_max));
  ARIA_CHECK_ARG(k_out && v_out && out_stride_b % 8 == 0 && out_stride_h % 8 == 0);
  ARIA_CHECK_ARG(n_rows > 0 && n_rows <= T_max);
  dim3 grid(B * H, (n_rows + KVQ_ROWS - 1) / KVQ_ROWS);
  ARIA_CHECK_ARG(grid.y <= 65535);
  kv_load_kernel<<<grid, 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint8_t*>(k_cache), static_cast<const uint8_t*>(v_cache), k_scale, v_scale, cache_stride_b, cache_stride_h,
      scale_stride_b, scale_stride_h, static_cast<__nv_bfloat16*>(k_out), static_cast<__nv_bfloat16*>(v_out), out_stride_b,
      out_stride_h, n_rows, H);
  return check_launch("kv_load_kernel");
}

extern "C" int aria_kv_append_paged_fp8(const void* k_new, const void* v_new, int64_t new_stride_b, int64_t new_stride_h,
                                        void* k_pool, void* v_pool, float* k_scale, float* v_scale, int64_t page_stride,
                                        int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h,
                                        const int32_t* block_table, int64_t block_table_stride, int32_t max_pages, int32_t n_pages,
                                        const int32_t* write_pos, int32_t R, int32_t H, aria_stream_t stream_) {
  ARIA_CHECK_ARG(k_new && v_new && block_table && write_pos && new_stride_b % 8 == 0 && new_stride_h % 8 == 0);
  ARIA_CHECK_ARG(pool_args_ok(k_pool, v_pool, k_scale, v_scale, page_stride, pool_stride_h, scale_page_stride, scale_stride_h,
                              n_pages, H));
  ARIA_CHECK_ARG(R > 0 && max_pages > 0 && block_table_stride >= max_pages);
  ARIA_CHECK_ARG(static_cast<int64_t>(R) * H < (1ll << 31) && static_cast<int64_t>(R) * block_table_stride < (1ll << 31));
  const int items = R * H;
  kv_quant_paged_kernel<false><<<(items + KVQ_ROWS - 1) / KVQ_ROWS, 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      const_cast<__nv_bfloat16*>(static_cast<const __nv_bfloat16*>(k_new)),
      const_cast<__nv_bfloat16*>(static_cast<const __nv_bfloat16*>(v_new)), new_stride_b, new_stride_h,
      static_cast<uint8_t*>(k_pool), static_cast<uint8_t*>(v_pool), k_scale, v_scale, page_stride, pool_stride_h, scale_page_stride,
      scale_stride_h, block_table, block_table_stride, max_pages, n_pages, write_pos, nullptr, 0, items, H);
  return check_launch("kv_quant_paged_kernel");
}

extern "C" int aria_kv_pages_store_varlen_fp8(void* k, void* v, int64_t src_stride_h, int32_t S_tot, void* k_pool, void* v_pool,
                                              float* k_scale, float* v_scale, int64_t page_stride, int64_t pool_stride_h,
                                              int64_t scale_page_stride, int64_t scale_stride_h, const int32_t* page_table,
                                              int64_t page_table_stride, int32_t max_pages, int32_t n_pages,
                                              const int32_t* prefix_lens, const int32_t* cu_seqlens, int32_t n_seg, int32_t H,
                                              aria_stream_t stream_) {
  ARIA_CHECK_ARG(k && v && page_table && prefix_lens && cu_seqlens);
  ARIA_CHECK_ARG(pool_args_ok(k_pool, v_pool, k_scale, v_scale, page_stride, pool_stride_h, scale_page_stride, scale_stride_h,
                              n_pages, H));
  ARIA_CHECK_ARG(S_tot >= n_seg && n_seg > 0 && max_pages > 0 && page_table_stride >= max_pages);
  ARIA_CHECK_ARG(static_cast<int64_t>(S_tot) * H < (1ll << 31) && src_stride_h >= static_cast<int64_t>(S_tot) * KVQ_D);
  ARIA_CHECK_ARG(static_cast<int64_t>(n_seg) * page_table_stride < (1ll << 31) && src_stride_h % 8 == 0);
  const int items = S_tot * H;
  kv_quant_paged_kernel<true><<<(items + KVQ_ROWS - 1) / KVQ_ROWS, 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<__nv_bfloat16*>(k), static_cast<__nv_bfloat16*>(v), KVQ_D, src_stride_h, static_cast<uint8_t*>(k_pool),
      static_cast<uint8_t*>(v_pool), k_scale, v_scale, page_stride, pool_stride_h, scale_page_stride, scale_stride_h, page_table,
      page_table_stride, max_pages, n_pages, prefix_lens, cu_seqlens, n_seg, items, H);
  return check_launch("kv_quant_paged_kernel");
}

extern "C" int aria_kv_pages_load_fp8(const void* k_pool, const void* v_pool, const float* k_scale, const float* v_scale,
                                      int64_t page_stride, int64_t pool_stride_h, int64_t scale_page_stride, int64_t scale_stride_h,
                                      const int32_t* pages, int32_t n_list, int32_t n_pages, void* k_out, void* v_out,
                                      int64_t out_page_stride, int64_t out_stride_h, int32_t H, aria_stream_t stream_) {
  ARIA_CHECK_ARG(pool_args_ok(k_pool, v_pool, k_scale, v_scale, page_stride, pool_stride_h, scale_page_stride, scale_stride_h,
                              n_pages, H));
  ARIA_CHECK_ARG(pages && k_out && v_out && n_list > 0 && static_cast<int64_t>(n_list) * H < (1ll << 31));
  ARIA_CHECK_ARG(out_stride_h % 8 == 0 && out_page_stride % 8 == 0 && out_stride_h >= PAGE_ROWS * KVQ_D &&
                 out_page_stride >= out_stride_h * H);
  kv_pages_load_kernel<<<dim3(n_list * H, PAGE_ROWS / KVQ_ROWS), 32 * KVQ_ROWS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint8_t*>(k_pool), static_cast<const uint8_t*>(v_pool), k_scale, v_scale, page_stride, pool_stride_h,
      scale_page_stride, scale_stride_h, pages, n_pages, static_cast<__nv_bfloat16*>(k_out), static_cast<__nv_bfloat16*>(v_out),
      out_page_stride, out_stride_h, H);
  return check_launch("kv_pages_load_kernel");
}
