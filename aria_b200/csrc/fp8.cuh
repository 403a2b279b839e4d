// e4m3 conversions shared by the quantisers (quant.cu, kv_fp8.cu) and the fp8 decode attention (attention.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>

namespace aria {

constexpr float E4M3_MAX = 448.f;

// 8 bf16 (one 16-byte chunk) / scale -> 8 e4m3 codes, low byte first; IEEE division, round to nearest even, saturating
__device__ __forceinline__ uint2 cast8_e4m3(const uint4 v, float s) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
  uint32_t packed[2] = {0u, 0u};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float x0 = __fdiv_rn(__uint_as_float(u[j] << 16), s);
    const float x1 = __fdiv_rn(__uint_as_float(u[j] & 0xFFFF0000u), s);
    const uint32_t pair = __nv_cvt_float2_to_fp8x2(make_float2(x0, x1), __NV_SATFINITE, __NV_E4M3);
    packed[j >> 1] |= (pair & 0xFFFFu) << (16 * (j & 1));
  }
  return make_uint2(packed[0], packed[1]);
}

// 4 e4m3 codes (low byte first) -> 4 floats, exactly: cvt.rn.f16x2.e4m3x2 widens two codes to f16 (every e4m3 value is an f16)
__device__ __forceinline__ float4 e4m3x4_to_float4(uint32_t u) {
  const __half2 lo(__nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(u & 0xFFFFu), __NV_E4M3));
  const __half2 hi(__nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(u >> 16), __NV_E4M3));
  const float2 a = __half22float2(lo), b = __half22float2(hi);
  return make_float4(a.x, a.y, b.x, b.y);
}

}  // namespace aria
