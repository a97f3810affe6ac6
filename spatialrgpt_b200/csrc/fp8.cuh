// E4M3 conversions of the FP8 W8A8 linears (fp8.cu's row quantizer, gemv.cu's FP8 decode GEMV; the definition: include/srgpt_b200.h
// srgpt_fp8).
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

namespace srgpt {
namespace fp8 {

// inv = 448 / a and the row scale a / 448 of a row whose max |x| is a (both 1 for an all-zero row)
__device__ __forceinline__ void row_scales(float a, float& inv, float& scale) {
  inv = a > 0.f ? __fdiv_rn(448.0f, a) : 1.0f;
  scale = a > 0.f ? __fdiv_rn(a, 448.0f) : 1.0f;
}

// two floats -> two E4M3 codes (round to nearest even, saturated to +-448), x in the low byte
__device__ __forceinline__ uint32_t e4m3x2(float x, float y) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(x, y), __NV_SATFINITE, __NV_E4M3);
}

// two E4M3 codes (the low 16 bits, the first in the low byte) -> their values as an element-type pair (exact: both element types hold
// every E4M3 value), the first in the low half
__device__ __forceinline__ uint32_t e4m3x2_to_elem2(uint32_t codes) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(codes & 0xffffu), __NV_E4M3);
#ifdef SRGPT_ELEM_F16
  return (uint32_t)h.x | ((uint32_t)h.y << 16);
#else
  return pack_bf16x2(__half2float(__ushort_as_half(h.x)), __half2float(__ushort_as_half(h.y)));
#endif
}

// 16 E4M3 codes (one 16-byte vector, code t in byte t) -> two element-type chunks of 8 weights
__device__ __forceinline__ void e4m3x16_to_elem(const uint4& v, uint4& lo, uint4& hi) {
  lo = make_uint4(e4m3x2_to_elem2(v.x), e4m3x2_to_elem2(v.x >> 16), e4m3x2_to_elem2(v.y), e4m3x2_to_elem2(v.y >> 16));
  hi = make_uint4(e4m3x2_to_elem2(v.z), e4m3x2_to_elem2(v.z >> 16), e4m3x2_to_elem2(v.w), e4m3x2_to_elem2(v.w >> 16));
}

}  // namespace fp8
}  // namespace srgpt
