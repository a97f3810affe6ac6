// NF4 weight-only quantization of the decoder's layer matrices (DESIGN.md §3 "NF4 decode weights"): the format bitsandbytes'
// quantize_4bit(quant_type="nf4", blocksize=64, compress_statistics=True) produces, as the reference's load_4bit path loads the LLM
// (llava/model/builder.py:51-60), with the double-quantized absmax resolved to one fp32 scale per block of 64 weights.
//
// A weight's value is round_to_elem(fl32(CODE[q] * scale)): it is dequantized to the element type and then multiplied, as
// bitsandbytes' Linear4bit does, so the NF4 decode GEMV and the element-type GEMV over the dequantized matrix are bit-identical.
//
// Planes the decode GEMV streams (srgpt_nf4):
//   * q [N, K/2] bytes in the GEMV's lane order: lane l of a warp owns chunks (8 weights) c = l + 32 i of a row and takes them in
//     batches of 4 (1024 weights per row), so batch b of a row is 512 bytes, lane l's 16 bytes at b * 512 + 16 l, chunk i's 8 codes in
//     32-bit word i of them, weight t of the chunk in bits 4t .. 4t + 3.  K must be a multiple of 1024.
//   * scale [N, K/64] fp32 in natural order (one per block of 64 weights = 8 chunks).
// The quantizer's own intermediate, `codes` [N, K/2], is in natural order: weight 2j in the high nibble of byte j, 2j + 1 in the low.
#pragma once
#include "common.cuh"

namespace srgpt {
namespace nf4 {

constexpr int BLOCK = 64;    // weights per absmax / scale
constexpr int BLOCK2 = 256;  // absmax values per second-level (double-quantization) scale
constexpr int BATCH = 1024;  // weights per row and GEMV batch

// the 16 NF4 values of QLoRA / bitsandbytes (fp32)
__host__ __device__ __forceinline__ float code_value(int i) {
  switch (i) {
    case 0: return -1.0f;
    case 1: return -0.6961928009986877f;
    case 2: return -0.5250730514526367f;
    case 3: return -0.39491748809814453f;
    case 4: return -0.28444138169288635f;
    case 5: return -0.18477343022823334f;
    case 6: return -0.09105003625154495f;
    case 7: return 0.0f;
    case 8: return 0.07958029955625534f;
    case 9: return 0.16093020141124725f;
    case 10: return 0.24611230194568634f;
    case 11: return 0.33791524171829224f;
    case 12: return 0.44070982933044434f;
    case 13: return 0.5626170039176941f;
    case 14: return 0.7229568362236023f;
    default: return 1.0f;
  }
}

// byte offset of chunk cc's 32-bit code word inside its row of the q plane
__host__ __device__ __forceinline__ int lane_offset(int cc) { return (cc >> 7) * 512 + (cc & 31) * 16 + ((cc >> 5) & 3) * 4; }

// the 8 weights of one chunk as element-type pairs in the layout unpack8 reads: tab = the 16 code values in shared memory (entry i in
// bank i, so the lanes' lookups never conflict), s = the chunk's scale
__device__ __forceinline__ uint4 dequant8(uint32_t word, float s, const float* tab) {
  float f[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) f[t] = __fmul_rn(tab[(word >> (4 * t)) & 15u], s);
  return pack8(f);
}

}  // namespace nf4
}  // namespace srgpt
