// Lossless 12-bit packing of bf16 weight matrices for the batch-1 decode GEMV (DESIGN.md §3 "Packed decode weights").
//
// A bf16 weight is sign (1) | exponent (8) | mantissa (7).  The exponents of one weight row sit in a narrow band, so a row
// keeps a base and each weight a 4-bit exponent code:
//   * sm plane, 1 byte per weight: sign << 7 | mantissa;
//   * ex plane, 4 bits per weight: code 0 = exponent field 0 (±0, subnormals), code c in 1..15 = exponent base + c - 1, with
//     base = max(1, row_max_exponent - 14);
//   * exceptions: a weight whose nonzero exponent lies below the window is stored with code 0, and (column << 8 | exponent)
//     goes into a per-row CSR list sorted by column, at most MAX_EXC_PER_ROW entries per row.
// The planes are laid out for the GEMV's lanes (gemv.cu): lane l of a warp owns chunks (8 weights) c = l + 32 i of a row and
// takes them in steps of 4 (a "batch" of 128 chunks = 1024 weights per row), so K must be a multiple of 1024.  Inside a batch,
// the sm bytes of a lane's chunks i = 0,1 and i = 2,3 are each one 16-byte vector, and its 4 ex words are one 16-byte vector:
// every load is a coalesced 512-byte warp access, 48 bytes per lane and row instead of 64.
#pragma once
#include "common.cuh"

namespace srgpt {
namespace pack12 {

constexpr int BATCH = 1024;          // weights per row and batch
constexpr int MAX_EXC_PER_ROW = 32;  // the GEMV keeps a row's exception list in one register per lane

// byte offset of chunk cc (weights 8 cc .. 8 cc + 7) inside its row of the sm plane (K bytes per row) ...
__host__ __device__ __forceinline__ int sm_offset(int cc) {
  return (cc >> 7) * 1024 + ((cc >> 6) & 1) * 512 + (cc & 31) * 16 + ((cc >> 5) & 1) * 8;
}
// ... and of its 32-bit code word inside its row of the ex plane (K / 2 bytes per row)
__host__ __device__ __forceinline__ int ex_offset(int cc) { return (cc >> 7) * 512 + (cc & 31) * 16 + ((cc >> 5) & 3) * 4; }
// weight t of a chunk: sm byte t of the chunk's 8, code in nibble nibble_of(t) of its word (the order decode_chunk needs)
__host__ __device__ __forceinline__ int nibble_of(int t) { return ((t & 1) << 2) | (t & 2) | (t >> 2); }

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(a), "r"(sel));
  return r;
}

// (a & 0x807F807F) | (b & 0x7F807F80) as one LOP3: sign and mantissa bits of two bf16 from a, exponent fields from b
__device__ __forceinline__ uint32_t merge_fields(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, 0x807F807F, 0xE4;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// The 8 weights of one chunk as bf16 pairs in the layout unpack8 reads: s_lo / s_hi = sm bytes of weights 0-3 / 4-7,
// e = the chunk's code word, bp = base - 1 of the row.  Code 0 yields exponent field 0; exceptions are patched afterwards.
// Per weight pair: one PRMT (sm byte into the low byte of the bf16 and its sign replicated over the high byte), one
// shift of the exponent bytes and one LOP3 that merges the two; per chunk 11 more for the code -> exponent step.
__device__ __forceinline__ uint4 decode_chunk(uint32_t s_lo, uint32_t s_hi, uint32_t e, uint32_t bp) {
  uint32_t x0 = e & 0x0F0F0F0Fu;         // bytes: codes of weights 0, 2, 1, 3
  uint32_t x1 = (e >> 4) & 0x0F0F0F0Fu;  // bytes: codes of weights 4, 6, 5, 7
  // + bp in every byte whose code is nonzero (code + 0x7F sets bit 7 exactly then; no byte carries: code + bp <= 254)
  x0 += (((x0 + 0x7F7F7F7Fu) >> 7) & 0x01010101u) * bp;
  x1 += (((x1 + 0x7F7F7F7Fu) >> 7) & 0x01010101u) * bp;
  uint4 w;
  w.x = merge_fields(prmt(s_lo, 0x9180u), x0 << 7);
  w.y = merge_fields(prmt(s_lo, 0xB3A2u), x0 >> 1);
  w.z = merge_fields(prmt(s_hi, 0x9180u), x1 << 7);
  w.w = merge_fields(prmt(s_hi, 0xB3A2u), x1 >> 1);
  return w;
}

}  // namespace pack12
}  // namespace srgpt
