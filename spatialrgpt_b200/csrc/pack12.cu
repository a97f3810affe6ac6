// Load-time kernels of the 12-bit decode weight packing (format: pack12.cuh).  One warp per row throughout.
#include "pack12.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace pack12 {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

__device__ __forceinline__ int exp_field(uint32_t bits16) { return (int)((bits16 >> 7) & 0xFFu); }
__device__ __forceinline__ uint32_t half_of(const uint4& v, int t) {
  const uint32_t w = t < 2 ? v.x : (t < 4 ? v.y : (t < 6 ? v.z : v.w));
  return (t & 1) ? (w >> 16) : (w & 0xFFFFu);
}

// per row: base, number of exceptions; *n_bad += rows holding Inf / NaN
__global__ void __launch_bounds__(THREADS) scan_kernel(const bf16* __restrict__ W, int ldw, int N, int K, uint8_t* __restrict__ base,
                                                       int* __restrict__ n_exc, int* __restrict__ n_bad) {
  const int r = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= N) return;
  const uint4* row = reinterpret_cast<const uint4*>(W + (size_t)r * ldw);
  const int nchunk = K >> 3;
  int mx = 0;
  for (int c = lane; c < nchunk; c += 32) {
    const uint4 v = row[c];
#pragma unroll
    for (int t = 0; t < 8; ++t) mx = max(mx, exp_field(half_of(v, t)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const int b = max(1, mx - 14);
  int n = 0;
  for (int c = lane; c < nchunk; c += 32) {
    const uint4 v = row[c];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int e = exp_field(half_of(v, t));
      n += (e != 0 && e < b) ? 1 : 0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if (lane == 0) {
    base[r] = (uint8_t)min(b, 255);
    n_exc[r] = n;
    if (mx == 255) atomicAdd(n_bad, 1);
  }
}

__global__ void __launch_bounds__(THREADS) pack_kernel(const bf16* __restrict__ W, int ldw, int N, int K, const uint8_t* __restrict__ base,
                                                       const int* __restrict__ row_ptr, uint8_t* __restrict__ sm, uint8_t* __restrict__ ex,
                                                       int* __restrict__ exc) {
  const int r = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= N) return;
  const uint4* row = reinterpret_cast<const uint4*>(W + (size_t)r * ldw);
  uint8_t* sm_row = sm + (size_t)r * K;
  uint8_t* ex_row = ex + (size_t)r * (K >> 1);
  const int b = base[r];
  int next = row_ptr[r];  // exceptions are appended in column order: chunk by chunk, lanes in order within a step of 32 chunks
  for (int c0 = 0; c0 < (K >> 3); c0 += 32) {
    const int c = c0 + lane;
    const uint4 v = row[c];
    uint32_t s[2] = {0u, 0u}, code_word = 0u;
    int n = 0;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const uint32_t h = half_of(v, t);
      const int e = exp_field(h);
      s[t >> 2] |= (((h >> 8) & 0x80u) | (h & 0x7Fu)) << (8 * (t & 3));
      if (e >= b) code_word |= (uint32_t)(e - b + 1) << (4 * nibble_of(t));
      else if (e != 0) ++n;
    }
    *reinterpret_cast<uint2*>(sm_row + sm_offset(c)) = make_uint2(s[0], s[1]);
    *reinterpret_cast<uint32_t*>(ex_row + ex_offset(c)) = code_word;
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    int at = next + incl - n;
    if (n > 0) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int e = exp_field(half_of(v, t));
        if (e != 0 && e < b) exc[at++] = ((8 * c + t) << 8) | e;
      }
    }
    next += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// the inverse, through the GEMV's own decode_chunk; exceptions are written after a __syncwarp by whichever lane reads them
__global__ void __launch_bounds__(THREADS) unpack_kernel(const uint8_t* __restrict__ sm, const uint8_t* __restrict__ ex, const uint8_t* __restrict__ base,
                                                         const int* __restrict__ row_ptr, const int* __restrict__ exc, int N, int K, bf16* __restrict__ W,
                                                         int ldw) {
  const int r = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= N) return;
  const uint8_t* sm_row = sm + (size_t)r * K;
  const uint8_t* ex_row = ex + (size_t)r * (K >> 1);
  bf16* out = W + (size_t)r * ldw;
  const uint32_t bp = (uint32_t)base[r] - 1u;
  for (int c = lane; c < (K >> 3); c += 32) {
    const uint2 s = *reinterpret_cast<const uint2*>(sm_row + sm_offset(c));
    const uint32_t e = *reinterpret_cast<const uint32_t*>(ex_row + ex_offset(c));
    reinterpret_cast<uint4*>(out)[c] = decode_chunk(s.x, s.y, e, bp);
  }
  __syncwarp();
  uint16_t* out16 = reinterpret_cast<uint16_t*>(out);
  for (int j = row_ptr[r] + lane; j < row_ptr[r + 1]; j += 32) {
    const int v = exc[j];
    out16[v >> 8] |= (uint16_t)((v & 0xFF) << 7);
  }
}

}  // namespace pack12
}  // namespace srgpt

using namespace srgpt;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" __attribute__((visibility("default"))) int srgpt_pack12_scan_bf16(const void* W, int ldw, int N, int K, unsigned char* base, int* n_exc,
                                                                               int* n_bad, void* stream) {
  SRGPT_CHECK_ARG(W && base && n_exc && n_bad && N > 0 && K > 0 && (K % pack12::BATCH) == 0 && ldw >= K && (ldw % 8) == 0 && aligned16(W));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_pack12_scan_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  pack12::scan_kernel<<<ceil_div(N, pack12::WARPS), pack12::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(W), ldw, N, K, base, n_exc, n_bad);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
#endif
}

extern "C" __attribute__((visibility("default"))) int srgpt_pack12_bf16(const void* W, int ldw, int N, int K, const unsigned char* base, const int* row_ptr,
                                                                          void* sm, void* ex, int* exc, void* stream) {
  SRGPT_CHECK_ARG(W && base && row_ptr && sm && ex && exc && N > 0 && K > 0 && (K % pack12::BATCH) == 0 && ldw >= K && (ldw % 8) == 0);
  SRGPT_CHECK_ARG(aligned16(W) && aligned16(sm) && aligned16(ex));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_pack12_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  pack12::pack_kernel<<<ceil_div(N, pack12::WARPS), pack12::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(W), ldw, N, K, base, row_ptr, reinterpret_cast<uint8_t*>(sm), reinterpret_cast<uint8_t*>(ex), exc);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
#endif
}

extern "C" __attribute__((visibility("default"))) int srgpt_unpack12_bf16(const srgpt_packed12* P, int N, int K, void* W, int ldw, void* stream) {
  SRGPT_CHECK_ARG(P && P->sm && P->ex && P->base && P->row_ptr && P->exc && W && N > 0 && K > 0 && (K % pack12::BATCH) == 0);
  SRGPT_CHECK_ARG(ldw >= K && (ldw % 8) == 0 && aligned16(W) && aligned16(P->sm) && aligned16(P->ex));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_unpack12_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  pack12::unpack_kernel<<<ceil_div(N, pack12::WARPS), pack12::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint8_t*>(P->sm), reinterpret_cast<const uint8_t*>(P->ex), P->base, P->row_ptr, P->exc, N, K,
      reinterpret_cast<bf16*>(W), ldw);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
#endif
}
