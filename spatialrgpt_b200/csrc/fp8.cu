// FP8 (E4M3) row quantization of the W8A8 decoder-layer linears (DESIGN.md §3, §7).  One definition for weights (once, at load time)
// and activations (before every FP8 GEMM):
//   a = max_k |x[r, k]| in fp32; inv = 448 / a and s[r] = a / 448 (both 1 when a == 0);
//   q[r, k] = e4m3(fl32(x[r, k] * inv)), round to nearest even with saturation to +-448 (cvt.rn.satfinite.e4m3x2.f32).
// The GEMM then computes y[m, n] = acc[m, n] * (s_x[m] * s_w[n]) with acc the exact fp32 sum of the E4M3 products (gemm_wgmma.cu).
#include "fp8.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace fp8 {

constexpr int THREADS = 256;

// One CTA per row, 8 elements (one 16-byte vector) per thread and step.  The row maximum is a max-reduction, exact in any order, so
// the scale does not depend on the thread count.  The second pass re-reads the row (L1 / L2 hits).  n_bad != NULL: counts the rows
// that hold Inf or NaN (the weight quantizer rejects them).
__global__ void __launch_bounds__(THREADS) quantize_rows_kernel(const bf16* __restrict__ x, int ldx, int K, uint8_t* __restrict__ q, int ldq,
                                                                float* __restrict__ scale, int* __restrict__ n_bad) {
  __shared__ float red[32];
  __shared__ int bad_any;
  const int r = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)r * ldx);
  const int nv = K / 8;
  if (threadIdx.x == 0) bad_any = 0;
  float m = 0.f;
  bool bad = false;
  for (int v = threadIdx.x; v < nv; v += THREADS) {
    float f[8];
    unpack8(src[v], f);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      bad |= !isfinite(f[t]);
      m = fmaxf(m, fabsf(f[t]));
    }
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (bad) bad_any = 1;
  m = red[0];
#pragma unroll
  for (int w = 1; w < THREADS / 32; ++w) m = fmaxf(m, red[w]);
  float inv, s;
  row_scales(m, inv, s);
  if (threadIdx.x == 0) scale[r] = s;
  uint2* dst = reinterpret_cast<uint2*>(q + (size_t)r * ldq);
  for (int v = threadIdx.x; v < nv; v += THREADS) {
    float f[8];
    unpack8(src[v], f);
    uint32_t c[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) c[t] = e4m3x2(__fmul_rn(f[2 * t], inv), __fmul_rn(f[2 * t + 1], inv));
    dst[v] = make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
  }
  __syncthreads();
  if (threadIdx.x == 0 && bad_any && n_bad != nullptr) atomicAdd(n_bad, 1);
}

static int quantize_rows(const void* x, int ldx, int M, int K, void* q, int ldq, float* scale, int* n_bad, void* stream) {
  SRGPT_CHECK_ARG(x != nullptr && q != nullptr && scale != nullptr && M > 0 && K > 0);
  SRGPT_CHECK_ARG((K % 16) == 0 && ldx >= K && (ldx % 8) == 0 && ldq >= K && (ldq % 16) == 0);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0);
  quantize_rows_kernel<<<M, THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const bf16*>(x), ldx, K,
                                                                                   reinterpret_cast<uint8_t*>(q), ldq, scale, n_bad);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

}  // namespace fp8
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_fp8_quantize_weight_bf16(const void* W, int ldw, int N, int K, void* q, float* scale,
                                                                                       int* n_bad, void* stream) {
  SRGPT_CHECK_ARG(n_bad != nullptr);
  return fp8::quantize_rows(W, ldw, N, K, q, K, scale, n_bad, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_fp8_quantize_act_bf16(const void* x, int ldx, int M, int K, void* q, int ldq, float* scale,
                                                                                    void* stream) {
  return fp8::quantize_rows(x, ldx, M, K, q, ldq, scale, nullptr, stream);
}
