// Load-time kernels of the NF4 weight-only quantization (format and value: nf4.cuh; rules: DESIGN.md §3).  The host runs them once per
// decoder-layer matrix, before the layer's matrices are fused (ops.nf4_quantize), then orders the fused codes for the decode GEMV and
// checks the lane-ordered planes against the dequantized copy (ops.nf4_planes).
#include "nf4.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace nf4 {

constexpr int THREADS = 256;

// One thread per block of 64 weights: absmax = max |w| (fp32), x = w * fl32(1 / absmax), code = the number of fp32 midpoints of the
// code table that x exceeds (nearest code, a tie going to the lower one); a NaN x (w = 0 against an infinite reciprocal, e.g. an
// all-zero block) takes code 7, the value 0.  *n_bad counts blocks holding Inf or NaN.
__global__ void __launch_bounds__(THREADS) quantize_kernel(const bf16* __restrict__ W, int ldw, int N, int K, uint8_t* __restrict__ codes,
                                                           float* __restrict__ absmax, int* __restrict__ n_bad) {
  const int kb = K / BLOCK;
  const long long blk = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (blk >= (long long)N * kb) return;
  const int r = (int)(blk / kb), j = (int)(blk - (long long)r * kb);
  const uint4* src = reinterpret_cast<const uint4*>(W + (size_t)r * ldw + (size_t)j * BLOCK);
  float f[BLOCK];
#pragma unroll
  for (int c = 0; c < BLOCK / 8; ++c) unpack8(src[c], f + 8 * c);
  float m = 0.f;
  bool bad = false;
#pragma unroll
  for (int t = 0; t < BLOCK; ++t) {
    bad |= !isfinite(f[t]);
    m = fmaxf(m, fabsf(f[t]));
  }
  if (bad) atomicAdd(n_bad, 1);
  absmax[blk] = m;
  float mid[15];
#pragma unroll
  for (int i = 0; i < 15; ++i) mid[i] = __fmul_rn(__fadd_rn(code_value(i), code_value(i + 1)), 0.5f);
  const float rcp = __frcp_rn(m);
  uint32_t out[8];
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    uint32_t word = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t byte = 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x = __fmul_rn(f[8 * w + 2 * k + h], rcp);
        uint32_t q = 0;
#pragma unroll
        for (int i = 0; i < 15; ++i) q += (x > mid[i]) ? 1u : 0u;
        if (isnan(x)) q = 7;
        byte |= q << (h == 0 ? 4 : 0);
      }
      word |= byte << (8 * k);
    }
    out[w] = word;
  }
  uint4* dst = reinterpret_cast<uint4*>(codes + (size_t)r * (K / 2) + (size_t)j * (BLOCK / 2));
  dst[0] = make_uint4(out[0], out[1], out[2], out[3]);
  dst[1] = make_uint4(out[4], out[5], out[6], out[7]);
}

// offset = mean of the matrix's absmax vector: summed in fp64 in index order (deterministic, unlike a parallel fp32 mean), rounded to fp32
__global__ void __launch_bounds__(THREADS) offset_kernel(const float* __restrict__ a, long long n, float* __restrict__ offset) {
  constexpr int TILE = THREADS * 8;
  __shared__ float tile[TILE];
  double s = 0.0;
  for (long long t0 = 0; t0 < n; t0 += TILE) {
    const int len = (int)min((long long)TILE, n - t0);
    for (int i = threadIdx.x; i < len; i += THREADS) tile[i] = a[t0 + i];
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < len; ++i) s += (double)tile[i];
    __syncthreads();
  }
  if (threadIdx.x == 0) *offset = (float)(s / (double)n);
}

// One CTA per block of 256 absmax values: v = absmax - offset, absmax2 = max |v| over the block, y = v * fl32(1 / absmax2) clamped to
// [-1, 1] (a NaN, from a block whose values all equal the offset, counts as 0), c = the nearest entry of the signed dynamic map (the
// lowest index on a tie), and the resolved scale fl32(map[c] * absmax2) + offset.
__global__ void __launch_bounds__(BLOCK2) double_quant_kernel(const float* __restrict__ a, long long n, const float* __restrict__ dyn_map,
                                                              const float* __restrict__ offset, float* __restrict__ scale) {
  __shared__ float smap[256];
  __shared__ float red[32];
  smap[threadIdx.x] = dyn_map[threadIdx.x];
  const long long i = (long long)blockIdx.x * BLOCK2 + threadIdx.x;
  const float off = *offset;
  const float v = i < n ? __fsub_rn(a[i], off) : 0.f;
  float m = warp_max(fabsf(v));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < BLOCK2 / 32; ++w) m = fmaxf(m, red[w]);
  if (i >= n) return;
  float y = __fmul_rn(v, __frcp_rn(m));
  y = isnan(y) ? 0.f : fminf(fmaxf(y, -1.f), 1.f);
  float best = INFINITY;
  int c = 0;
  for (int k = 0; k < 256; ++k) {
    const float d = fabsf(__fsub_rn(y, smap[k]));
    if (d < best) {
      best = d;
      c = k;
    }
  }
  scale[i] = __fadd_rn(__fmul_rn(smap[c], m), off);
}

// natural-order codes + scales -> the element-type matrix (one thread per chunk of 8 weights)
__global__ void __launch_bounds__(THREADS) dequantize_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ scale, int N, int K,
                                                             bf16* __restrict__ W, int ldw) {
  const int nch = K / 8;
  const long long g = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (g >= (long long)N * nch) return;
  const int r = (int)(g / nch), cc = (int)(g - (long long)r * nch);
  const uint32_t u = *reinterpret_cast<const uint32_t*>(codes + (size_t)r * (K / 2) + (size_t)cc * 4);
  const float s = scale[(size_t)r * (K / BLOCK) + cc / 8];
  float f[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) f[t] = __fmul_rn(code_value((u >> (8 * (t >> 1) + ((t & 1) ? 0 : 4))) & 15u), s);
  reinterpret_cast<uint4*>(W + (size_t)r * ldw)[cc] = pack8(f);
}

// natural order -> lane order: chunk cc's 4 bytes move to lane_offset(cc) with the nibbles of every byte swapped (weight t at bits 4t)
__global__ void __launch_bounds__(THREADS) lane_order_kernel(const uint8_t* __restrict__ codes, int N, int K, uint8_t* __restrict__ q) {
  const int nch = K / 8;
  const long long g = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (g >= (long long)N * nch) return;
  const int r = (int)(g / nch), cc = (int)(g - (long long)r * nch);
  const uint32_t u = *reinterpret_cast<const uint32_t*>(codes + (size_t)r * (K / 2) + (size_t)cc * 4);
  *reinterpret_cast<uint32_t*>(q + (size_t)r * (K / 2) + lane_offset(cc)) = ((u >> 4) & 0x0F0F0F0Fu) | ((u & 0x0F0F0F0Fu) << 4);
}

// the lane-ordered planes -> the element-type matrix, through the decode GEMV's own dequant8
__global__ void __launch_bounds__(THREADS) unpack_kernel(const uint8_t* __restrict__ q, const float* __restrict__ scale, int N, int K,
                                                         bf16* __restrict__ W, int ldw) {
  __shared__ float tab[16];
  if (threadIdx.x < 16) tab[threadIdx.x] = code_value(threadIdx.x);
  __syncthreads();
  const int nch = K / 8;
  const long long g = (long long)blockIdx.x * THREADS + threadIdx.x;
  if (g >= (long long)N * nch) return;
  const int r = (int)(g / nch), cc = (int)(g - (long long)r * nch);
  const uint32_t word = *reinterpret_cast<const uint32_t*>(q + (size_t)r * (K / 2) + lane_offset(cc));
  reinterpret_cast<uint4*>(W + (size_t)r * ldw)[cc] = dequant8(word, scale[(size_t)r * (K / BLOCK) + cc / 8], tab);
}

static int grid_of(long long n) { return (int)((n + THREADS - 1) / THREADS); }

}  // namespace nf4
}  // namespace srgpt

using namespace srgpt;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

extern "C" __attribute__((visibility("default"))) int srgpt_nf4_quantize_bf16(const void* W, int ldw, int N, int K, unsigned char* codes, float* absmax,
                                                                                int* n_bad, void* stream) {
  SRGPT_CHECK_ARG(W && codes && absmax && n_bad && N > 0 && K > 0 && (K % nf4::BLOCK) == 0 && ldw >= K && (ldw % 8) == 0);
  SRGPT_CHECK_ARG(aligned16(W) && aligned16(codes) && aligned4(absmax));
  nf4::quantize_kernel<<<nf4::grid_of((long long)N * (K / nf4::BLOCK)), nf4::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(W), ldw, N, K, codes, absmax, n_bad);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_nf4_double_quant(const float* absmax, long long n, const float* dyn_map, float* offset,
                                                                               float* scale, void* stream) {
  SRGPT_CHECK_ARG(absmax && dyn_map && offset && scale && n > 0 && n <= (long long)0x7fffffff * nf4::BLOCK2);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  nf4::offset_kernel<<<1, nf4::THREADS, 0, st>>>(absmax, n, offset);
  SRGPT_CHECK_LAUNCH();
  nf4::double_quant_kernel<<<(int)((n + nf4::BLOCK2 - 1) / nf4::BLOCK2), nf4::BLOCK2, 0, st>>>(absmax, n, dyn_map, offset, scale);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_nf4_dequantize_bf16(const unsigned char* codes, const float* scale, int N, int K, void* W,
                                                                                  int ldw, void* stream) {
  SRGPT_CHECK_ARG(codes && scale && W && N > 0 && K > 0 && (K % nf4::BLOCK) == 0 && ldw >= K && (ldw % 8) == 0);
  SRGPT_CHECK_ARG(aligned4(codes) && aligned4(scale) && aligned16(W));
  nf4::dequantize_kernel<<<nf4::grid_of((long long)N * (K / 8)), nf4::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      codes, scale, N, K, reinterpret_cast<bf16*>(W), ldw);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_nf4_lane_order(const unsigned char* codes, int N, int K, unsigned char* q, void* stream) {
  SRGPT_CHECK_ARG(codes && q && codes != q && N > 0 && K > 0 && (K % nf4::BATCH) == 0 && aligned4(codes) && aligned16(q));
  nf4::lane_order_kernel<<<nf4::grid_of((long long)N * (K / 8)), nf4::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(codes, N, K, q);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_nf4_unpack_bf16(const srgpt_nf4* P, int N, int K, void* W, int ldw, void* stream) {
  SRGPT_CHECK_ARG(P && P->q && P->scale && W && N > 0 && K > 0 && (K % nf4::BATCH) == 0 && ldw >= K && (ldw % 8) == 0);
  SRGPT_CHECK_ARG(aligned16(P->q) && aligned4(P->scale) && aligned16(W));
  nf4::unpack_kernel<<<nf4::grid_of((long long)N * (K / 8)), nf4::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      P->q, P->scale, N, K, reinterpret_cast<bf16*>(W), ldw);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
