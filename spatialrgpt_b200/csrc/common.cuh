// Shared device/host helpers for the sm_90a kernels behind the srgpt C-ABI (include/srgpt_b200.h).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace srgpt {

// ---- host-side error plumbing: every extern "C" entry returns 0 or a negative code, never throws
enum : int {
  SRGPT_OK = 0,
  SRGPT_ERR_INVALID = -1,   // bad argument (shape / alignment / null)
  SRGPT_ERR_CUDA = -2,      // CUDA runtime / driver error (see srgpt_last_error)
  SRGPT_ERR_UNSUPPORTED = -3,
};

void set_last_error(const char* fmt, ...);

#define SRGPT_CHECK_ARG(cond)                                                              \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      ::srgpt::set_last_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, #cond);   \
      return ::srgpt::SRGPT_ERR_INVALID;                                                   \
    }                                                                                      \
  } while (0)

#define SRGPT_CHECK_CUDA(expr)                                                             \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::srgpt::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                \
                              cudaGetErrorString(_e));                                     \
      return ::srgpt::SRGPT_ERR_CUDA;                                                      \
    }                                                                                      \
  } while (0)

#define SRGPT_CHECK_LAUNCH() SRGPT_CHECK_CUDA(cudaGetLastError())

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
int sm_count();  // cached multiProcessorCount of the current device

// ---- optional in-kernel timeline (srgpt_trace_begin / srgpt_trace_end): each traced launch owns 4 u64 slots
//      [0] min globaltimer at CTA start, [1] min globaltimer after griddepcontrol.wait, [2] max globaltimer at CTA
//      end, [3] CTA count.  Costs 3 atomics per CTA; disabled (nullptr) unless a trace buffer is installed.
unsigned long long* trace_next_slot();  // host: returns the 4-slot record for the next launch, or nullptr
bool pdl_enabled();                      // false when SRGPT_NO_PDL=1 (debug knob: plain stream-ordered launches)
bool env_flag(const char* name);

// ---- device helpers
// The 16-bit element type of this build.  The library is compiled twice from the same sources: libsrgpt_b200.so computes in bfloat16
// (the reference's eval default, llava/eval/eval_spatial.py:206-212) and libsrgpt_b200_f16.so (-DSRGPT_ELEM_F16) in IEEE half (the
// loader default, llava/model/builder.py:62; llava/eval/eval_region_cls.py:316-317).  Every rounding point is the same in both - the
// fp32 accumulators are rounded to the element type exactly where torch would materialise a tensor - so the kernels are written once
// against the alias `bf16` and these helpers; only the conversions, the mma.sync / wgmma operand formats and the tensor-map data
// type differ.  srgpt_elem_type() reports which build a loaded library is.
#ifdef SRGPT_ELEM_F16
typedef __half bf16;
#define SRGPT_ELEM_PTX "f16"
#define SRGPT_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_FLOAT16
__device__ __forceinline__ float e2f(bf16 x) { return __half2float(x); }
__device__ __forceinline__ bf16 f2e(float x) { return __float2half_rn(x); }
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu))); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u >> 16))); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
#else
typedef __nv_bfloat16 bf16;
#define SRGPT_ELEM_PTX "bf16"
#define SRGPT_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
__device__ __forceinline__ float e2f(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ bf16 f2e(float x) { return __float2bfloat16_rn(x); }
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
#endif

__device__ __forceinline__ float bf16_round(float x) { return e2f(f2e(x)); }

// 8 bf16 (one 16-byte vector) -> 8 floats
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  f[0] = bf16_lo(v.x); f[1] = bf16_hi(v.x);
  f[2] = bf16_lo(v.y); f[3] = bf16_hi(v.y);
  f[4] = bf16_lo(v.z); f[5] = bf16_hi(v.z);
  f[6] = bf16_lo(v.w); f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 v;
  v.x = pack_bf16x2(f[0], f[1]);
  v.y = pack_bf16x2(f[2], f[3]);
  v.z = pack_bf16x2(f[4], f[5]);
  v.w = pack_bf16x2(f[6], f[7]);
  return v;
}

// streaming 16-byte load that does not allocate in L1 (weights / features read exactly once)
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void trace_mark(unsigned long long* rec, int which) {
  if (rec != nullptr && threadIdx.x == 0) {
    const unsigned long long t = globaltimer_ns();
    if (which == 2) {
      atomicMax(rec + 2, t);
      atomicAdd(rec + 3, 1ull);
    } else {
      atomicMin(rec + which, t);
    }
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum; `red` is >= 32 floats of shared memory; every thread gets the result
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// Arg max over wide rows (rowops.cu argmax_wide_kernel, logits_process.cu): one CTA per ARGMAX_SEG columns, the segments of a row
// meet in a 64-bit atomicMax on (float_order_bits(value) << 32 | ~index) - max value first, lowest index on ties.
constexpr int ARGMAX_SEG = 4096;
__device__ __forceinline__ unsigned int float_order_bits(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// host: keys [rows] (u64, as above) -> the arg max index of each row, in place (rowops.cu)
void argmax_unpack(long long* keys, int rows, cudaStream_t stream);

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_tanh(float x) {
  // tanh on the SFU (MUFU.TANH, rel. error ~2^-11): the result is rounded to bf16 (2^-8) right after, and the
  // libm tanhf (~25 instructions) made the SigLIP fc1 epilogue longer than its main loop
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}
// CLIP's "quick_gelu" (HF QuickGELUActivation: input * torch.sigmoid(1.702 * input)) - three element-type torch ops, so the
// product 1.702 x and the sigmoid are each rounded to the element type before the final multiply (x is already rounded)
__device__ __forceinline__ float quick_gelu(float x) {
  const float t = bf16_round(1.702f * x);
  const float s = bf16_round(1.0f / (1.0f + __expf(-t)));
  return x * s;
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

}  // namespace srgpt
