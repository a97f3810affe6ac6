// Classifier-free guidance of a decode step (generate(guidance_scale=, negative_prompt_ids=); DESIGN.md §4, §7).
//
// Reference: HF UnbatchedClassifierFreeGuidanceLogitsProcessor.__call__ (transformers generation/logits_process.py), which
// GenerationMixin._get_logits_processor puts first in the processor list when guidance_scale is not None and != 1 (generate() at
// llava_llama.py:212):
//     scores = log_softmax(scores);  u = log_softmax(uncond_logits[:, -1]);  guided = g * (scores - u) + u
// Here the rows step decodes every prompt b (row b) and its unconditional branch (row B + b) side by side; the fp32 logits of both sit
// in logits [2B, V].  One CTA per row pair makes three passes over the two rows (the second and third from L2): the maxima, the sums of
// exp(x - m), then the guided row and its arg max, every row read and written in 16-byte vectors.  log_softmax is torch's (x - m) - log(sum exp(x - m)) with accurate expf / logf; the
// sum order is this kernel's own fixed tree, so the log-probs may differ from torch's in the last bits, and two calls are bit-identical.
// The combine is three separately rounded fp32 operations (no FMA contraction).  The arg max key is argmax_wide's: the largest value,
// the lowest index on ties, NaN never wins (an all-NaN row picks 0).  g is read from device memory, so a captured step serves any scale.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace guidance {

constexpr int THREADS = 512;
constexpr int NW = THREADS / 32;

// programmatic dependent launch, as the decode kernels around this one use it (gemv.cu)
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename K, typename... Args>
static int launch_pdl(K kernel, int grid, int block, void* stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.stream = reinterpret_cast<cudaStream_t>(stream);
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
  return SRGPT_OK;
}

// f(j, x) over every element of the fp32 row p [V]: thread-strided scalars up to the first 16-byte boundary, 16-byte vectors, then the
// tail.  Each thread visits its columns in increasing order.
template <typename F>
__device__ __forceinline__ void for_row(const float* __restrict__ p, int V, F f) {
  const int head = min(V, (int)(((16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15) >> 2));
  const int nvec = (V - head) >> 2, tail0 = head + nvec * 4;
  if ((int)threadIdx.x < head) f((int)threadIdx.x, p[threadIdx.x]);
  const float4* v = reinterpret_cast<const float4*>(p + head);
  for (int i = threadIdx.x; i < nvec; i += THREADS) {
    const float4 q = v[i];
    const int j = head + 4 * i;
    f(j, q.x);
    f(j + 1, q.y);
    f(j + 2, q.z);
    f(j + 3, q.w);
  }
  for (int j = tail0 + threadIdx.x; j < V; j += THREADS) f(j, p[j]);
}

// block-wide maximum over the threads' values (fmaxf: a NaN is dropped unless every value is NaN); every thread gets the result
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  return warp_max(lane < NW ? red[lane] : -INFINITY);
}

__device__ __forceinline__ unsigned long long argmax_key(float v, int j) {
  return v == v ? ((unsigned long long)float_order_bits(v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)j) : 0ull;
}

__device__ __forceinline__ unsigned long long warp_max_key(unsigned long long k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ok = __shfl_xor_sync(0xffffffffu, k, o);
    k = ok > k ? ok : k;
  }
  return k;
}

// Pair b: rows b (conditional) and B + b (unconditional) of logits [2B, V] -> guided row b [V]; lse (optional) [2B][2] = {m, log sum
// exp(x - m)} of each row; ids (optional, greedy) ids[b] = ids[B + b] = the arg max of the guided row.
__global__ void __launch_bounds__(THREADS)
guidance_rows_kernel(const float* __restrict__ logits, int V, int B, const float* __restrict__ scale, float* __restrict__ guided,
                     float* __restrict__ lse, long long* __restrict__ ids) {
  __shared__ float red[NW];
  __shared__ unsigned long long kred[NW];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const float* c = logits + (size_t)b * V;
  const float* u = logits + (size_t)(B + b) * V;
  float* out = guided + (size_t)b * V;

  float mc = -INFINITY, mu = -INFINITY;
  for_row(c, V, [&](int, float x) { mc = fmaxf(mc, x); });
  for_row(u, V, [&](int, float x) { mu = fmaxf(mu, x); });
  mc = block_max(mc, red);
  mu = block_max(mu, red);
  float sc = 0.f, su = 0.f;
  for_row(c, V, [&](int, float x) { sc += expf(__fsub_rn(x, mc)); });
  for_row(u, V, [&](int, float x) { su += expf(__fsub_rn(x, mu)); });
  const float lc = logf(block_sum(sc, red));
  const float lu = logf(block_sum(su, red));
  if (lse != nullptr && threadIdx.x == 0) {
    lse[2 * b] = mc;
    lse[2 * b + 1] = lc;
    lse[2 * (B + b)] = mu;
    lse[2 * (B + b) + 1] = lu;
  }
  const float g = *scale;
  unsigned long long best = 0ull;
  auto guide = [&](int j, float x, float y) {  // x = c[j], y = u[j] -> the guided value, written by the caller
    const float s = __fsub_rn(__fsub_rn(x, mc), lc);
    const float q = __fsub_rn(__fsub_rn(y, mu), lu);
    const float r = __fadd_rn(__fmul_rn(g, __fsub_rn(s, q)), q);
    const unsigned long long k = argmax_key(r, j);
    best = k > best ? k : best;
    return r;
  };
  // c and out share their alignment (both rows start at b * V, both bases 16-byte aligned).  u is d elements past a 16-byte boundary
  // at the same column (d is the same for the whole vector body), so its 4 columns are taken from the aligned vector that holds the
  // first and, when d > 0, the next one - the aligned vector holding u[j + 3], never past the row's last 16-byte chunk.
  const int head = min(V, (int)(((16 - (reinterpret_cast<uintptr_t>(c) & 15)) & 15) >> 2));
  const int nvec = (V - head) >> 2, tail0 = head + nvec * 4;
  if ((int)threadIdx.x < head) out[threadIdx.x] = guide(threadIdx.x, c[threadIdx.x], u[threadIdx.x]);
  const int d = (int)((reinterpret_cast<uintptr_t>(u + head) & 15) >> 2);
  const float4* cv = reinterpret_cast<const float4*>(c + head);
  const float4* uv = reinterpret_cast<const float4*>(u + head - d);
  float4* ov = reinterpret_cast<float4*>(out + head);
  for (int i = threadIdx.x; i < nvec; i += THREADS) {
    const float4 x = cv[i];
    const float4 a = uv[i];
    float4 y = a;
    if (d != 0) {
      const float4 n = uv[i + 1];
      y = d == 1 ? make_float4(a.y, a.z, a.w, n.x) : d == 2 ? make_float4(a.z, a.w, n.x, n.y) : make_float4(a.w, n.x, n.y, n.z);
    }
    const int j = head + 4 * i;
    float4 r;
    r.x = guide(j, x.x, y.x);
    r.y = guide(j + 1, x.y, y.y);
    r.z = guide(j + 2, x.z, y.z);
    r.w = guide(j + 3, x.w, y.w);
    ov[i] = r;
  }
  for (int j = tail0 + threadIdx.x; j < V; j += THREADS) out[j] = guide(j, c[j], u[j]);
  if (ids == nullptr) return;
  best = warp_max_key(best);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) kred[warp] = best;
  __syncthreads();
  if (warp == 0) {
    best = warp_max_key(lane < NW ? kred[lane] : 0ull);
    if (lane == 0) {
      const long long t = best == 0ull ? 0ll : (long long)(0xFFFFFFFFu - (unsigned int)(best & 0xFFFFFFFFull));
      ids[b] = t;
      ids[B + b] = t;
    }
  }
}

// ids[B + b] = ids[b]: a prompt's drawn token is its unconditional branch's next token too
__global__ void pair_ids_kernel(long long* __restrict__ ids, int B) {
  pdl_launch_dependents();
  pdl_wait();
  if ((int)threadIdx.x < B) ids[B + threadIdx.x] = ids[threadIdx.x];
}

}  // namespace guidance
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_guidance_rows(const float* logits, int V, int B, const float* scale, float* guided,
                                                                          float* lse, long long* ids, void* stream) {
  SRGPT_CHECK_ARG(logits && scale && guided && V > 0 && B >= 1 && B <= SRGPT_SPEC_T_MAX / 2);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (reinterpret_cast<uintptr_t>(guided) & 15) == 0);
  SRGPT_CHECK_ARG(guided + (size_t)B * V <= logits || logits + (size_t)2 * B * V <= guided);  // the guided rows overwrite no logits
  return guidance::launch_pdl(guidance::guidance_rows_kernel, B, guidance::THREADS, stream, logits, V, B, scale, guided, lse, ids);
}

extern "C" __attribute__((visibility("default"))) int srgpt_guidance_pair_ids(long long* ids, int B, void* stream) {
  SRGPT_CHECK_ARG(ids && B >= 1 && B <= SRGPT_SPEC_T_MAX / 2);
  return guidance::launch_pdl(guidance::pair_ids_kernel, 1, 32, stream, ids, B);
}
