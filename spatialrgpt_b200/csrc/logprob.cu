// Row log-softmax at target tokens (llava_llama.forward(labels=) and LlamaDecoder.score_candidates; DESIGN.md §7).
//
// Reference: LlamaForCausalLM.forward (modeling_llama.py:1044-1058) takes the element-type lm_head output, widens it with .float()
// and runs CrossEntropyLoss (log_softmax + NLL, mean over the targets that are not IGNORE_INDEX) over the shifted rows.  Here the
// element-type rows are read directly: each element is widened to fp32 exactly as .float() does, and no fp32 copy of the logits is
// made.  Kernel 1 (one CTA per row) makes one pass over the row with 16-byte loads and keeps a running (max, sum of exp) per thread,
// merged in a fixed tree: lse = m + log(sum exp(x - m)).  Kernel 2 (one CTA) gathers logits[row_i, target_i] - lse[row_i] for the n
// pairs and reduces their mean in a fixed order.  No atomics on values: two calls on the same input are bit-identical.
#include <vector>

#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace logprob {

constexpr int ROW_THREADS = 512;
constexpr int PAIR_THREADS = 1024;
constexpr int UNROLL = 4;  // 16-byte vectors in flight per thread
constexpr long long IGNORE = -100;  // IGNORE_INDEX (constants.py)

// (m, s) represents s * exp(m): the running maximum and the sum of exp(x - m) over the elements seen.  An empty set is (-inf, 0).
// -inf elements add nothing; a NaN element makes s NaN, and a +inf one makes it NaN through exp(inf - inf), as torch's log_softmax.
__device__ __forceinline__ void merge(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) {  // both empty (or NaN sums over -inf maxima)
    s = s + s2;
    return;
  }
  s = s * __expf(m - mn) + s2 * __expf(m2 - mn);
  m = mn;
}

__device__ __forceinline__ float term(float x, float m) { return x == -INFINITY ? 0.f : __expf(x - m); }

__device__ __forceinline__ void add8(const uint4& v, float& m, float& s) {
  float f[8];
  unpack8(v, f);
  float vm = f[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) vm = fmaxf(vm, f[i]);
  float vs = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) vs += term(f[i], vm);
  merge(m, s, vm, vs);
}

__device__ __forceinline__ void add1(float x, float& m, float& s) { merge(m, s, x, term(x, x)); }

__global__ void __launch_bounds__(ROW_THREADS)
row_lse_kernel(const bf16* __restrict__ logits, long long ld, int V, float* __restrict__ lse) {
  __shared__ float sm[ROW_THREADS / 32], ss[ROW_THREADS / 32];
  const bf16* row = logits + (size_t)blockIdx.x * ld;
  // elements before the first 16-byte boundary, the aligned vectors, the tail
  const int head = min(V, (int)(((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15) >> 1));
  const int nvec = (V - head) >> 3;
  const int tail0 = head + nvec * 8;
  const uint4* vec = reinterpret_cast<const uint4*>(row + head);
  float m = -INFINITY, s = 0.f;
  const int tid = threadIdx.x;
  if (tid < head) add1(e2f(row[tid]), m, s);
  if (tid < V - tail0) add1(e2f(row[tail0 + tid]), m, s);
  for (int c0 = tid; c0 < nvec; c0 += UNROLL * ROW_THREADS) {
    uint4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
      if (c0 + u * ROW_THREADS < nvec) v[u] = ld_stream16(vec + c0 + u * ROW_THREADS);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
      if (c0 + u * ROW_THREADS < nvec) add8(v[u], m, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    merge(m, s, m2, s2);
  }
  const int lane = tid & 31, warp = tid >> 5;
  if (lane == 0) { sm[warp] = m; ss[warp] = s; }
  __syncthreads();
  if (warp == 0) {
    m = lane < ROW_THREADS / 32 ? sm[lane] : -INFINITY;
    s = lane < ROW_THREADS / 32 ? ss[lane] : 0.f;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {  // ROW_THREADS / 32 = 16 partials
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      merge(m, s, m2, s2);
    }
    if (lane == 0) lse[blockIdx.x] = m == -INFINITY ? __int_as_float(0x7fc00000) : m + logf(s);
  }
}

// pairs[i] = (row, target) with target in [0, V) or IGNORE (-100): logprob[i] = logits[row, target] - lse[row] (0 when ignored);
// loss (when given) = -(sum of the non-ignored logprob) / (their count), NaN when there are none.  Thread t sums pairs t, t + T, ...
// in order, then a fixed tree: the order never depends on timing.
__global__ void __launch_bounds__(PAIR_THREADS)
pair_logprob_kernel(const bf16* __restrict__ logits, long long ld, const int2* __restrict__ pairs, int n, const float* __restrict__ lse,
                    float* __restrict__ logprob, float* __restrict__ loss) {
  __shared__ float red[32];
  __shared__ int cred[32];
  float sum = 0.f;
  int cnt = 0;
  for (int i = threadIdx.x; i < n; i += PAIR_THREADS) {
    const int2 p = pairs[i];
    float lp = 0.f;
    if (p.y != (int)IGNORE) {
      lp = e2f(logits[(size_t)p.x * ld + p.y]) - lse[p.x];
      sum += lp;
      ++cnt;
    }
    logprob[i] = lp;
  }
  if (loss == nullptr) return;
  sum = block_sum(sum, red);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) cred[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < PAIR_THREADS / 32; ++w) total += cred[w];
    *loss = total > 0 ? -sum / (float)total : __int_as_float(0x7fc00000);
  }
}

}  // namespace logprob
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_token_logprobs(const void* logits, long long ld, int rows, int V, const int* pair_rows,
                                                                           const long long* pair_targets, int n, void* workspace,
                                                                           long long workspace_bytes, float* lse, float* logprob, float* loss,
                                                                           void* stream) {
  SRGPT_CHECK_ARG(logits && lse && rows > 0 && V > 0 && ld >= V && n >= 0);
  SRGPT_CHECK_ARG(n == 0 || (pair_rows && pair_targets && logprob && workspace && workspace_bytes >= (long long)n * 8));
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0);
  std::vector<int2> host((size_t)n);
  for (int i = 0; i < n; ++i) {
    const int r = pair_rows[i];
    const long long t = pair_targets[i];
    if (r < 0 || r >= rows || (t != logprob::IGNORE && (t < 0 || t >= V))) {
      set_last_error("srgpt_token_logprobs: pair %d = (row %d, target %lld) is outside %d rows x %d columns (target -100 = ignored)", i, r,
                     t, rows, V);
      return SRGPT_ERR_INVALID;
    }
    host[i] = make_int2(r, (int)t);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bf16* x = reinterpret_cast<const bf16*>(logits);
  if (n > 0) SRGPT_CHECK_CUDA(cudaMemcpyAsync(workspace, host.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
  logprob::row_lse_kernel<<<rows, logprob::ROW_THREADS, 0, st>>>(x, ld, V, lse);
  SRGPT_CHECK_LAUNCH();
  if (n > 0 || loss != nullptr) {
    logprob::pair_logprob_kernel<<<1, logprob::PAIR_THREADS, 0, st>>>(x, ld, reinterpret_cast<const int2*>(workspace), n, lse, logprob, loss);
    SRGPT_CHECK_LAUNCH();
  }
  return SRGPT_OK;
}
