// Contrastive search (generate(penalty_alpha=, top_k=); DESIGN.md §7): the degeneration penalty of every candidate row of a step and the
// per-prompt choice among a prompt's k candidates.
//
// Reference: HF GenerationMixin.contrastive_search + _ranking_fast (transformers 4.37.2 generation/utils.py), behind generate() at
// llava_llama.py:212 when num_beams == 1, do_sample is false, penalty_alpha > 0 and top_k > 1:
//     pen[i]   = max_j cos(context_hidden[j], next_hidden[i])        (every earlier position of the sequence, prompt rows included)
//     score[i] = (1 - alpha) * top_k_probs[i] - alpha * pen[i];   sel = argmax_i score[i]   (first index on ties)
// Row g * k + i of the batched step is candidate i of prompt g; the context of prompt g is its final-norm hidden rows ctx[g, 0 .. L_g),
// L_g = pos[g * k] (the position the candidates are processed at).  Nothing here is read from the host: alpha, the positions and the
// step counter live in device memory, so one captured graph serves every request of the same shape.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace contrastive {

constexpr int PEN_THREADS = 256;
constexpr int PEN_WARPS = PEN_THREADS / 32;
constexpr int CHUNK = 32;  // context rows per CTA
constexpr int KC = 8;      // candidates staged in shared memory at once (one per warp for their norms)
constexpr int SEL_THREADS = 256;
constexpr int K_MAX = 64;
constexpr int PEN_SMEM_MAX = 200 * 1024;  // KC staged candidate rows: H <= 12800

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const bf16* e = reinterpret_cast<const bf16*>(&u);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = e2f(e[j]);
}

// CTA (chunk c, prompt g): rows [c * CHUNK, min(L_g, (c + 1) * CHUNK)) of ctx[g].  Each context row is read once per group of KC
// candidates (once for k <= KC); its sum of squares and its KC dot products come out of the same pass, fp32 accumulation, one warp per
// row.  partial[g, c, i] = the largest cosine of candidate i over the chunk's rows (fmaxf: a NaN cosine, from a zero row, is dropped).
__global__ void __launch_bounds__(PEN_THREADS)
penalty_kernel(const bf16* __restrict__ cand, int ldc, const bf16* __restrict__ ctx, int L_cap, int H, const int* __restrict__ pos, int k,
               float* __restrict__ partial, int n_chunks) {
  extern __shared__ uint4 s_cand[];  // [KC][H / 8]
  __shared__ float s_norm[KC];
  __shared__ float s_best[PEN_WARPS][KC];
  const int g = blockIdx.y, c = blockIdx.x;
  const int L = pos[(size_t)g * k];
  const int r0 = c * CHUNK, r1 = min(min(L, L_cap), r0 + CHUNK);
  if (r0 >= r1) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nv = H >> 3;
  for (int i0 = 0; i0 < k; i0 += KC) {
    const int nk = min(KC, k - i0);
    __syncthreads();  // the previous group's candidates are no longer read
    for (int v = threadIdx.x; v < nk * nv; v += PEN_THREADS) {
      const int i = v / nv, j = v - i * nv;
      s_cand[v] = reinterpret_cast<const uint4*>(cand + (size_t)(g * k + i0 + i) * ldc)[j];
    }
    __syncthreads();
    if (warp < nk) {
      float ss = 0.f, f[8];
      for (int j = lane; j < nv; j += 32) {
        unpack8(s_cand[warp * nv + j], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) ss += f[e] * f[e];
      }
      ss = warp_sum(ss);
      if (lane == 0) s_norm[warp] = sqrtf(ss);
    }
    __syncthreads();
    float best[KC];
#pragma unroll
    for (int i = 0; i < KC; ++i) best[i] = -INFINITY;
    for (int r = r0 + warp; r < r1; r += PEN_WARPS) {
      const uint4* row = reinterpret_cast<const uint4*>(ctx + ((size_t)g * L_cap + r) * H);
      float acc[KC], ss = 0.f, x[8], y[8];
#pragma unroll
      for (int i = 0; i < KC; ++i) acc[i] = 0.f;
      for (int j = lane; j < nv; j += 32) {
        unpack8(row[j], x);
#pragma unroll
        for (int e = 0; e < 8; ++e) ss += x[e] * x[e];
#pragma unroll
        for (int i = 0; i < KC; ++i) {
          if (i < nk) {
            unpack8(s_cand[i * nv + j], y);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[i] += x[e] * y[e];
          }
        }
      }
      const float norm = sqrtf(warp_sum(ss));
#pragma unroll
      for (int i = 0; i < KC; ++i) {
        if (i < nk) best[i] = fmaxf(best[i], warp_sum(acc[i]) / (norm * s_norm[i]));
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < KC; ++i) s_best[warp][i] = best[i];
    }
    __syncthreads();
    if ((int)threadIdx.x < nk) {
      float m = -INFINITY;
      for (int w = 0; w < PEN_WARPS; ++w) m = fmaxf(m, s_best[w][threadIdx.x]);
      partial[((size_t)g * n_chunks + c) * k + i0 + threadIdx.x] = m;
    }
  }
}

// One CTA per prompt g.  pen = the maximum of the chunks' partial maxima in chunk order (no float atomics: a replay is bit-reproducible);
// p = exp(log-prob); score = fl(fl(a0 * p) - fl(a1 * pen)) with alpha = {a0, a1} = {1 - alpha, alpha} as fp32 (the host rounds 1 - alpha
// from double, as torch rounds a Python scalar), each operation rounded on its own as torch's eager ops round them.
// The largest score wins, the lowest index on ties; a candidate with token < 0 never wins.  Then the chosen token goes to
// out_ids[*step * B + g], the chosen final-norm row is appended to ctx[g] at L_g, its logits row becomes next_logits[g], the k rows'
// positions advance, and the last CTA to finish advances *step (atomic ticket, returned to zero).
__global__ void __launch_bounds__(SEL_THREADS)
select_kernel(const float* __restrict__ cand_scores, const int* __restrict__ cand_tokens, const float* __restrict__ partial, int n_chunks,
              const float* __restrict__ alpha, const bf16* __restrict__ xn, int ldx, int H, const bf16* __restrict__ logits, int ldl, int V,
              bf16* __restrict__ ctx, int L_cap, bf16* __restrict__ next_logits, int ldn, int* pos, int k, int B, long long* __restrict__ out_ids,
              int* step, unsigned int* ticket, int* __restrict__ sel, float* __restrict__ pen_out, float* __restrict__ score_out) {
  __shared__ float s_score[K_MAX];
  __shared__ int s_sel;
  const int g = blockIdx.x, tid = threadIdx.x;
  const int L = pos[(size_t)g * k];
  const int nch = min((L + CHUNK - 1) / CHUNK, n_chunks);
  if (tid < k) {
    float pen = -INFINITY;
    for (int c = 0; c < nch; ++c) pen = fmaxf(pen, partial[((size_t)g * n_chunks + c) * k + tid]);
    const float p = expf(cand_scores[(size_t)g * k + tid]);
    const float s = __fsub_rn(__fmul_rn(alpha[0], p), __fmul_rn(alpha[1], pen));
    s_score[tid] = s;
    pen_out[(size_t)g * k + tid] = pen;
    score_out[(size_t)g * k + tid] = s;
  }
  __syncthreads();
  if (tid == 0) {
    int b = -1;
    for (int i = 0; i < k; ++i)
      if (cand_tokens[(size_t)g * k + i] >= 0 && (b < 0 || s_score[i] > s_score[b])) b = i;
    b = b < 0 ? 0 : b;
    s_sel = b;
    sel[g] = b;
    out_ids[(size_t)(*step) * B + g] = cand_tokens[(size_t)g * k + b];
  }
  __syncthreads();
  const int r = g * k + s_sel;
  if (L < L_cap) {
    const uint4* src = reinterpret_cast<const uint4*>(xn + (size_t)r * ldx);
    uint4* dst = reinterpret_cast<uint4*>(ctx + ((size_t)g * L_cap + L) * H);
#pragma unroll 1
    for (int v = tid; v < (H >> 3); v += SEL_THREADS) dst[v] = src[v];
  }
  const uint4* lsrc = reinterpret_cast<const uint4*>(logits + (size_t)r * ldl);
  uint4* ldst = reinterpret_cast<uint4*>(next_logits + (size_t)g * ldn);
#pragma unroll 1
  for (int v = tid; v < (V >> 3); v += SEL_THREADS) ldst[v] = lsrc[v];
  for (int j = (V & ~7) + tid; j < V; j += SEL_THREADS) next_logits[(size_t)g * ldn + j] = logits[(size_t)r * ldl + j];
  __syncthreads();  // every thread has read pos[g * k] (L) before it moves
  if (tid < k) pos[(size_t)g * k + tid] = L + 1;
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1u) == (unsigned int)(B - 1)) {  // every CTA has read *step
      *ticket = 0u;
      *step += 1;
    }
  }
}

}  // namespace contrastive
}  // namespace srgpt

using namespace srgpt;
using namespace srgpt::contrastive;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" __attribute__((visibility("default"))) long long srgpt_contrastive_partial_floats(int B, int k, int L_cap) {
  if (B <= 0 || k <= 0 || L_cap <= 0) return -1;
  return (long long)B * ((L_cap + CHUNK - 1) / CHUNK) * k;
}

extern "C" __attribute__((visibility("default"))) int srgpt_contrastive_penalty_bf16(const void* cand, int ldc, const void* ctx, int L_cap, int H,
                                                                                     const int* pos, int B, int k, float* partial, void* stream) {
  SRGPT_CHECK_ARG(cand && ctx && pos && partial && B > 0 && B <= 65535 && k >= 1 && k <= K_MAX && L_cap > 0 && H > 0 && (H % 8) == 0);
  SRGPT_CHECK_ARG(ldc >= H && (ldc % 8) == 0 && aligned16(cand) && aligned16(ctx));
  const int smem = KC * H * (int)sizeof(bf16);
  SRGPT_CHECK_ARG(smem <= PEN_SMEM_MAX);
  static bool configured = false;
  if (!configured) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(penalty_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PEN_SMEM_MAX));
    configured = true;
  }
  const int n_chunks = (L_cap + CHUNK - 1) / CHUNK;
  penalty_kernel<<<dim3(n_chunks, B), PEN_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(cand), ldc, reinterpret_cast<const bf16*>(ctx), L_cap, H, pos, k, partial, n_chunks);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_contrastive_select_bf16(
    const float* cand_scores, const int* cand_tokens, const float* partial, const float* alpha, const void* xn, int ldx, int H,
    const void* logits, int ldl, int V, void* ctx, int L_cap, void* next_logits, int ldn, int* pos, int B, int k, long long* out_ids, int* step,
    void* ticket, int* sel, float* pen, float* score, void* stream) {
  SRGPT_CHECK_ARG(cand_scores && cand_tokens && partial && alpha && xn && logits && ctx && next_logits && pos && out_ids && step && ticket && sel &&
                  pen && score);
  SRGPT_CHECK_ARG(B > 0 && k >= 1 && k <= K_MAX && H > 0 && (H % 8) == 0 && V > 0 && L_cap > 0);
  SRGPT_CHECK_ARG(ldx >= H && ldl >= V && ldn >= V && (ldx % 8) == 0 && (ldl % 8) == 0 && (ldn % 8) == 0);
  SRGPT_CHECK_ARG(aligned16(xn) && aligned16(logits) && aligned16(ctx) && aligned16(next_logits));
  select_kernel<<<B, SEL_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      cand_scores, cand_tokens, partial, (L_cap + CHUNK - 1) / CHUNK, alpha, reinterpret_cast<const bf16*>(xn), ldx, H,
      reinterpret_cast<const bf16*>(logits), ldl, V, reinterpret_cast<bf16*>(ctx), L_cap, reinterpret_cast<bf16*>(next_logits), ldn, pos, k, B,
      out_ids, step, reinterpret_cast<unsigned int*>(ticket), sel, pen, score);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
