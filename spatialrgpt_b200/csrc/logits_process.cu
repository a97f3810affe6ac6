// HF's logits processors on the device: repetition penalty, no-repeat n-grams, bad words and the minimum length, applied to R rows of
// next-token logits, followed by the greedy choice over the processed rows.
//
// Reference: the generation kwargs the reference forwards to HF generate() (llava/model/language_model/llava_llama.py:212,
// `self.llm.generate(inputs_embeds=..., **generation_kwargs)`; llava/eval/model_vqa.py:76 carries `no_repeat_ngram_size=3`); the
// arithmetic is transformers' RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor (a
// SequenceBiasLogitsProcessor with a -inf bias), MinLengthLogitsProcessor and MinNewTokensLengthLogitsProcessor, in the order
// _get_logits_processor builds them.  HF is called with inputs_embeds, so its input_ids are the generated tokens only: the history
// here is the generated ids already in device memory (out_ids of the one-token step, the [step, B] table of the batched step).
//
// One CTA per (4096-column segment, row) - the grid of argmax_wide_kernel.  Each CTA scans the row's history for the tokens that
// fall into its segment and marks them in three 512-byte shared bitmaps:
//   pen  - tokens of the history (the repetition penalty, once per distinct token: a bitmap has no write race and no duplicates),
//   bad  - bad-word bans (HF adds a -inf bias: scores + bias, which also turns -0.0 into +0.0 wherever the processor is on),
//   kill - n-gram bans and the EOS ids below the minimum length (HF assigns -inf).
// Then it rewrites its segment in processor order and feeds the arg max key of rowops.cu (max value, lowest index on ties, NaN
// never wins) into a 64-bit atomicMax per row.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace logits_process {

constexpr int THREADS = 256;
constexpr int WORDS = ARGMAX_SEG / 32;
enum : int { F_PENALTY = 1, F_NGRAM = 2, F_BAD = 4, F_MINLEN = 8 };

__device__ __forceinline__ void mark(unsigned int* map, long long tok, int c0) {
  const long long d = tok - c0;
  if (d >= 0 && d < ARGMAX_SEG) atomicOr(map + (d >> 5), 1u << (d & 31));
}
__device__ __forceinline__ bool in_seg(long long tok, int c0) { return tok >= c0 && tok < (long long)c0 + ARGMAX_SEG; }

__device__ __forceinline__ float load_logit(const float* p) { return *p; }
__device__ __forceinline__ float load_logit(const bf16* p) { return e2f(*p); }

// spec (int32, device) = {flags, n-gram size, minimum new tokens, n_eos, n_bad, eos[n_eos], bad_off[n_bad + 1], bad_tok[...]};
// fparams = {penalty, 1 / penalty} (fp32, the reciprocal rounded as ATen's CUDA division by a scalar rounds it).
template <typename T>
__global__ void __launch_bounds__(THREADS)
logits_process_kernel(const T* __restrict__ logits, int ld, int V, const long long* __restrict__ hist, int hist_row_stride,
                      int hist_tok_stride, int hist_cap, const int* __restrict__ step, int step_offset, const float* __restrict__ fparams,
                      const int* __restrict__ spec, int spec_cap, float* __restrict__ out, int ldo, unsigned long long* __restrict__ keys) {
  __shared__ unsigned int s_pen[WORDS], s_bad[WORDS], s_kill[WORDS];
  __shared__ unsigned long long sk[THREADS / 32];
  const int tid = threadIdx.x, r = blockIdx.y;
  const int c0 = blockIdx.x * ARGMAX_SEG, c1 = min(V, c0 + ARGMAX_SEG);
  const long long* h = hist + (size_t)r * hist_row_stride;
  const size_t ts = (size_t)hist_tok_stride;
  const int n = max(0, min((step != nullptr ? *step : 0) + step_offset, hist_cap));  // tokens generated so far
  const int flags = spec[0];
  for (int i = tid; i < WORDS; i += THREADS) {
    s_pen[i] = 0u;
    s_bad[i] = 0u;
    s_kill[i] = 0u;
  }
  __syncthreads();
  if (flags & F_PENALTY)
    for (int t = tid; t < n; t += THREADS) mark(s_pen, h[t * ts], c0);
  if (flags & F_NGRAM) {
    // fairseq's rule (_calc_banned_ngram_tokens): ban the token that followed every earlier occurrence of the last g - 1 tokens
    const int g = spec[1];
    for (int i = tid; i + g <= n; i += THREADS) {
      const long long tok = h[(size_t)(i + g - 1) * ts];
      if (!in_seg(tok, c0)) continue;
      bool eq = true;
      for (int j = 0; j < g - 1 && eq; ++j) eq = h[(size_t)(i + j) * ts] == h[(size_t)(n - g + 1 + j) * ts];
      if (eq) mark(s_kill, tok, c0);
    }
  }
  const int n_eos = min(spec[3], max(0, spec_cap - 5));
  if (flags & F_BAD) {
    const int nb = spec[4];
    const int* off = spec + 5 + n_eos;
    const int* toks = off + nb + 1;
    for (int j = tid; j < nb; j += THREADS) {
      const int a = off[j], L = off[j + 1] - a;
      const int last = toks[a + L - 1];
      if (!in_seg(last, c0)) continue;
      if (L > 1) {
        if (L > n) continue;  // HF skips a sequence longer than the history (not L - 1)
        bool eq = true;
        for (int q = 0; q < L - 1 && eq; ++q) eq = h[(size_t)(n - L + 1 + q) * ts] == (long long)toks[a + q];
        if (!eq) continue;
      }
      mark(s_bad, last, c0);
    }
  }
  if ((flags & F_MINLEN) && n < spec[2])
    for (int j = tid; j < n_eos; j += THREADS) mark(s_kill, spec[5 + j], c0);
  __syncthreads();

  const float pen = fparams[0], inv_pen = fparams[1];
  const bool bad_on = (flags & F_BAD) != 0;
  const T* row = logits + (size_t)r * ld;
  float* orow = out != nullptr ? out + (size_t)r * ldo : nullptr;
  unsigned long long best = 0ull;
  for (int c = c0 + tid; c < c1; c += THREADS) {
    float v = load_logit(row + c);
    const int d = c - c0;
    const unsigned int bit = 1u << (d & 31);
    if (s_pen[d >> 5] & bit) v = v < 0.f ? v * pen : v * inv_pen;
    if (bad_on) v = v + ((s_bad[d >> 5] & bit) ? -INFINITY : 0.f);
    if (s_kill[d >> 5] & bit) v = -INFINITY;
    if (orow != nullptr) orow[c] = v;
    if (v == v) {
      const unsigned long long k = ((unsigned long long)float_order_bits(v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)c);
      best = k > best ? k : best;
    }
  }
  if (keys == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ok = __shfl_xor_sync(0xffffffffu, best, o);
    best = ok > best ? ok : best;
  }
  if ((tid & 31) == 0) sk[tid >> 5] = best;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < THREADS / 32; ++w) best = sk[w] > best ? sk[w] : best;
    atomicMax(keys + r, best);
  }
}

// the one-token step's bookkeeping after processing: out_ids[*step + step_offset] = the processed choice, next_x = its embedding row
__global__ void __launch_bounds__(256)
logits_pick_kernel(const long long* __restrict__ ids, const int* __restrict__ step, int step_offset, long long* __restrict__ out_ids,
                   const bf16* __restrict__ embed_table, bf16* __restrict__ next_x, int K) {
  const long long tok = ids[0];
  if (threadIdx.x == 0) out_ids[*step + step_offset] = tok;
  if (embed_table != nullptr) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)tok * K);
    for (int c = threadIdx.x; c < (K >> 3); c += blockDim.x) reinterpret_cast<uint4*>(next_x)[c] = src[c];
  }
}

}  // namespace logits_process
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_logits_process(const void* logits, int logits_f32, int ld, int rows, int V,
                                                                           const long long* hist, int hist_row_stride, int hist_tok_stride,
                                                                           int hist_cap, const int* step, int step_offset, const float* fparams,
                                                                           const int* spec, int spec_cap, float* out, int ldo, long long* ids,
                                                                           void* stream) {
  SRGPT_CHECK_ARG(logits && fparams && spec && rows > 0 && rows <= 65535 && V > 0 && ld >= V && spec_cap >= 5);
  SRGPT_CHECK_ARG(logits_f32 == 0 || logits_f32 == 1);
  SRGPT_CHECK_ARG(out != nullptr || ids != nullptr);
  SRGPT_CHECK_ARG(out == nullptr || ldo >= V);
  SRGPT_CHECK_ARG(hist_cap >= 0 && (hist_cap == 0 || (hist != nullptr && hist_tok_stride > 0 && hist_row_stride >= 0)));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ids != nullptr) SRGPT_CHECK_CUDA(cudaMemsetAsync(ids, 0, (size_t)rows * sizeof(long long), st));
  const dim3 grid(ceil_div(V, ARGMAX_SEG), rows);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(ids);
  const long long* h = hist_cap > 0 ? hist : nullptr;
  if (logits_f32)
    logits_process::logits_process_kernel<float><<<grid, logits_process::THREADS, 0, st>>>(
        reinterpret_cast<const float*>(logits), ld, V, h, hist_row_stride, hist_tok_stride, hist_cap, step, step_offset, fparams, spec,
        spec_cap, out, ldo, keys);
  else
    logits_process::logits_process_kernel<bf16><<<grid, logits_process::THREADS, 0, st>>>(
        reinterpret_cast<const bf16*>(logits), ld, V, h, hist_row_stride, hist_tok_stride, hist_cap, step, step_offset, fparams, spec,
        spec_cap, out, ldo, keys);
  SRGPT_CHECK_LAUNCH();
  if (ids != nullptr) {
    argmax_unpack(ids, rows, st);
    SRGPT_CHECK_LAUNCH();
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_logits_pick_token(const long long* ids, const int* step, int step_offset,
                                                                              long long* out_ids, const void* embed_table, void* next_x, int K,
                                                                              void* stream) {
  SRGPT_CHECK_ARG(ids && step && out_ids);
  SRGPT_CHECK_ARG((embed_table == nullptr) == (next_x == nullptr));
  SRGPT_CHECK_ARG(embed_table == nullptr || ((K % 8) == 0 && K > 0 && (reinterpret_cast<uintptr_t>(embed_table) & 15) == 0 &&
                                             (reinterpret_cast<uintptr_t>(next_x) & 15) == 0));
  logits_process::logits_pick_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      ids, step, step_offset, out_ids, reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(next_x), K);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
