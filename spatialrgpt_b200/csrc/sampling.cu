// Temperature / nucleus (top-p) sampling of the next token from one row of fp32 logits, on the device.
//
// Reference: the generation kwargs the reference's callers pass to HF generate() when temperature > 0 - do_sample=True,
// temperature, top_p (llava/eval/eval_spatial.py:231-236, llava/eval/model_vqa.py:72-78, demo/gradio_web_server_multi.py:208-212);
// the arithmetic is HF's TemperatureLogitsWarper + TopPLogitsWarper + multinomial (third party, transformers 4.37.2):
//   scores = logits / T;  keep the top_k scores (GenerationConfig default 50);  p = softmax over them;  keep the smallest set of
//   highest-probability tokens whose mass reaches top_p (at least one token);  renormalise;  draw one token.
// HF sorts the whole vocabulary every step; here ONE 1024-thread CTA makes a few passes over the 128 K logits (L2 resident):
//   max -> normaliser -> the top-k and nucleus cuts by exact searches over the logits' 32-bit keys (sample_row)
//   -> a draw u * mass(kept set) located with a block prefix sum over index-ordered chunks.
// The draw uses a counter-based generator (splitmix64 of seed and step), so a request is reproducible given its seed; it is
// NOT torch's Philox stream, so sampled ids are comparable with the reference in distribution only (tests check the support and
// the frequencies against the torch nucleus).  Greedy decoding (the graded mode) never runs this kernel.
// A batch of sequences draws in one launch of sample_rows_kernel: one such CTA per row, the same arithmetic (sample_row) over fp32 rows or
// the element-type rows of the batched lm_head, each row with its own seed.
// The *_warped kernels add HF's TypicalLogitsWarper, EpsilonLogitsWarper and EtaLogitsWarper (transformers 5.5, same in 4.37.2) after
// top-p, in HF's order, as sample_row<T, true>; sample_row<T, false> is the original arithmetic, which the original kernels keep.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace sampling {

constexpr int THREADS = 1024;

__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < (THREADS >> 5)) ? red[lane] : -INFINITY;
  return warp_max(t);
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < (THREADS >> 5)) ? red[lane] : 0.f;
  return warp_sum(t);
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ float logit(const float* __restrict__ x, int i) { return x[i]; }
__device__ __forceinline__ float logit(const bf16* __restrict__ x, int i) { return e2f(x[i]); }  // exact: torch's .float() of the row

// Order-preserving 32-bit key of a float (a <= b iff key(a) <= key(b) for non-NaN a, b; -0 folded into +0, which compare equal).
__device__ __forceinline__ unsigned key_of(float x) {
  const unsigned u = __float_as_uint(__fadd_rn(x, 0.f));
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float of_key(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// The smallest logit whose fl(x / t) reaches fl(xc / t): the cut at logit xc widened over every token HF's x / T ties with it
// (x -> fl(x / t) is monotone for t > 0 but not one-to-one, so distinct logits can share a scaled value).
template <typename T>
__device__ __forceinline__ float widen_cut(const T* __restrict__ logits, int V, float xc, float t, float* red) {
  const float sc = __fdiv_rn(xc, t);
  float lo = xc;
  for (int i = threadIdx.x; i < V; i += THREADS) {
    const float x = logit(logits, i);
    if (x < lo && __fdiv_rn(x, t) >= sc) lo = x;
  }
  return -block_reduce_max(-lo, red);
}

// Whether the token of logit x and probability p is in the set the draw picks from: x >= x_keep (top-k and top-p), and with CUTS
// the typical / epsilon / eta cuts of sample_row, whose state s_cut = {c, d*, top logit of K1, p cut} it computes.
template <bool CUTS>
__device__ __forceinline__ bool kept(float x, float p, float m, float inv_t, float x_keep, const float* s_cut) {
  if constexpr (CUTS) return x >= x_keep && fabsf(s_cut[0] - (x - m) * inv_t) <= s_cut[1] && (x >= s_cut[2] || p >= s_cut[3]);
  else return x >= x_keep;
}

// The draw of one row of V logits (fp32 or the element type) by the whole 1024-thread CTA; every thread returns the token.
// params = {temperature, top_p, top_k (0 = off)} and the seed live in device memory, so one captured CUDA graph serves any request.
// CUTS: params = {temperature, top_p, top_k, typical_p, epsilon, eta}; a warper acts where HF turns it on (typical_p < 1,
// 0 < epsilon < 1, 0 < eta < 1) on the set the earlier cuts kept, and the draw and the warped row use the final set.
template <typename T, bool CUTS = false>
__device__ __forceinline__ int sample_row(const T* __restrict__ logits, int V, const float* __restrict__ params,
                                          const unsigned long long* __restrict__ seed_ptr, const int* __restrict__ step, int step_offset,
                                          float* __restrict__ warped) {
  __shared__ float red[32];
  __shared__ float s_scan[THREADS];
  __shared__ int s_tok;
  const float inv_t = 1.0f / fmaxf(params[0], 1e-6f);
  const float top_p = params[1];
  const int top_k = (int)params[2];
  const int tid = threadIdx.x;
  // contiguous chunk of the vocabulary per thread (index order matters for the final walk)
  const int per = (V + THREADS - 1) / THREADS;
  const int lo = min(V, tid * per), hi = min(V, lo + per);

  float m = -INFINITY;
  for (int i = lo; i < hi; ++i) m = fmaxf(m, logit(logits, i));
  m = block_reduce_max(m, red);
  float z = 0.f;
  for (int i = lo; i < hi; ++i) z += __expf((logit(logits, i) - m) * inv_t);
  z = block_reduce_sum(z, red);
  const float inv_z = 1.0f / z;

  // The cuts select on logit keys, exactly: HF compares fl(x / T), which is monotone in x, so the k-th largest x / T is fl(x_k / T) of
  // the k-th largest logit x_k, and a cut at logit xc keeps {fl(x / T) >= fl(xc / T)} = {x >= widen_cut(xc)}.  (A cut on the probability
  // value cannot tell apart probabilities below its resolution, nor the probabilities that underflow to 0 where HF keeps finite scores.)
  // The key searches count in index-strided order (integer counts do not depend on it); the masses the draw uses are summed per chunk.
  // top-k first (HF's warper order: temperature, top_k, top_p; GenerationConfig's default top_k is 50): the k-th largest key, found bit
  // by bit from the top (the largest c with count{key >= c} >= k); every token tied with it in x / T stays in.
  const float t = params[0];
  float x_floor = -INFINITY, mass_floor = 1.f;
  if (top_k > 0 && top_k < V) {
    unsigned c = 0u;
    for (int b = 31; b >= 0; --b) {
      const unsigned cand = c | (1u << b);
      float n = 0.f;
      for (int i = tid; i < V; i += THREADS) n += key_of(logit(logits, i)) >= cand ? 1.f : 0.f;
      if (block_reduce_sum(n, red) >= (float)top_k) c = cand;
    }
    x_floor = widen_cut(logits, V, of_key(c), t, red);
    float s = 0.f;
    for (int i = lo; i < hi; ++i) {
      const float x = logit(logits, i);
      s += (x >= x_floor) ? __expf((x - m) * inv_t) * inv_z : 0.f;
    }
    mass_floor = block_reduce_sum(s, red);
  }
  // nucleus inside the top-k set: the largest key c with mass{key >= c} >= top_p * mass(top-k set), searched over the bits below the
  // common prefix of the top-k cut's key and the top logit's key (c lies between them); the top logit is always kept (>= 1 token).
  float x_keep = x_floor, mass = mass_floor;
  if (top_p < 1.0f) {
    const float target = top_p * mass_floor;
    const unsigned kf = key_of(x_floor), km = key_of(m);
    unsigned c = kf;
    if (kf != km) {
      const int hb = 31 - __clz(kf ^ km);
      c = kf & ~((2u << hb) - 1u);  // the common prefix (hb = 31: none)
      for (int b = hb; b >= 0; --b) {
        const unsigned cand = c | (1u << b), cut = max(cand, kf);
        float s = 0.f;
        for (int i = tid; i < V; i += THREADS) {
          const float x = logit(logits, i);
          s += key_of(x) >= cut ? __expf((x - m) * inv_t) * inv_z : 0.f;
        }
        if (block_reduce_sum(s, red) >= target) c = cand;
      }
      c = min(max(c, kf), km);
    }
    x_keep = widen_cut(logits, V, of_key(c), t, red);
    float s = 0.f;
    for (int i = lo; i < hi; ++i) {
      const float x = logit(logits, i);
      s += (x >= x_keep) ? __expf((x - m) * inv_t) * inv_z : 0.f;
    }
    mass = block_reduce_sum(s, red);
  }

  // Typical, epsilon and eta cuts (CUTS) over the kept set K0 = {x >= x_keep}, each on what the previous one left.  With s = the scaled
  // logit (x - m) / T and q = p / mass(K0), -log q - H = E_q[s] - s, so typical's deviation is |c - s| with c = E_q[s]; the kept set is
  // {|c - s| <= d*}, d* the smallest deviation whose set reaches typical_p of the mass (HF keeps every token up to the deviation at
  // which the sorted cumulative mass first reaches typical_p, ties included), found by bisection on d.  Epsilon keeps
  // p >= epsilon * mass(K1); eta keeps p >= min(eta, sqrt(eta) * exp(-H2)) * mass(K2), H2 the entropy of K2; both keep the tokens
  // tied at the largest logit of K1 (HF's min_tokens_to_keep = 1).  All cuts together: kept<true>.
  __shared__ float s_cut[4];  // c, d*, the top logit of K1 and the p cut, read by kept() (the kernel has no registers to spare)
  if constexpr (CUTS) {  // the loops unroll by 8: the factor at which the three kernels fit 64 registers without local memory
    float c_typ = 0.f, d_keep = INFINITY, x_top = -INFINITY, cut = 0.f;
    const float typical_p = params[3], eps = params[4], eta = params[5];
    const bool typ_on = typical_p < 1.0f, eps_on = eps > 0.f && eps < 1.0f, eta_on = eta > 0.f && eta < 1.0f;
    if (typ_on) {
      float a = 0.f, b = 0.f;
      #pragma unroll 8
      for (int i = lo; i < hi; ++i) {
        const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
        if (x >= x_keep && p > 0.f) { a += p; b += p * s; }
      }
      const float a0 = block_reduce_sum(a, red);
      c_typ = block_reduce_sum(b, red) / a0;
      float dm = 0.f;
      #pragma unroll 8
      for (int i = lo; i < hi; ++i) {
        const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
        if (x >= x_keep && p > 0.f) dm = fmaxf(dm, fabsf(c_typ - s));
      }
      float lo_d = 0.f, hi_d = block_reduce_max(dm, red);  // invariant: mass{|c - s| <= hi_d} >= typical_p * a0
      const float target = typical_p * a0;
      for (int it = 0; it < 26; ++it) {
        const float mid = 0.5f * (lo_d + hi_d);
        float sm = 0.f;
        #pragma unroll 8
        for (int i = lo; i < hi; ++i) {
          const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
          sm += (x >= x_keep && p > 0.f && fabsf(c_typ - s) <= mid) ? p : 0.f;
        }
        sm = block_reduce_sum(sm, red);
        if (sm >= target) hi_d = mid; else lo_d = mid;
      }
      d_keep = hi_d;
    }
    if (eps_on || eta_on) {
      float a = 0.f, xm = -INFINITY;
      #pragma unroll 8
      for (int i = lo; i < hi; ++i) {
        const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
        if (x >= x_keep && fabsf(c_typ - s) <= d_keep) { a += p; xm = fmaxf(xm, x); }
      }
      const float a1 = block_reduce_sum(a, red);
      x_top = block_reduce_max(xm, red);
      if (eps_on) cut = eps * a1;
      if (eta_on) {
        float a2 = 0.f, b2 = 0.f;
        #pragma unroll 8
        for (int i = lo; i < hi; ++i) {
          const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
          if (x >= x_keep && p > 0.f && fabsf(c_typ - s) <= d_keep && (x >= x_top || p >= cut)) { a2 += p; b2 += p * s; }
        }
        a2 = block_reduce_sum(a2, red);
        b2 = block_reduce_sum(b2, red);
        const float h2 = __logf(a2 / inv_z) - b2 / a2;  // entropy of K2: E_q[-log q], -log q = log(z * mass) - s
        cut = fmaxf(cut, fminf(eta, sqrtf(eta) * __expf(-h2)) * a2);
      }
    }
    if (typ_on || eps_on || eta_on) {
      float sm = 0.f;
      #pragma unroll 8
      for (int i = lo; i < hi; ++i) {
        const float x = logit(logits, i), s = (x - m) * inv_t, p = __expf(s) * inv_z;
        sm += (x >= x_keep && fabsf(c_typ - s) <= d_keep && (x >= x_top || p >= cut)) ? p : 0.f;
      }
      mass = block_reduce_sum(sm, red);
    }
    if (tid == 0) { s_cut[0] = c_typ; s_cut[1] = d_keep; s_cut[2] = x_top; s_cut[3] = cut; }
    __syncthreads();
  }

  // the warped row (HF's output_scores of a sampled step): logits / T for the tokens the draw can pick (the set the top-k cut, the
  // nucleus and the CUTS kept), -inf for every other token.  A true fp32 division, as TemperatureLogitsWarper divides.
  if (warped != nullptr) {
    for (int i = tid; i < V; i += THREADS) {
      const float x = logit(logits, i);
      warped[i] = kept<CUTS>(x, __expf((x - m) * inv_t) * inv_z, m, inv_t, x_keep, s_cut) ? __fdiv_rn(x, t) : -INFINITY;
    }
  }

  // draw
  const unsigned long long ctr = (unsigned long long)(*step + step_offset);
  const unsigned long long r = splitmix64(*seed_ptr ^ splitmix64(ctr));
  const float u = ((float)(r >> 40) + 0.5f) * (1.0f / 16777216.0f) * mass;  // (0, mass)
  float local = 0.f;
  for (int i = lo; i < hi; ++i) {
    const float x = logit(logits, i), p = __expf((x - m) * inv_t) * inv_z;
    local += kept<CUTS>(x, p, m, inv_t, x_keep, s_cut) ? p : 0.f;
  }
  s_scan[tid] = local;
  __syncthreads();
  // inclusive scan over the 1024 chunk masses (Hillis-Steele; 10 steps)
  for (int off = 1; off < THREADS; off <<= 1) {
    const float add = tid >= off ? s_scan[tid - off] : 0.f;
    __syncthreads();
    s_scan[tid] += add;
    __syncthreads();
  }
  if (tid == 0) s_tok = -1;
  __syncthreads();
  const float before = tid == 0 ? 0.f : s_scan[tid - 1];
  const float total = s_scan[THREADS - 1];
  const float uu = fminf(u, total * 0.99999994f);  // rounding of the chunk-summed mass vs the scan total
  if (uu >= before && uu < s_scan[tid] && hi > lo) {
    float acc = before;
    int pick = -1, last_kept = -1;
    for (int i = lo; i < hi; ++i) {
      const float x = logit(logits, i), p = __expf((x - m) * inv_t) * inv_z;
      if (p > 0.f && kept<CUTS>(x, p, m, inv_t, x_keep, s_cut)) {  // a kept token of p = 0 (exp underflow, -inf) is never drawn
        last_kept = i;
        acc += p;
        if (acc > uu) { pick = i; break; }
      }
    }
    s_tok = pick >= 0 ? pick : last_kept;
  }
  __syncthreads();
  int tok = s_tok;
  if (tok < 0) {  // numerically impossible corner (all chunk boundaries missed): fall back to the arg max
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = lo; i < hi; ++i)
      if (logit(logits, i) > best) { best = logit(logits, i); bi = i; }
    __shared__ float sb[THREADS];
    __shared__ int si[THREADS];
    sb[tid] = best; si[tid] = bi;
    __syncthreads();
    if (tid == 0) {
      for (int k = 1; k < THREADS; ++k)
        if (sb[k] > best || (sb[k] == best && si[k] < bi)) { best = sb[k]; bi = si[k]; }
      s_tok = bi == 0x7fffffff ? 0 : bi;
    }
    __syncthreads();
    tok = s_tok;
  }
  return tok;
}

__global__ void __launch_bounds__(THREADS, 1)
sample_top_p_kernel(const float* __restrict__ logits, int V, const float* __restrict__ params, const unsigned long long* __restrict__ seed_ptr, const int* __restrict__ step,
                    int step_offset, long long* __restrict__ out_ids, const bf16* __restrict__ embed_table, bf16* __restrict__ next_x, int K,
                    float* __restrict__ scores, long long step_stride) {
  float* warped = scores != nullptr ? scores + (long long)(*step + step_offset) * step_stride : nullptr;
  const int tok = sample_row(logits, V, params, seed_ptr, step, step_offset, warped);
  if (threadIdx.x == 0) out_ids[*step + step_offset] = (long long)tok;
  if (embed_table != nullptr && next_x != nullptr) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)tok * K);
    for (int c = threadIdx.x; c < (K >> 3); c += THREADS) reinterpret_cast<uint4*>(next_x)[c] = src[c];
  }
}

// R rows at once, one CTA per row: row r = logits + r * ld draws with seeds[r] at counter *step + step_offset -> ids[r].
// Each row's token is the one sample_top_p_kernel draws from that row in fp32 with the same seed and counter.
template <typename T>
__global__ void __launch_bounds__(THREADS, 1)
sample_rows_kernel(const T* __restrict__ logits, long long ld, int V, const float* __restrict__ params, const unsigned long long* __restrict__ seeds,
                   const int* __restrict__ step, int step_offset, long long* __restrict__ ids, float* __restrict__ scores, long long step_stride) {
  const int r = blockIdx.x;
  float* warped = scores != nullptr ? scores + (long long)(*step + step_offset) * step_stride + (long long)r * V : nullptr;
  const int tok = sample_row(logits + (size_t)r * ld, V, params, seeds + r, step, step_offset, warped);
  if (threadIdx.x == 0) ids[r] = (long long)tok;
}

// sample_top_p_kernel and sample_rows_kernel with the typical / epsilon / eta cuts (params float[6]).
__global__ void __launch_bounds__(THREADS, 1)
sample_top_p_warped_kernel(const float* __restrict__ logits, int V, const float* __restrict__ params, const unsigned long long* __restrict__ seed_ptr,
                           const int* __restrict__ step, int step_offset, long long* __restrict__ out_ids, const bf16* __restrict__ embed_table,
                           bf16* __restrict__ next_x, int K, float* __restrict__ scores, long long step_stride) {
  float* warped = scores != nullptr ? scores + (long long)(*step + step_offset) * step_stride : nullptr;
  const int tok = sample_row<float, true>(logits, V, params, seed_ptr, step, step_offset, warped);
  if (threadIdx.x == 0) out_ids[*step + step_offset] = (long long)tok;
  if (embed_table != nullptr && next_x != nullptr) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)tok * K);
    for (int c = threadIdx.x; c < (K >> 3); c += THREADS) reinterpret_cast<uint4*>(next_x)[c] = src[c];
  }
}

template <typename T>
__global__ void __launch_bounds__(THREADS, 1)
sample_rows_warped_kernel(const T* __restrict__ logits, long long ld, int V, const float* __restrict__ params, const unsigned long long* __restrict__ seeds,
                          const int* __restrict__ step, int step_offset, long long* __restrict__ ids, float* __restrict__ scores, long long step_stride) {
  const int r = blockIdx.x;
  float* warped = scores != nullptr ? scores + (long long)(*step + step_offset) * step_stride + (long long)r * V : nullptr;
  const int tok = sample_row<T, true>(logits + (size_t)r * ld, V, params, seeds + r, step, step_offset, warped);
  if (threadIdx.x == 0) ids[r] = (long long)tok;
}

}  // namespace sampling
}  // namespace srgpt

using namespace srgpt;

namespace {
int launch_sample_top_p(const float* logits, int V, const float* params, const unsigned long long* seed, const int* step, int step_offset,
                        long long* out_ids, const void* embed_table, void* next_x, int K, float* scores, long long step_stride, void* stream,
                        bool cuts = false) {
  SRGPT_CHECK_ARG(logits && params && seed && step && out_ids && V > 0);
  SRGPT_CHECK_ARG((embed_table == nullptr) == (next_x == nullptr));
  SRGPT_CHECK_ARG(embed_table == nullptr || ((K % 8) == 0 && K > 0 && (reinterpret_cast<uintptr_t>(embed_table) & 15) == 0 &&
                                             (reinterpret_cast<uintptr_t>(next_x) & 15) == 0));
  SRGPT_CHECK_ARG(scores == nullptr || step_stride >= V);
  (cuts ? sampling::sample_top_p_warped_kernel : sampling::sample_top_p_kernel)<<<1, sampling::THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, V, params, seed, step, step_offset, out_ids, reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(next_x), K,
      scores, step_stride);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

int launch_sample_rows(const void* logits, int logits_f32, int ld, int R, int V, const float* params, const unsigned long long* seeds,
                       const int* step, int step_offset, long long* ids, float* scores, long long step_stride, void* stream, bool cuts = false) {
  SRGPT_CHECK_ARG(logits && params && seeds && step && ids && R > 0 && R <= 65535 && V > 0 && ld >= V);
  SRGPT_CHECK_ARG(logits_f32 == 0 || logits_f32 == 1);
  SRGPT_CHECK_ARG(scores == nullptr || step_stride >= (long long)R * V);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (logits_f32)
    (cuts ? sampling::sample_rows_warped_kernel<float> : sampling::sample_rows_kernel<float>)<<<R, sampling::THREADS, 0, st>>>(
        reinterpret_cast<const float*>(logits), ld, V, params, seeds, step, step_offset, ids, scores, step_stride);
  else
    (cuts ? sampling::sample_rows_warped_kernel<bf16> : sampling::sample_rows_kernel<bf16>)<<<R, sampling::THREADS, 0, st>>>(
        reinterpret_cast<const bf16*>(logits), ld, V, params, seeds, step, step_offset, ids, scores, step_stride);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
}  // namespace

// Overwrites out_ids[*step + step_offset] (and, when given, next_x = embed_table[token]) with a token sampled from
// softmax(logits / temperature) restricted to its top-p nucleus.  `params` = device float[3] {temperature, top_p, top_k (0 = off)},
// `seed` = device u64 (read at run time: a captured graph must not freeze the seed of the request it was captured under).
// Called right after srgpt_lm_head_argmax_bf16 (which already advanced *step): step_offset = -1.
extern "C" __attribute__((visibility("default"))) int srgpt_sample_top_p_f32(const float* logits, int V, const float* params, const unsigned long long* seed,
                                                                             const int* step, int step_offset, long long* out_ids,
                                                                             const void* embed_table, void* next_x, int K, void* stream) {
  return launch_sample_top_p(logits, V, params, seed, step, step_offset, out_ids, embed_table, next_x, K, nullptr, 0, stream);
}

// The same draw, and the warped row it drew from -> scores + (*step + step_offset) * step_stride.
extern "C" __attribute__((visibility("default"))) int srgpt_sample_top_p_scores_f32(const float* logits, int V, const float* params,
                                                                                    const unsigned long long* seed, const int* step, int step_offset,
                                                                                    long long* out_ids, const void* embed_table, void* next_x, int K,
                                                                                    float* scores, long long step_stride, void* stream) {
  SRGPT_CHECK_ARG(scores != nullptr);
  return launch_sample_top_p(logits, V, params, seed, step, step_offset, out_ids, embed_table, next_x, K, scores, step_stride, stream);
}

// Draws one token per row for R rows of logits [R, ld] (fp32 when logits_f32, else the element type) -> ids[R].  Row r draws with
// seeds[r] at counter *step + step_offset, exactly as srgpt_sample_top_p_f32 draws from that row converted to fp32.
extern "C" __attribute__((visibility("default"))) int srgpt_sample_rows(const void* logits, int logits_f32, int ld, int R, int V, const float* params,
                                                                        const unsigned long long* seeds, const int* step, int step_offset,
                                                                        long long* ids, void* stream) {
  return launch_sample_rows(logits, logits_f32, ld, R, V, params, seeds, step, step_offset, ids, nullptr, 0, stream);
}

// The same draws, and row r's warped row -> scores + (*step + step_offset) * step_stride + r * V.
extern "C" __attribute__((visibility("default"))) int srgpt_sample_rows_scores(const void* logits, int logits_f32, int ld, int R, int V,
                                                                               const float* params, const unsigned long long* seeds, const int* step,
                                                                               int step_offset, long long* ids, float* scores, long long step_stride,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(scores != nullptr);
  return launch_sample_rows(logits, logits_f32, ld, R, V, params, seeds, step, step_offset, ids, scores, step_stride, stream);
}

// The same four entry points with HF's typical, epsilon and eta warpers after top-p: `params` = device float[6] {temperature, top_p,
// top_k (0 = off), typical_p (>= 1 = off), epsilon_cutoff, eta_cutoff (each off outside (0, 1))}.  With all three off the draw and the
// warped row are those of the float[3] entry points.
extern "C" __attribute__((visibility("default"))) int srgpt_sample_warped_f32(const float* logits, int V, const float* params, const unsigned long long* seed,
                                                                              const int* step, int step_offset, long long* out_ids,
                                                                              const void* embed_table, void* next_x, int K, void* stream) {
  return launch_sample_top_p(logits, V, params, seed, step, step_offset, out_ids, embed_table, next_x, K, nullptr, 0, stream, true);
}

extern "C" __attribute__((visibility("default"))) int srgpt_sample_warped_scores_f32(const float* logits, int V, const float* params,
                                                                                     const unsigned long long* seed, const int* step, int step_offset,
                                                                                     long long* out_ids, const void* embed_table, void* next_x, int K,
                                                                                     float* scores, long long step_stride, void* stream) {
  SRGPT_CHECK_ARG(scores != nullptr);
  return launch_sample_top_p(logits, V, params, seed, step, step_offset, out_ids, embed_table, next_x, K, scores, step_stride, stream, true);
}

extern "C" __attribute__((visibility("default"))) int srgpt_sample_rows_warped(const void* logits, int logits_f32, int ld, int R, int V,
                                                                               const float* params, const unsigned long long* seeds, const int* step,
                                                                               int step_offset, long long* ids, void* stream) {
  return launch_sample_rows(logits, logits_f32, ld, R, V, params, seeds, step, step_offset, ids, nullptr, 0, stream, true);
}

extern "C" __attribute__((visibility("default"))) int srgpt_sample_rows_warped_scores(const void* logits, int logits_f32, int ld, int R, int V,
                                                                                      const float* params, const unsigned long long* seeds,
                                                                                      const int* step, int step_offset, long long* ids, float* scores,
                                                                                      long long step_stride, void* stream) {
  SRGPT_CHECK_ARG(scores != nullptr);
  return launch_sample_rows(logits, logits_f32, ld, R, V, params, seeds, step, step_offset, ids, scores, step_stride, stream, true);
}
