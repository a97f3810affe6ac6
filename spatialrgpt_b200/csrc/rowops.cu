// Row-wise HBM-bound kernels: LayerNorm (+GELU), DownSample+LayerNorm, RMSNorm, patchify, splice,
// argmax.  All use 16-byte vector accesses with threads mapped along the contiguous (channel) dim.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {

void set_last_error(const char* fmt, ...);

// ---------------------------------------------------------------------------------------------
// LayerNorm: one CTA per row, each thread keeps up to MAXV 16-byte chunks of the row in registers.
// ---------------------------------------------------------------------------------------------
constexpr int LN_THREADS = 128;
constexpr int LN_MAXV = 5;  // cols <= 128 * 5 * 8 = 5120

struct DownsampleGather {  // optional: build the input row from 4 source rows (DownSampleBlock)
  int enabled;
  int side;      // source side (27)
  int half;      // ceil(side/2) (14)
  int C;         // source channels
};

template <bool GATHER>
__global__ void __launch_bounds__(LN_THREADS)
layernorm_kernel(const bf16* __restrict__ x, int ldx, const bf16* __restrict__ weight, const bf16* __restrict__ bias,
                 bf16* __restrict__ y, int ldy, int cols, float eps, int act, DownsampleGather g) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const int nchunk = cols >> 3;
  float v[LN_MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = threadIdx.x + i * LN_THREADS;
    if (c < nchunk) {
      uint4 u;
      if (GATHER) {
        // output token (a, b) of image n gathers x[2b+dy? ...]: see base_projector.py:44-52.
        // out[n, a*half + b, q*C + ch] with q = 2*qa + qb  <-  x[n, (2b + qa)*side + (2a + qb), ch]
        const int per_img = g.half * g.half;
        const int n = row / per_img, t = row % per_img;
        const int a = t / g.half, b = t % g.half;
        const int col = c << 3;
        const int q = col / g.C, ch = col % g.C;
        const int sy = 2 * b + (q >> 1), sx = 2 * a + (q & 1);
        if (sy < g.side && sx < g.side) {
          u = *reinterpret_cast<const uint4*>(x + ((size_t)n * g.side * g.side + (size_t)sy * g.side + sx) * g.C + ch);
        } else {
          u = make_uint4(0, 0, 0, 0);
        }
      } else {
        u = *reinterpret_cast<const uint4*>(x + (size_t)row * ldx + (c << 3));
      }
      unpack8(u, v[i]);
#pragma unroll
      for (int t = 0; t < 8; ++t) sum += v[i][t];
    }
  }
  const float mean = block_sum(sum, red) / (float)cols;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = threadIdx.x + i * LN_THREADS;
    if (c < nchunk) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const float d = v[i][t] - mean;
        sq += d * d;
      }
    }
  }
  const float var = block_sum(sq, red) / (float)cols;
  const float rstd = rsqrtf(var + eps);
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = threadIdx.x + i * LN_THREADS;
    if (c < nchunk) {
      float w[8], b[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(weight + (c << 3)), w);
      unpack8(*reinterpret_cast<const uint4*>(bias + (c << 3)), b);
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        float r = (v[i][t] - mean) * rstd * w[t] + b[t];
        if (act == 1) r = gelu_erf(bf16_round(r));
        o[t] = r;
      }
      *reinterpret_cast<uint4*>(y + (size_t)row * ldy + (c << 3)) = pack8(o);
    }
  }
}

// LayerNorm for short rows (cols <= 1280, e.g. the 1152 channels of SigLIP): one WARP per row, rows strided over a fixed
// grid.  The CTA-per-row kernel above is slow on a 64-image tower's 65536 x 1152 activations (53 calls per request batch): a
// 2.3 KB row per 128-thread CTA leaves too few bytes in flight and pays two block reductions.  Here a lane holds up to 5 16-byte chunks, reductions are warp shuffles, 64 warps per SM stream rows.
constexpr int LNW_WARPS = 8;
__global__ void __launch_bounds__(LNW_WARPS * 32)
layernorm_warp_kernel(const bf16* __restrict__ x, int ldx, const bf16* __restrict__ weight, const bf16* __restrict__ bias,
                      bf16* __restrict__ y, int ldy, int rows, int cols, float eps, int act) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunk = cols >> 3;
  const float inv_cols = 1.f / (float)cols;
  for (int row = blockIdx.x * LNW_WARPS + warp; row < rows; row += gridDim.x * LNW_WARPS) {
    float v[LN_MAXV][8];
    float sum = 0.f;
    const bf16* xr = x + (size_t)row * ldx;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i) {
      const int c = lane + i * 32;
      if (c < nchunk) {
        unpack8(ld_stream16(xr + (c << 3)), v[i]);
#pragma unroll
        for (int t = 0; t < 8; ++t) sum += v[i][t];
      }
    }
    const float mean = warp_sum(sum) * inv_cols;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i) {
      if (lane + i * 32 < nchunk) {
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float d = v[i][t] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) * inv_cols + eps);
    bf16* yr = y + (size_t)row * ldy;
#pragma unroll
    for (int i = 0; i < LN_MAXV; ++i) {
      const int c = lane + i * 32;
      if (c < nchunk) {
        float w[8], b[8], o[8];
        unpack8(*reinterpret_cast<const uint4*>(weight + (c << 3)), w);
        unpack8(*reinterpret_cast<const uint4*>(bias + (c << 3)), b);
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          float r = (v[i][t] - mean) * rstd * w[t] + b[t];
          if (act == 1) r = gelu_erf(bf16_round(r));
          o[t] = r;
        }
        *reinterpret_cast<uint4*>(yr + (c << 3)) = pack8(o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// RMSNorm (Llama): y = weight * bf16(x * rsqrt(mean(x^2) + eps))
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LN_THREADS)
rmsnorm_kernel(const bf16* __restrict__ x, int ldx, const bf16* __restrict__ weight, bf16* __restrict__ y, int ldy,
               int cols, float eps) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const int nchunk = cols >> 3;
  float v[LN_MAXV][8];
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = threadIdx.x + i * LN_THREADS;
    if (c < nchunk) {
      unpack8(*reinterpret_cast<const uint4*>(x + (size_t)row * ldx + (c << 3)), v[i]);
#pragma unroll
      for (int t = 0; t < 8; ++t) sq += v[i][t] * v[i][t];
    }
  }
  const float rstd = rsqrtf(block_sum(sq, red) / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = threadIdx.x + i * LN_THREADS;
    if (c < nchunk) {
      float w[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(weight + (c << 3)), w);
#pragma unroll
      for (int t = 0; t < 8; ++t) o[t] = w[t] * bf16_round(v[i][t] * rstd);
      *reinterpret_cast<uint4*>(y + (size_t)row * ldy + (c << 3)) = pack8(o);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// patchify: images [n,3,R,R] -> A [n*P*P, ldk], col = c*ps*ps + ky*ps + kx (Conv2d weight flatten order)
// ---------------------------------------------------------------------------------------------
template <typename SrcT>
__global__ void patchify_kernel(const SrcT* __restrict__ img, bf16* __restrict__ A, int R, int ps, int ldk) {
  const int P = R / ps;
  const int row = blockIdx.x;  // n*P*P + py*P + px
  const int n = row / (P * P), t = row % (P * P);
  const int py = t / P, px = t % P;
  const int kk = 3 * ps * ps;
  for (int col = threadIdx.x; col < ldk; col += blockDim.x) {
    float val = 0.f;
    if (col < kk) {
      const int c = col / (ps * ps), r = col % (ps * ps);
      const int ky = r / ps, kx = r % ps;
      val = (float)img[(((size_t)n * 3 + c) * R + (py * ps + ky)) * R + (px * ps + kx)];
    }
    A[(size_t)row * ldk + col] = f2e(val);
  }
}

// ---------------------------------------------------------------------------------------------
// CLIP embeddings: out[n, 0] = cls + pos[0]; out[n, 1 + t] = patch[n, t] + pos[1 + t]   (one element-type add, like torch's)
// ---------------------------------------------------------------------------------------------
__global__ void clip_embed_kernel(const bf16* __restrict__ patch, const bf16* __restrict__ cls, const bf16* __restrict__ pos,
                                  bf16* __restrict__ out, int T, int D) {
  const int row = blockIdx.x;  // n * (T + 1) + s
  const int n = row / (T + 1), s = row % (T + 1);
  const uint4* a = reinterpret_cast<const uint4*>(s == 0 ? cls : patch + ((size_t)n * T + (s - 1)) * D);
  const uint4* b = reinterpret_cast<const uint4*>(pos + (size_t)s * D);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)row * D);
  for (int c = threadIdx.x; c < (D >> 3); c += blockDim.x) {
    float fa[8], fb[8];
    unpack8(a[c], fa);
    unpack8(b[c], fb);
#pragma unroll
    for (int t = 0; t < 8; ++t) fa[t] += fb[t];
    dst[c] = pack8(fa);
  }
}

// ---------------------------------------------------------------------------------------------
// splice: out[r,:] = src[src_id[r]][src_row[r],:]
// ---------------------------------------------------------------------------------------------
__global__ void splice_kernel(const bf16* s0, const bf16* s1, const bf16* s2, const bf16* s3, const int* __restrict__ src_id,
                              const int* __restrict__ src_row, bf16* __restrict__ out, int cols) {
  const int r = blockIdx.x;
  const int id = src_id[r];
  const bf16* base = id == 0 ? s0 : (id == 1 ? s1 : (id == 2 ? s2 : s3));
  const uint4* src = reinterpret_cast<const uint4*>(base + (size_t)src_row[r] * cols);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)r * cols);
  for (int c = threadIdx.x; c < (cols >> 3); c += blockDim.x) dst[c] = src[c];
}

// ---------------------------------------------------------------------------------------------
// argmax over fp32 rows, first index on ties
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float argmax_load(const float* p) { return *p; }
__device__ __forceinline__ float argmax_load(const bf16* p) { return e2f(*p); }

template <typename T>
__global__ void __launch_bounds__(256) argmax_kernel(const T* __restrict__ x, int ldx, int cols, long long* __restrict__ out) {
  __shared__ float sv[8];
  __shared__ int si[8];
  const T* row = x + (size_t)blockIdx.x * ldx;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    const float v = argmax_load(row + c);
    if (v > best || (v == best && c < bi)) { best = v; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
    out[blockIdx.x] = bi == 0x7fffffff ? 0 : bi;  // a row of NaNs compares false everywhere: report index 0, never the sentinel
  }
}

// Wide rows (a vocabulary of 128 K per sequence of a batched decode step): one CTA per 4096-column segment, the segments of a row
// meet in a 64-bit atomicMax on (order-preserving value bits << 32 | ~index) - max value first, lowest index on ties, and
// associative, so the result does not depend on the arrival order.  out[] holds the packed key until argmax_unpack_kernel.
// (ARGMAX_SEG and float_order_bits live in common.cuh: logits_process.cu builds the same key)
template <typename T>
__global__ void __launch_bounds__(256) argmax_wide_kernel(const T* __restrict__ x, int ldx, int cols, unsigned long long* __restrict__ keys) {
  __shared__ unsigned long long sk[8];
  const T* row = x + (size_t)blockIdx.y * ldx;
  const int c0 = blockIdx.x * ARGMAX_SEG, c1 = min(cols, c0 + ARGMAX_SEG);
  unsigned long long best = 0ull;
  for (int c = c0 + threadIdx.x; c < c1; c += blockDim.x) {
    const float v = argmax_load(row + c);
    if (v == v) {  // NaN never wins (an all-NaN row reports index 0 through the zero key)
      const unsigned long long k = ((unsigned long long)float_order_bits(v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)c);
      best = k > best ? k : best;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ok = __shfl_xor_sync(0xffffffffu, best, o);
    best = ok > best ? ok : best;
  }
  if ((threadIdx.x & 31) == 0) sk[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) best = sk[w] > best ? sk[w] : best;
    atomicMax(keys + blockIdx.y, best);
  }
}
__global__ void argmax_unpack_kernel(long long* __restrict__ out, int rows) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) {
    const unsigned long long k = reinterpret_cast<unsigned long long*>(out)[r];
    out[r] = k == 0ull ? 0ll : (long long)(0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull));
  }
}

void argmax_unpack(long long* keys, int rows, cudaStream_t stream) {
  argmax_unpack_kernel<<<ceil_div(rows, 256), 256, 0, stream>>>(keys, rows);
}

// ---------------------------------------------------------------------------------------------
// beam search candidates: per beam row, log_softmax of the (element-type rounded) logits + the beam's running score, and the
// n_cand best (score, token) of the row in (score desc, token asc) order.  One 1024-thread CTA per row; the row (<= 256 KB) is
// re-read from L2 once per candidate: pass j finds the successor of candidate j-1 in that order, so no selection state is kept.
// ---------------------------------------------------------------------------------------------
constexpr int BEAM_THREADS = 1024;
__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* sk) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ov = __shfl_xor_sync(0xffffffffu, v, o);
    v = ov > v ? ov : v;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sk[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long t = sk[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long ov = __shfl_xor_sync(0xffffffffu, t, o);
    t = ov > t ? ov : t;
  }
  return t;
}
// SCORED (diverse beam search, beam.cu group_select_kernel): the candidates are ranked by their fp32 score ((v - m) - lse) + bs, token
// asc on ties, rather than by the logit, so a row's list is exactly its top n_cand in the order the group merge uses even where the
// rounding of + bs ties different logits; and the row's (m, lse) go to stats[row], so the merge can score any other token of the row.
template <bool SCORED>
__device__ __forceinline__ void beam_candidates_row(const bf16* __restrict__ logits, int ldx, int V, const float* __restrict__ beam_scores, int n_cand,
                                                    float* __restrict__ cand_scores, int* __restrict__ cand_tokens, float* __restrict__ logprobs,
                                                    long long ldo, float2* __restrict__ stats) {
  __shared__ unsigned long long sk[32];
  __shared__ float sred[32];
  const bf16* row = logits + (size_t)blockIdx.x * ldx;
  const int tid = threadIdx.x;
  // log-sum-exp in fp32 over the rounded logits (torch: log_softmax(logits.float(), -1))
  float m = -INFINITY;
  for (int c = tid; c < V; c += BEAM_THREADS) {
    const float v = e2f(row[c]);
    if (v == v) m = fmaxf(m, v);
  }
  m = warp_max(m);
  if ((tid & 31) == 0) sred[tid >> 5] = m;
  __syncthreads();
  m = warp_max(sred[tid & 31]);
  float z = 0.f;
  for (int c = tid; c < V; c += BEAM_THREADS) {
    const float v = e2f(row[c]);
    if (v == v) z += expf(v - m);
  }
  z = block_sum(z, sred);
  const float lse = logf(z);
  if (logprobs != nullptr) {  // the whole log_softmax row (HF's output_scores of a beam step), before the beam score is added
    float* orow = logprobs + (size_t)blockIdx.x * ldo;
    for (int c = tid; c < V; c += BEAM_THREADS) orow[c] = (e2f(row[c]) - m) - lse;
  }
  const float bs = beam_scores[blockIdx.x];
  if (SCORED && tid == 0) stats[blockIdx.x] = make_float2(m, lse);
  // key = (order-preserving bits of the logit (SCORED: of the score), ~token): the maximum key below the previous one is the next candidate
  unsigned long long prev = ~0ull;
  for (int j = 0; j < n_cand; ++j) {
    unsigned long long best = 0ull;
    for (int c = tid; c < V; c += BEAM_THREADS) {
      const float v = e2f(row[c]);
      if (v == v) {
        const unsigned long long k = ((unsigned long long)float_order_bits(SCORED ? ((v - m) - lse) + bs : v) << 32) |
                                     (unsigned long long)(0xFFFFFFFFu - (unsigned int)c);
        if (k < prev && k > best) best = k;
      }
    }
    best = block_max_u64(best, sk);
    if (tid == 0) {
      if (best == 0ull) {  // fewer than n_cand finite logits
        cand_scores[(size_t)blockIdx.x * n_cand + j] = -INFINITY;
        cand_tokens[(size_t)blockIdx.x * n_cand + j] = -1;
      } else {
        const int tok = (int)(0xFFFFFFFFu - (unsigned int)(best & 0xFFFFFFFFull));
        const float v = e2f(row[tok]);
        cand_scores[(size_t)blockIdx.x * n_cand + j] = ((v - m) - lse) + bs;
        cand_tokens[(size_t)blockIdx.x * n_cand + j] = tok;
      }
    }
    prev = best == 0ull ? 0ull : best;
  }
}
__global__ void __launch_bounds__(BEAM_THREADS)
beam_candidates_kernel(const bf16* __restrict__ logits, int ldx, int V, const float* __restrict__ beam_scores, int n_cand, float* __restrict__ cand_scores,
                       int* __restrict__ cand_tokens, float* __restrict__ logprobs, long long ldo) {
  beam_candidates_row<false>(logits, ldx, V, beam_scores, n_cand, cand_scores, cand_tokens, logprobs, ldo, nullptr);
}
__global__ void __launch_bounds__(BEAM_THREADS)
beam_candidates_scored_kernel(const bf16* __restrict__ logits, int ldx, int V, const float* __restrict__ beam_scores, int n_cand,
                              float* __restrict__ cand_scores, int* __restrict__ cand_tokens, float2* __restrict__ stats) {
  beam_candidates_row<true>(logits, ldx, V, beam_scores, n_cand, cand_scores, cand_tokens, nullptr, 0, stats);
}

// ---------------------------------------------------------------------------------------------
// batched decode bookkeeping: one CTA per sequence b: out_ids[*step * B + b] = ids[b]; h[b,:] = embed[ids[b],:]; ++pos[b];
// the last CTA to finish (atomic ticket) advances *step, so one launch serves the whole batch inside a CUDA graph
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
decode_batch_advance_kernel(const long long* __restrict__ ids, const bf16* __restrict__ embed, bf16* __restrict__ h, int H, long long* __restrict__ out_ids,
                            int* step, int* pos, int B, unsigned int* ticket) {
  const int b = blockIdx.x;
  const long long tok = ids[b];
  const uint4* src = reinterpret_cast<const uint4*>(embed + (size_t)tok * H);
  uint4* dst = reinterpret_cast<uint4*>(h + (size_t)b * H);
  for (int c = threadIdx.x; c < (H >> 3); c += blockDim.x) dst[c] = src[c];
  if (threadIdx.x == 0) {
    out_ids[(size_t)(*step) * B + b] = tok;
    pos[b] += 1;
    __threadfence();
    if (atomicAdd(ticket, 1u) == (unsigned int)(B - 1)) {  // every CTA has read *step
      *ticket = 0u;
      *step += 1;
    }
  }
}

}  // namespace srgpt

using namespace srgpt;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" __attribute__((visibility("default"))) int srgpt_layernorm_bf16(const void* x, int ldx, const void* weight, const void* bias, void* y, int ldy, int rows,
                                    int cols, float eps, int act, void* stream) {
  SRGPT_CHECK_ARG(x && weight && bias && y && rows > 0 && cols > 0);
  SRGPT_CHECK_ARG((cols % 8) == 0 && cols <= LN_THREADS * LN_MAXV * 8);
  SRGPT_CHECK_ARG((ldx % 8) == 0 && (ldy % 8) == 0 && ldx >= cols && ldy >= cols);
  SRGPT_CHECK_ARG(aligned16(x) && aligned16(weight) && aligned16(bias) && aligned16(y));
  SRGPT_CHECK_ARG(act == 0 || act == 1);
  if (cols <= 32 * LN_MAXV * 8 && rows >= 4 * LNW_WARPS) {  // short rows: one warp per row
    const int ctas = ceil_div(rows, LNW_WARPS);
    const int grid = ctas < sm_count() * 8 ? ctas : sm_count() * 8;
    layernorm_warp_kernel<<<grid, LNW_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(weight), reinterpret_cast<const bf16*>(bias),
        reinterpret_cast<bf16*>(y), ldy, rows, cols, eps, act);
    SRGPT_CHECK_LAUNCH();
    return SRGPT_OK;
  }
  DownsampleGather g{0, 0, 0, 0};
  layernorm_kernel<false><<<rows, LN_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(weight), reinterpret_cast<const bf16*>(bias),
      reinterpret_cast<bf16*>(y), ldy, cols, eps, act, g);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_downsample_layernorm_bf16(const void* x, const void* weight, const void* bias, void* y, int n_img,
                                               int side, int C, float eps, void* stream) {
  SRGPT_CHECK_ARG(x && weight && bias && y && n_img > 0 && side > 0 && C > 0);
  SRGPT_CHECK_ARG((C % 8) == 0 && 4 * C <= LN_THREADS * LN_MAXV * 8);
  SRGPT_CHECK_ARG(aligned16(x) && aligned16(weight) && aligned16(bias) && aligned16(y));
  const int half = (side + 1) / 2;
  DownsampleGather g{1, side, half, C};
  const int rows = n_img * half * half;
  layernorm_kernel<true><<<rows, LN_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(x), 0, reinterpret_cast<const bf16*>(weight), reinterpret_cast<const bf16*>(bias),
      reinterpret_cast<bf16*>(y), 4 * C, 4 * C, eps, 0, g);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_rmsnorm_bf16(const void* x, int ldx, const void* weight, void* y, int ldy, int rows, int cols, float eps,
                                  void* stream) {
  SRGPT_CHECK_ARG(x && weight && y && rows > 0 && cols > 0);
  SRGPT_CHECK_ARG((cols % 8) == 0 && cols <= LN_THREADS * LN_MAXV * 8);
  SRGPT_CHECK_ARG((ldx % 8) == 0 && (ldy % 8) == 0 && ldx >= cols && ldy >= cols);
  SRGPT_CHECK_ARG(aligned16(x) && aligned16(weight) && aligned16(y));
  rmsnorm_kernel<<<rows, LN_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<const bf16*>(weight), reinterpret_cast<bf16*>(y), ldy, cols, eps);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_patchify_bf16(const void* images, int src_is_bf16, void* A, int n, int R, int ps, int ldk, void* stream) {
  SRGPT_CHECK_ARG(images && A && n > 0 && R > 0 && ps > 0 && (R % ps) == 0);
  SRGPT_CHECK_ARG(ldk >= 3 * ps * ps && (ldk % 8) == 0);
  const int P = R / ps;
  const int rows = n * P * P;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (src_is_bf16)
    patchify_kernel<bf16><<<rows, 128, 0, st>>>(reinterpret_cast<const bf16*>(images), reinterpret_cast<bf16*>(A), R, ps, ldk);
  else
    patchify_kernel<float><<<rows, 128, 0, st>>>(reinterpret_cast<const float*>(images), reinterpret_cast<bf16*>(A), R, ps, ldk);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_clip_embed_bf16(const void* patch_embeds, const void* class_embedding, const void* position_embedding,
                                                                               void* out, int n_img, int T, int D, void* stream) {
  SRGPT_CHECK_ARG(patch_embeds && class_embedding && position_embedding && out && n_img > 0 && T > 0 && D > 0 && (D % 8) == 0);
  SRGPT_CHECK_ARG(((reinterpret_cast<uintptr_t>(patch_embeds) | reinterpret_cast<uintptr_t>(class_embedding) | reinterpret_cast<uintptr_t>(position_embedding) |
                    reinterpret_cast<uintptr_t>(out)) & 15) == 0);
  clip_embed_kernel<<<n_img * (T + 1), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(patch_embeds), reinterpret_cast<const bf16*>(class_embedding), reinterpret_cast<const bf16*>(position_embedding),
      reinterpret_cast<bf16*>(out), T, D);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_splice_rows_bf16(const void* src0, const void* src1, const void* src2, const void* src3,
                                      const int* src_id, const int* src_row, void* out, int rows, int cols, void* stream) {
  SRGPT_CHECK_ARG(src0 && src_id && src_row && out && rows > 0 && cols > 0 && (cols % 8) == 0);
  SRGPT_CHECK_ARG(aligned16(src0) && aligned16(src1) && aligned16(src2) && aligned16(src3) && aligned16(out));
  splice_kernel<<<rows, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(src0), reinterpret_cast<const bf16*>(src1), reinterpret_cast<const bf16*>(src2),
      reinterpret_cast<const bf16*>(src3), src_id, src_row, reinterpret_cast<bf16*>(out), cols);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_argmax_f32(const float* x, int rows, int cols, long long* out, void* stream) {
  SRGPT_CHECK_ARG(x && out && rows > 0 && cols > 0);
  argmax_kernel<float><<<rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, cols, cols, out);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_argmax_bf16(const void* x, int ldx, int rows, int cols, long long* out, void* stream) {
  SRGPT_CHECK_ARG(x && out && rows > 0 && cols > 0 && ldx >= cols);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cols > 4 * ARGMAX_SEG && rows <= 65535) {
    // wide rows: one CTA per 4096-column segment instead of one CTA per row (32 rows of 128 K logits would otherwise run on 32 CTAs)
    SRGPT_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)rows * sizeof(long long), st));
    argmax_wide_kernel<bf16><<<dim3(ceil_div(cols, ARGMAX_SEG), rows), 256, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, cols,
                                                                                   reinterpret_cast<unsigned long long*>(out));
    SRGPT_CHECK_LAUNCH();
    argmax_unpack_kernel<<<ceil_div(rows, 256), 256, 0, st>>>(out, rows);
    SRGPT_CHECK_LAUNCH();
    return SRGPT_OK;
  }
  argmax_kernel<bf16><<<rows, 256, 0, st>>>(reinterpret_cast<const bf16*>(x), ldx, cols, out);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// Beam-search candidates (HF GenerationMixin.beam_search, transformers 4.37.2 generation/utils.py: log_softmax of the next-token logits +
// beam_scores, then torch.topk over the flattened [num_beams x vocab] table; call site llava_llama.py:212 with num_beams > 1): per beam row
// the n_cand best (log_softmax(logits)[token] + beam_scores[row], token), ties towards the lower token id.  The host merges the
// num_beams x n_cand pairs (the global top-2k is a subset of the per-row top-2k).
extern "C" __attribute__((visibility("default"))) int srgpt_beam_candidates_bf16(const void* logits, int ldx, int n_beams, int V, const float* beam_scores, int n_cand,
                                                                                  float* cand_scores, int* cand_tokens, void* stream) {
  return srgpt_beam_candidates_scores_bf16(logits, ldx, n_beams, V, beam_scores, n_cand, cand_scores, cand_tokens, nullptr, 0, stream);
}

// The same candidates, and (when logprobs is given) every row's whole log_softmax -> logprobs [n_beams, ldo] fp32.
extern "C" __attribute__((visibility("default"))) int srgpt_beam_candidates_scores_bf16(const void* logits, int ldx, int n_beams, int V,
                                                                                         const float* beam_scores, int n_cand, float* cand_scores,
                                                                                         int* cand_tokens, float* logprobs, long long ldo, void* stream) {
  SRGPT_CHECK_ARG(logits && beam_scores && cand_scores && cand_tokens && n_beams > 0 && V > 0 && ldx >= V && n_cand > 0 && n_cand <= V);
  SRGPT_CHECK_ARG(logprobs == nullptr || ldo >= V);
  beam_candidates_kernel<<<n_beams, BEAM_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const bf16*>(logits), ldx, V, beam_scores, n_cand,
                                                                                             cand_scores, cand_tokens, logprobs, ldo);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// Diverse beam search's candidates (llama_decoder.generate_beam_batch with num_beam_groups > 1): per row the n_cand best (score, token) in
// (score desc, token asc) order of the score itself, and the row's (max, log-sum-exp) -> stats [n_beams] float2.
extern "C" __attribute__((visibility("default"))) int srgpt_beam_candidates_scored_bf16(const void* logits, int ldx, int n_beams, int V,
                                                                                         const float* beam_scores, int n_cand, float* cand_scores,
                                                                                         int* cand_tokens, float* stats, void* stream) {
  SRGPT_CHECK_ARG(logits && beam_scores && cand_scores && cand_tokens && stats && n_beams > 0 && V > 0 && ldx >= V && n_cand > 0 && n_cand <= V);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(stats) & 7) == 0);
  beam_candidates_scored_kernel<<<n_beams, BEAM_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(logits), ldx, V, beam_scores, n_cand, cand_scores, cand_tokens, reinterpret_cast<float2*>(stats));
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// A decode step's score rows (HF's output_scores of a greedy step): row r of rows [R, ld] (fp32, or the element type widened exactly, as
// .float() widens it) -> scores + (*step + step_offset) * step_stride + r * row_stride.  The index is read at run time, so one captured
// decode graph writes every step's rows.  grid = (column blocks, R).
__device__ __forceinline__ float widen(float x) { return x; }
__device__ __forceinline__ float widen(bf16 x) { return e2f(x); }
template <typename T>
__global__ void __launch_bounds__(256)
step_scores_kernel(const T* __restrict__ rows, long long ld, int V, const int* __restrict__ step, int step_offset, float* __restrict__ scores,
                   long long step_stride, long long row_stride) {
  const T* src = rows + (size_t)blockIdx.y * ld;
  float* dst = scores + (long long)(*step + step_offset) * step_stride + (long long)blockIdx.y * row_stride;
  for (int c = blockIdx.x * 256 + threadIdx.x; c < V; c += gridDim.x * 256) dst[c] = widen(src[c]);
}

extern "C" __attribute__((visibility("default"))) int srgpt_step_scores(const void* rows, int rows_f32, long long ld, int R, int V, const int* step,
                                                                        int step_offset, float* scores, long long step_stride, long long row_stride,
                                                                        void* stream) {
  SRGPT_CHECK_ARG(rows && step && scores && R > 0 && R <= 65535 && V > 0 && ld >= V && row_stride >= V && step_stride >= 0);
  SRGPT_CHECK_ARG(rows_f32 == 0 || rows_f32 == 1);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(ceil_div(V, 256 * 16), R);
  if (rows_f32)
    step_scores_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(rows), ld, V, step, step_offset, scores, step_stride, row_stride);
  else
    step_scores_kernel<bf16><<<grid, 256, 0, st>>>(reinterpret_cast<const bf16*>(rows), ld, V, step, step_offset, scores, step_stride, row_stride);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// Batched greedy decode bookkeeping after the row-wise arg max of a step: ids [B] -> out_ids[*step, :], next embedding rows, ++pos[b],
// ++*step.  `ticket` = one zeroed device uint (returned to zero by the kernel).
extern "C" __attribute__((visibility("default"))) int srgpt_decode_batch_advance(const long long* ids, const void* embed_table, void* h, int H, long long* out_ids,
                                                                                 int* step, int* pos, int B, void* ticket, void* stream) {
  SRGPT_CHECK_ARG(ids && embed_table && h && out_ids && step && pos && ticket && B > 0 && H > 0 && (H % 8) == 0);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(embed_table) & 15) == 0 && (reinterpret_cast<uintptr_t>(h) & 15) == 0);
  decode_batch_advance_kernel<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(ids, reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(h), H,
                                                                                     out_ids, step, pos, B, reinterpret_cast<unsigned int*>(ticket));
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// flags[r] = 1 when row r of a and row r of b ([rows, row_bytes], rows contiguous) hold the same bytes, else 0.  The prompt-prefix
// cache compares a request's images / depths / masks with the ones it kept from the previous request on the device.
__global__ void rows_equal_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, long long row_bytes, int* __restrict__ flags) {
  const uint8_t* ra = a + (size_t)blockIdx.x * row_bytes;
  const uint8_t* rb = b + (size_t)blockIdx.x * row_bytes;
  int same = 1;
  const bool vec = ((reinterpret_cast<uintptr_t>(ra) | reinterpret_cast<uintptr_t>(rb)) & 15) == 0;
  long long i = 0;
  if (vec) {
    const long long n16 = row_bytes / 16;
    for (long long k = threadIdx.x; k < n16; k += blockDim.x) {
      const uint4 x = reinterpret_cast<const uint4*>(ra)[k], y = reinterpret_cast<const uint4*>(rb)[k];
      same &= (x.x == y.x) & (x.y == y.y) & (x.z == y.z) & (x.w == y.w);
    }
    i = n16 * 16;
  }
  for (long long k = i + threadIdx.x; k < row_bytes; k += blockDim.x) same &= ra[k] == rb[k];
  same = __syncthreads_and(same);
  if (threadIdx.x == 0) flags[blockIdx.x] = same;
}

extern "C" __attribute__((visibility("default"))) int srgpt_rows_equal(const void* a, const void* b, int rows, long long row_bytes, int* flags, void* stream) {
  SRGPT_CHECK_ARG(a && b && flags && rows > 0 && row_bytes > 0);
  rows_equal_kernel<<<rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const uint8_t*>(a), reinterpret_cast<const uint8_t*>(b),
                                                                              row_bytes, flags);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
