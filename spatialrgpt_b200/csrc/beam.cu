// Device side of beam search over a batch of prompts (llama_decoder.generate_beam_batch; DESIGN.md §7): the per-prompt merge of the
// beam rows' candidates, and the KV page copies that replicate each prompt into its beams and make a beam's generated rows follow
// its parent; the group-by-group choice of diverse beam search.  Also the one-position KV broadcast of contrastive search (llama_decoder.generate_contrastive).
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {

constexpr int SELECT_THREADS = 256;
constexpr int SELECT_MAX = 4096;  // k * n_cand candidates of one prompt, staged in shared memory

// (score desc, beam asc, token asc): the flat-index order of HF's topk over a prompt's [num_beams x vocab] table on ties
__device__ __forceinline__ bool select_before(float sa, int ba, int ta, float sb, int bb, int tb) {
  return sa > sb || (sa == sb && (ba < bb || (ba == bb && ta < tb)));
}

// One CTA per prompt g: rows g*k .. g*k+k-1 of the candidates table.  Every valid candidate's rank is the number of valid candidates
// before it in the merge order (the order is strict: a row holds each token once), so each lands in its slot with no sort state.
__global__ void __launch_bounds__(SELECT_THREADS)
beam_select_kernel(const float* __restrict__ cand_scores, const int* __restrict__ cand_tokens, int k, int n_cand, float* __restrict__ out_scores,
                   int* __restrict__ out_beams, int* __restrict__ out_tokens) {
  __shared__ float ss[SELECT_MAX];
  __shared__ int st[SELECT_MAX];
  __shared__ int n_valid;
  const int N = k * n_cand;
  const size_t in0 = (size_t)blockIdx.x * N, out0 = (size_t)blockIdx.x * n_cand;
  if (threadIdx.x == 0) n_valid = 0;
  int valid = 0;
  for (int i = threadIdx.x; i < N; i += SELECT_THREADS) {
    ss[i] = cand_scores[in0 + i];
    st[i] = cand_tokens[in0 + i];
    valid += st[i] >= 0;
  }
  __syncthreads();
  atomicAdd(&n_valid, valid);
  for (int i = threadIdx.x; i < N; i += SELECT_THREADS) {
    const int t = st[i];
    if (t < 0) continue;
    const float s = ss[i];
    const int b = i / n_cand;
    int rank = 0;
    for (int j = 0; j < N && rank < n_cand; ++j)
      rank += st[j] >= 0 && select_before(ss[j], j / n_cand, st[j], s, b, t);
    if (rank < n_cand) {
      out_scores[out0 + rank] = s;
      out_beams[out0 + rank] = b;
      out_tokens[out0 + rank] = t;
    }
  }
  __syncthreads();
  for (int r = n_valid + threadIdx.x; r < n_cand; r += SELECT_THREADS) {  // fewer valid candidates than slots
    out_scores[out0 + r] = -INFINITY;
    out_beams[out0 + r] = -1;
    out_tokens[out0 + r] = -1;
  }
}

// Diverse beam search (HF group_beam_search + HammingDiversityLogitsProcessor + BeamSearchScorer.process, transformers 4.37.2; DESIGN.md
// §4): one CTA per prompt walks its G groups of gs = k / G beams in order.  Group g's pool holds, for each of its rows, the row's L
// candidates of beam_candidates_scored_kernel and every token an earlier group chose in this step; each is scored from its own logit
// as fl(fl(logp - fl(lambda * c)) + s), c = how often the earlier groups chose it, logp = fl(fl(v - m) - lse).  A row's list is its top L
// by unpenalised score and at most k - gs of them are penalised, so with L >= n_cand + k - gs every token outside the pool has n_cand
// pool entries of its own row before it: the pool's top n_cand is the group's exact top n_cand of its gs x V table.
// Outputs: the ranked candidates of each (prompt, group), and the gs next (parent, token) pairs of HF's process rule (EOS candidates
// become no beam); a done group emits pad_id from its first beam.  The tokens chosen go to shared memory for the later groups.
constexpr int GROUP_POOL_MAX = 4096;  // gs * (L + k - gs) candidates of one group, as 64-bit keys
constexpr int GROUP_CAND_MAX = 512;
constexpr int GROUP_K_MAX = 64;        // gs - 1 fits the key's 6 beam bits
constexpr unsigned int GROUP_TOKEN_BITS = 26;
constexpr unsigned int GROUP_TOKEN_MASK = (1u << GROUP_TOKEN_BITS) - 1u;

__device__ __forceinline__ float float_from_order_bits(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

__global__ void __launch_bounds__(SELECT_THREADS)
group_select_kernel(const bf16* __restrict__ logits, int ldx, int V, const float2* __restrict__ stats, const float* __restrict__ beam_scores,
                    const int* __restrict__ cand_tokens, int L, int k, int G, int n_cand, const int* __restrict__ eos, int n_eos, int pad_id,
                    float lambda, const int* __restrict__ done, float* __restrict__ out_scores, int* __restrict__ out_beams,
                    int* __restrict__ out_tokens, int* __restrict__ next_beams, int* __restrict__ next_tokens) {
  __shared__ unsigned long long pool[GROUP_POOL_MAX];
  __shared__ unsigned long long top[GROUP_CAND_MAX];
  __shared__ int chosen[GROUP_K_MAX];
  __shared__ int n_valid;
  const int b = blockIdx.x, gs = k / G;
  for (int g = 0; g < G; ++g) {
    const int row0 = b * k + g * gs, n_prev = g * gs, per_row = L + n_prev, N = gs * per_row;
    const size_t o = ((size_t)b * G + g) * n_cand;
    if (done[b * G + g]) {  // BeamSearchScorer.process: pad_token_id for every beam, index 0 of the group
      for (int r = threadIdx.x; r < n_cand; r += SELECT_THREADS) {
        out_scores[o + r] = -INFINITY;
        out_beams[o + r] = -1;
        out_tokens[o + r] = -1;
      }
      for (int i = threadIdx.x; i < gs; i += SELECT_THREADS) {
        next_beams[row0 + i] = g * gs;
        next_tokens[row0 + i] = pad_id;
        chosen[n_prev + i] = pad_id;
      }
      __syncthreads();
      continue;
    }
    if (threadIdx.x == 0) n_valid = 0;
    __syncthreads();
    int valid = 0;
    for (int e = threadIdx.x; e < N; e += SELECT_THREADS) {
      const int i = e / per_row, j = e - i * per_row, r = row0 + i;
      const int* list = cand_tokens + (size_t)r * L;
      int t = -1;
      if (j < L) {
        t = list[j];
      } else {  // an earlier group's choice: once per row, and only when the row's list does not hold it
        t = chosen[j - L];
        for (int q = 0; q < j - L && t >= 0; ++q) t = chosen[q] == t ? -1 : t;
        for (int q = 0; q < L && t >= 0; ++q) t = list[q] == t ? -1 : t;
      }
      unsigned long long key = 0ull;
      if (t >= 0 && t < V) {
        const float v = e2f(logits[(size_t)r * ldx + t]);
        if (v == v) {
          int c = 0;
          for (int q = 0; q < n_prev; ++q) c += chosen[q] == t;
          const float2 ml = stats[r];
          float s = __fsub_rn(__fsub_rn(v, ml.x), ml.y);
          if (c > 0) s = __fsub_rn(s, __fmul_rn(lambda, (float)c));
          s = __fadd_rn(s, beam_scores[r]);
          // (score desc, beam asc, token asc) as one descending key; (beam, token) is unique in the pool
          key = ((unsigned long long)float_order_bits(s) << 32) | ((unsigned long long)(gs - 1 - i) << GROUP_TOKEN_BITS) |
                (unsigned long long)(GROUP_TOKEN_MASK - (unsigned int)t);
          ++valid;
        }
      }
      pool[e] = key;
    }
    atomicAdd(&n_valid, valid);
    __syncthreads();
    for (int e = threadIdx.x; e < N; e += SELECT_THREADS) {
      const unsigned long long key = pool[e];
      if (key == 0ull) continue;
      int rank = 0;
      for (int q = 0; q < N && rank < n_cand; ++q) rank += pool[q] > key;
      if (rank < n_cand) top[rank] = key;
    }
    __syncthreads();
    const int n_top = min(n_valid, n_cand);
    for (int r = threadIdx.x; r < n_cand; r += SELECT_THREADS) {
      const unsigned long long key = top[r];
      const bool ok = r < n_top;
      out_scores[o + r] = ok ? float_from_order_bits((unsigned int)(key >> 32)) : -INFINITY;
      out_beams[o + r] = ok ? gs - 1 - (int)((key >> GROUP_TOKEN_BITS) & 63u) : -1;
      out_tokens[o + r] = ok ? (int)(GROUP_TOKEN_MASK - (unsigned int)(key & GROUP_TOKEN_MASK)) : -1;
    }
    if (threadIdx.x == 0) {  // process: an EOS candidate closes a hypothesis (rank < gs) or is skipped; the others fill the beams in rank order
      int nb = 0;
      for (int r = 0; r < n_top && nb < gs; ++r) {
        const int t = (int)(GROUP_TOKEN_MASK - (unsigned int)(top[r] & GROUP_TOKEN_MASK));
        bool is_eos = false;
        for (int q = 0; q < n_eos; ++q) is_eos |= eos[q] == t;
        if (is_eos) continue;
        next_beams[row0 + nb] = g * gs + gs - 1 - (int)((top[r] >> GROUP_TOKEN_BITS) & 63u);
        next_tokens[row0 + nb] = t;
        chosen[n_prev + nb] = t;
        ++nb;
      }
      for (; nb < gs; ++nb) {  // out of non-EOS candidates: HF raises; the host does too
        next_beams[row0 + nb] = -1;
        next_tokens[row0 + nb] = -1;
        chosen[n_prev + nb] = -1;
      }
    }
    __syncthreads();
  }
}

// KV page copies.  blockIdx.y = pair, blockIdx.x = layer * 2 + (0: K, 1: V); each unit is `rows` contiguous rows of one page half.
// pass 0: pairs [0, n_staged) are copied into their workspace slot, the others straight to their destination page;
// pass 1: the staged pairs go from the workspace to their destination.  A pair outside the cache or the page is skipped.
constexpr int COPY_THREADS = 256;
__global__ void __launch_bounds__(COPY_THREADS)
kv_copy_kernel(uint8_t* __restrict__ pages, int n_pages, int page_rows, int row_bytes, const int4* __restrict__ pairs, int n_staged,
               uint8_t* __restrict__ ws, int pass) {
  const int p = blockIdx.y;
  const int4 pr = pairs[p];  // (src page, dst page, first row, rows)
  if (pr.x < 0 || pr.x >= n_pages || pr.y < 0 || pr.y >= n_pages || pr.z < 0 || pr.w < 0 || pr.z + pr.w > page_rows) return;
  const int layer = blockIdx.x >> 1, half = blockIdx.x & 1;
  const size_t half_bytes = (size_t)page_rows * row_bytes;
  const size_t layer_bytes = (size_t)n_pages * 2 * half_bytes;
  const size_t in_page = (size_t)half * half_bytes + (size_t)pr.z * row_bytes;
  const size_t slot = ((size_t)p * gridDim.x + blockIdx.x) * half_bytes + (size_t)pr.z * row_bytes;  // this unit's rows in the workspace
  const uint8_t* src = pass == 0 ? pages + layer * layer_bytes + (size_t)pr.x * 2 * half_bytes + in_page : ws + slot;
  uint8_t* dst = pass == 0 && p < n_staged ? ws + slot : pages + layer * layer_bytes + (size_t)pr.y * 2 * half_bytes + in_page;
  const int n16 = pr.w * row_bytes / 16;
  for (int c = threadIdx.x; c < n16; c += COPY_THREADS) reinterpret_cast<uint4*>(dst)[c] = reinterpret_cast<const uint4*>(src)[c];
}

// Contrastive search keeps the k rows of a prompt identical: after the choice, row g * k + sel[g] holds the only K / V of the position
// just written that the prompt keeps.  blockIdx.x = layer * 2 + (0: K, 1: V), blockIdx.y = prompt g; each thread reads one 16-byte
// piece of the chosen row once and writes it to the k - 1 siblings.  The position is pos[g * k + sel[g]] + pos_offset; a page id outside
// the cache, a position outside the page table or a selection outside [0, k) leaves the prompt untouched.
__global__ void __launch_bounds__(COPY_THREADS)
kv_broadcast_kernel(uint8_t* __restrict__ pages, int n_pages, int page_rows, int row_bytes, const int* __restrict__ page_tables, int pt_stride,
                    const int* __restrict__ pos, int pos_offset, const int* __restrict__ sel, int k) {
  const int g = blockIdx.y, s = sel[g];
  if (s < 0 || s >= k) return;
  const int src_row = g * k + s;
  const int p = pos[src_row] + pos_offset;
  if (p < 0 || p / page_rows >= pt_stride) return;
  const int j = p / page_rows;
  const int src_page = page_tables[(size_t)src_row * pt_stride + j];
  if (src_page < 0 || src_page >= n_pages) return;
  const int layer = blockIdx.x >> 1, half = blockIdx.x & 1;
  const size_t half_bytes = (size_t)page_rows * row_bytes;
  const size_t in_page = (size_t)half * half_bytes + (size_t)(p - j * page_rows) * row_bytes;
  uint8_t* base = pages + (size_t)layer * n_pages * 2 * half_bytes;
  const uint4* src = reinterpret_cast<const uint4*>(base + (size_t)src_page * 2 * half_bytes + in_page);
  const int n16 = row_bytes / 16;
  for (int c = threadIdx.x; c < n16; c += COPY_THREADS) {
    const uint4 v = src[c];
    for (int i = 0; i < k; ++i) {
      const int dst_page = page_tables[(size_t)(g * k + i) * pt_stride + j];
      if (i == s || dst_page < 0 || dst_page >= n_pages) continue;
      reinterpret_cast<uint4*>(base + (size_t)dst_page * 2 * half_bytes + in_page)[c] = v;
    }
  }
}

}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_beam_select(const float* cand_scores, const int* cand_tokens, int n_groups, int k,
                                                                        int n_cand, float* out_scores, int* out_beams, int* out_tokens, void* stream) {
  SRGPT_CHECK_ARG(cand_scores && cand_tokens && out_scores && out_beams && out_tokens && n_groups > 0 && k > 0 && n_cand > 0);
  SRGPT_CHECK_ARG((long long)k * n_cand <= SELECT_MAX);
  beam_select_kernel<<<n_groups, SELECT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(cand_scores, cand_tokens, k, n_cand, out_scores,
                                                                                              out_beams, out_tokens);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_beam_group_select(const void* logits, int ldx, int V, const float* stats,
                                                                              const float* beam_scores, const int* cand_tokens, int L,
                                                                              int n_prompts, int k, int n_groups, int n_cand, const int* eos,
                                                                              int n_eos, int pad_id, float diversity_penalty, const int* done,
                                                                              float* out_scores, int* out_beams, int* out_tokens,
                                                                              int* next_beams, int* next_tokens, void* stream) {
  SRGPT_CHECK_ARG(logits && stats && beam_scores && cand_tokens && done && out_scores && out_beams && out_tokens && next_beams && next_tokens);
  SRGPT_CHECK_ARG(V > 0 && (unsigned int)V <= GROUP_TOKEN_MASK + 1u && ldx >= V && n_prompts > 0 && n_prompts <= 65535);
  SRGPT_CHECK_ARG(n_groups >= 1 && k >= n_groups && k <= GROUP_K_MAX && k % n_groups == 0 && n_cand > 0 && n_cand <= GROUP_CAND_MAX);
  SRGPT_CHECK_ARG(L > 0 && L <= V && (long long)(k / n_groups) * (L + k - k / n_groups) <= GROUP_POOL_MAX);
  SRGPT_CHECK_ARG(n_eos >= 0 && (n_eos == 0 || eos) && pad_id >= 0 && pad_id < V && (reinterpret_cast<uintptr_t>(stats) & 7) == 0);
  group_select_kernel<<<n_prompts, SELECT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(logits), ldx, V, reinterpret_cast<const float2*>(stats), beam_scores, cand_tokens, L, k, n_groups, n_cand,
      eos, n_eos, pad_id, diversity_penalty, done, out_scores, out_beams, out_tokens, next_beams, next_tokens);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) long long srgpt_kv_copy_workspace_bytes(int n_staged, int n_layers, int page_rows, int row_bytes) {
  if (n_staged < 0 || n_layers <= 0 || page_rows <= 0 || row_bytes <= 0) return -1;
  return (long long)n_staged * n_layers * 2 * page_rows * row_bytes;
}

extern "C" __attribute__((visibility("default"))) int srgpt_kv_copy_pages(void* pages, int n_layers, int n_pages, int page_rows, int row_bytes,
                                                                          const int* pairs, int n_pairs, int n_staged, void* workspace,
                                                                          long long workspace_bytes, void* stream) {
  SRGPT_CHECK_ARG(pages && pairs && n_layers > 0 && n_pages > 0 && page_rows > 0 && row_bytes > 0 && (row_bytes % 16) == 0);
  SRGPT_CHECK_ARG(n_pairs > 0 && n_pairs <= 65535 && n_staged >= 0 && n_staged <= n_pairs && 2 * n_layers <= 65535);
  SRGPT_CHECK_ARG(((reinterpret_cast<uintptr_t>(pages) | reinterpret_cast<uintptr_t>(pairs) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0);
  SRGPT_CHECK_ARG(n_staged == 0 || (workspace && workspace_bytes >= srgpt_kv_copy_workspace_bytes(n_staged, n_layers, page_rows, row_bytes)));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int4* pr = reinterpret_cast<const int4*>(pairs);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  kv_copy_kernel<<<dim3(2 * n_layers, n_pairs), COPY_THREADS, 0, st>>>(reinterpret_cast<uint8_t*>(pages), n_pages, page_rows, row_bytes, pr,
                                                                        n_staged, ws, 0);
  SRGPT_CHECK_LAUNCH();
  if (n_staged > 0) {
    kv_copy_kernel<<<dim3(2 * n_layers, n_staged), COPY_THREADS, 0, st>>>(reinterpret_cast<uint8_t*>(pages), n_pages, page_rows, row_bytes, pr,
                                                                           n_staged, ws, 1);
    SRGPT_CHECK_LAUNCH();
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_kv_broadcast_rows(void* pages, int n_layers, int n_pages, int page_rows, int row_bytes,
                                                                              const int* page_tables, int pt_stride, const int* pos, int pos_offset,
                                                                              const int* sel, int n_groups, int k, void* stream) {
  SRGPT_CHECK_ARG(pages && page_tables && pos && sel && n_layers > 0 && n_pages > 0 && page_rows > 0 && row_bytes > 0 && (row_bytes % 16) == 0);
  SRGPT_CHECK_ARG(pt_stride > 0 && n_groups > 0 && n_groups <= 65535 && k >= 1 && 2 * n_layers <= 65535);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(pages) & 15) == 0);
  kv_broadcast_kernel<<<dim3(2 * n_layers, n_groups), COPY_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<uint8_t*>(pages), n_pages, page_rows, row_bytes, page_tables, pt_stride, pos, pos_offset, sel, k);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
