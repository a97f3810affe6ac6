// Kernels behind forward(output_attentions=True, output_hidden_states=True) (DESIGN.md §4, §7):
//   * attn_probs_kernel : the causal attention probabilities softmax(Q K^T * scale) of one layer, written in the element type
//     straight into the caller's [n_seqs, n_heads, out_rows, out_rows] blocks - the S x S matrix the flash kernels never build.
//   * store_rows_kernel : copies the residual rows of packed sequences into a padded [n_seqs, out_rows, H] output (optionally at the
//     device step counter: generate()'s per-step hidden states).
//   * decode_stats_kernel / decode_probs_kernel : the probabilities of one-token decode steps over the paged KV cache, written at the
//     device step in generate()'s padded column layout (generate(output_attentions=True)).
// Reference: HF eager_attention_forward (softmax in fp32, then cast to the query dtype) and LlamaModel's hidden-state capture.
#include "common.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace probs {

// One CTA = 64 output rows of one (sequence, head); 4 warps of 16 rows each, mma.sync m16n8k16 with fp32 accumulation.
// mma.sync rather than wgmma: each warp's accumulator fragment holds whole 16-row strips, so the row max / sum of pass 1 and the
// normalised stores of pass 2 need only quad shuffles, and the kernel's cost is dominated by the probabilities it writes (2 bytes per
// 256 FLOP of Q K^T at head_dim 128, about the H100's FLOP-per-byte balance), not by the tensor-core issue rate.
constexpr int BM = 64, BN = 64, HD = 128, LD = HD + 8, NTHREADS = 128;

struct Smem {
  bf16 q[BM][LD];
  bf16 k[2][BN][LD];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32." SRGPT_ELEM_PTX "." SRGPT_ELEM_PTX ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// rows row0 .. row0 + 63 of one head of a sequence of len rows into a [64][LD] tile; rows outside [0, len) are zero
__device__ __forceinline__ void load_tile(bf16 (*dst)[LD], const bf16* __restrict__ src, int ld, int row0, int len) {
  for (int i = threadIdx.x; i < 64 * (HD / 8); i += NTHREADS) {
    const int r = i / (HD / 8), c = i % (HD / 8);
    const int row = row0 + r;
    if (row >= 0 && row < len)
      cp_async16(&dst[r][c * 8], src + (size_t)row * ld + c * 8);
    else
      *reinterpret_cast<uint4*>(&dst[r][c * 8]) = make_uint4(0, 0, 0, 0);
  }
}

// two neighbouring probabilities at columns c, c + 1 of an output row (c may be odd: the blocks sit at any padding offset)
__device__ __forceinline__ void store2(bf16* row, int c, float p0, float p1, int out_rows) {
  bf16* p = row + c;
  if (c >= 0 && c + 1 < out_rows && (reinterpret_cast<uintptr_t>(p) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(p0, p1);
    return;
  }
  if (c >= 0 && c < out_rows) p[0] = f2e(p0);
  if (c + 1 >= 0 && c + 1 < out_rows) p[1] = f2e(p1);
}

// zeros at columns [c0, c1) of one row, by the 32 lanes of a warp: 16-byte stores between an unaligned head and tail
__device__ __forceinline__ void zero_span(bf16* row, int c0, int c1, int lane) {
  if (c0 >= c1) return;
  const int mis = (int)((reinterpret_cast<uintptr_t>(row + c0) >> 1) & 7);
  const int head = min(c1 - c0, mis ? 8 - mis : 0);
  if (lane < head) row[c0 + lane] = f2e(0.f);
  const int v0 = c0 + head, nv = (c1 - v0) >> 3;
  for (int i = lane; i < nv; i += 32) *reinterpret_cast<uint4*>(row + v0 + 8 * i) = make_uint4(0, 0, 0, 0);
  const int t0 = v0 + 8 * nv;
  if (lane < c1 - t0) row[t0 + lane] = f2e(0.f);
}

// Grid (ceil(out_rows / 64), n_heads, n_seqs).  Output row o of sequence b holds its local row o - row_off[b]; the block's other rows
// and columns are zero.  Two passes over the key tiles up to the tile's diagonal: pass 1 the fp32 row max and sum (base 2, online),
// pass 2 recomputes the scores and stores exp2(s - m) / l.  K tiles stream through a double-buffered cp.async ring across both passes.
__global__ void __launch_bounds__(NTHREADS)
attn_probs_kernel(const bf16* __restrict__ q, int q_ld, const bf16* __restrict__ k, int k_ld, const int* __restrict__ cu_seqlens, int seqlen,
                  int group, float scale_log2, bf16* __restrict__ out, long long seq_stride, long long head_stride, long long ld, int out_rows,
                  const int* __restrict__ row_off) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int head = blockIdx.y, b = blockIdx.z, kvh = head / group;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lr = lane & 7, lmat = lane >> 3, g = lane >> 2, t4 = lane & 3;
  const int row_base = cu_seqlens != nullptr ? cu_seqlens[b] : 0;
  const int len = cu_seqlens != nullptr ? cu_seqlens[b + 1] - row_base : seqlen;
  const int off = row_off != nullptr ? row_off[b] : 0;
  const int o0 = blockIdx.x * BM, q0 = o0 - off;  // first output row of the tile, and its local row
  const int q_last = min(q0 + BM, len) - 1;
  const int nt = q_last < max(q0, 0) ? 0 : (q_last + BN) / BN;  // key tiles up to the diagonal of the tile's last valid row
  const bf16* qb = q + (size_t)row_base * q_ld + head * HD;
  const bf16* kb = k + (size_t)row_base * k_ld + kvh * HD;
  bf16* ob = out + b * seq_stride + head * head_stride;

  const int total = 2 * nt;
  if (total > 0) {
    load_tile(sm.q, qb, q_ld, q0, len);
    load_tile(sm.k[0], kb, k_ld, 0, len);
    cp_async_commit();
  }
  uint32_t qf[HD / 16][4];
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, inv[2] = {0.f, 0.f};
  const int qi0 = q0 + warp * 16 + g;  // local rows qi0 and qi0 + 8 of this thread
  const int r0 = o0 + warp * 16 + g;   // their output rows

  for (int it = 0; it < total; ++it) {
    const int cur = it & 1, j = it < nt ? it : it - nt;
    if (it + 1 < total) {
      load_tile(sm.k[cur ^ 1], kb, k_ld, (it + 1 < nt ? it + 1 : it + 1 - nt) * BN, len);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (it == 0) {
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) ldmatrix_x4(qf[kk], &sm.q[warp * 16 + lr + (lmat & 1) * 8][kk * 16 + (lmat >> 1) * 8]);
    }
    float s[BN / 8][4];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int np = 0; np < BN / 16; ++np) {
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        uint32_t bfr[4];
        ldmatrix_x4(bfr, &sm.k[cur][np * 16 + lr + (lmat >> 1) * 8][kk * 16 + (lmat & 1) * 8]);
        mma_16816(s[2 * np], qf[kk], bfr[0], bfr[1]);
        mma_16816(s[2 * np + 1], qf[kk], bfr[2], bfr[3]);
      }
    }
    // scale to base 2, causal mask (a key after the query, or a query outside the sequence)
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kv = j * BN + nb * 8 + 2 * t4 + (e & 1);
        const int qi = qi0 + (e >> 1) * 8;
        s[nb][e] = (kv > qi || qi >= len) ? -INFINITY : s[nb][e] * scale_log2;
      }
    }
    if (it < nt) {  // pass 1: running max and sum
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int nb = 0; nb < BN / 8; ++nb) {
        mx[0] = fmaxf(mx[0], fmaxf(s[nb][0], s[nb][1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[nb][2], s[nb][3]));
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(m_run[r], mx[r]);
        const float m_use = m_new == -INFINITY ? 0.f : m_new;
        float rs = 0.f;
#pragma unroll
        for (int nb = 0; nb < BN / 8; ++nb) rs += exp2f(s[nb][2 * r] - m_use) + exp2f(s[nb][2 * r + 1] - m_use);
        l_run[r] = l_run[r] * exp2f(m_run[r] - m_use) + rs;
        m_run[r] = m_new;
      }
    } else {  // pass 2: normalised probabilities
      if (it == nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
          l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
          inv[r] = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
          if (m_run[r] == -INFINITY) m_run[r] = 0.f;
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int orow = r0 + 8 * r;
        if (orow >= out_rows) continue;
        bf16* row = ob + orow * ld;
#pragma unroll
        for (int nb = 0; nb < BN / 8; ++nb) {
          const int c = off + j * BN + nb * 8 + 2 * t4;
          store2(row, c, exp2f(s[nb][2 * r] - m_run[r]) * inv[r], exp2f(s[nb][2 * r + 1] - m_run[r]) * inv[r], out_rows);
        }
      }
    }
    __syncthreads();  // every warp is done with buffer `cur` before it is refilled
  }
  // the rest of the tile's rows: columns before the sequence's block and after the last key tile
  const int c_lo = min(max(off, 0), out_rows), c_hi = max(c_lo, min(off + nt * BN, out_rows));
  for (int rr = warp; rr < BM; rr += NTHREADS / 32) {
    const int orow = o0 + rr;
    if (orow >= out_rows) break;
    bf16* row = ob + orow * ld;
    zero_span(row, 0, c_lo, lane);
    zero_span(row, c_hi, out_rows, lane);
  }
}

// Row r of x [rows, H] (sequence s of the packed rows, local row r - cu[s]) -> dst + s * seq_stride + (row_off[s] + local) * ld, and
// + (*step + step_offset) * step_stride when step != NULL.
__global__ void __launch_bounds__(128)
store_rows_kernel(const bf16* __restrict__ x, int H, int n_seqs, const int* __restrict__ cu_seqlens, bf16* __restrict__ dst, long long seq_stride,
                  long long ld, const int* __restrict__ row_off, const int* __restrict__ step, int step_offset, long long step_stride) {
  const int row = blockIdx.x;
  if (step != nullptr) dst += (long long)(*step + step_offset) * step_stride;
  int seq = 0, local = row;
  if (cu_seqlens != nullptr) {  // largest s with cu_seqlens[s] <= row
    int lo = 0, hi = n_seqs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (cu_seqlens[mid] <= row) lo = mid; else hi = mid - 1;
    }
    seq = lo;
    local = row - cu_seqlens[seq];
  }
  const int off = row_off != nullptr ? row_off[seq] : 0;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row * H);
  uint4* d = reinterpret_cast<uint4*>(dst + seq * seq_stride + (long long)(off + local) * ld);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) d[i] = src[i];
}

int store_rows(const void* x, int rows, int H, int n_seqs, const int* cu_seqlens, void* dst, long long seq_stride, long long ld, const int* row_off,
               void* stream, const int* step, int step_offset, long long step_stride) {
  SRGPT_CHECK_ARG(x && dst && rows > 0 && n_seqs >= 1 && (cu_seqlens != nullptr || n_seqs == 1));
  SRGPT_CHECK_ARG((H % 8) == 0 && (ld % 8) == 0 && (seq_stride % 8) == 0 && ld >= H && (step_stride % 8) == 0);
  SRGPT_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0);
  store_rows_kernel<<<rows, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const bf16*>(x), H, n_seqs, cu_seqlens,
                                                                              reinterpret_cast<bf16*>(dst), seq_stride, ld, row_off, step,
                                                                              step_offset, step_stride);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}


// ---- one-token decode steps over the paged cache ---------------------------------------------------------------------------------
// Query row r (position pos[r], so keys 0 .. pos[r]) of a step, heads kvh * G .. kvh * G + G - 1 of KV head kvh.  A quad of lanes takes
// one key (each lane 32 of its 128 dimensions, 16-byte loads in four interleaved strips, so a quad reads 64 contiguous bytes per load),
// and the quad's partial dot products meet by two xor shuffles: each K row is read once for the whole GQA group.  The logits are those
// of attn_probs_kernel: fp32 dot products of the rotated q and k, times scale * log2(e); the softmax is exp2f(s - m) / sum in fp32.
// Two launches over the same grid (128-key chunks of the key range, KV heads, rows), so that a long context spreads over many SMs:
// decode_stats_kernel writes each chunk's (max, sum) per head to ws, decode_probs_kernel combines the chunks of its row in chunk order
// and writes the probabilities of its chunk of output columns.
constexpr int DCHUNK = 128, DTHREADS = 128, DMAX_GROUP = 8;

struct DecodeArgs {
  const bf16* q;
  int q_ld;
  const bf16* kv_pages;
  const int* page_tables;
  int pt_stride, page_size, n_kv_heads, group;
  const int* pos;
  float scale_log2;
  const int* off;
  const int* n_prompt;
  int T, n_cols;
  const int* step;
  int step_offset;
  bf16* out;
  long long step_stride, row_stride, head_stride;
  float2* ws;  // [rows][n_heads][ceil(n_cols / DCHUNK)]
};

// the group's query rows as fp32 in shared memory
__device__ __forceinline__ void load_q_group(const DecodeArgs& a, float (*qs)[HD], int r, int kvh) {
  const bf16* src = a.q + (size_t)r * a.q_ld + (size_t)kvh * a.group * HD;
  for (int i = threadIdx.x; i < a.group * HD; i += DTHREADS) qs[i / HD][i % HD] = e2f(src[i]);
}

// the group's logits (base 2) of key j, in every lane of the quad
__device__ __forceinline__ void key_logits(const DecodeArgs& a, const int* pt, int kvh, int j, const float (*qs)[HD], float* s) {
  const int ql = threadIdx.x & 3;
  const unsigned qmask = 0xfu << (threadIdx.x & 28);  // the quad: the other quads of the warp may be on another key or done
  const int page = pt[j / a.page_size], slot = j % a.page_size;
  const bf16* kp = a.kv_pages + (((size_t)page * 2 + 0) * a.page_size + slot) * (size_t)a.n_kv_heads * HD + kvh * HD;
  float k[32];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 u = *reinterpret_cast<const uint4*>(kp + (i * 4 + ql) * 8);
    const bf16* e = reinterpret_cast<const bf16*>(&u);
#pragma unroll
    for (int t = 0; t < 8; ++t) k[i * 8 + t] = e2f(e[t]);
  }
#pragma unroll
  for (int g = 0; g < DMAX_GROUP; ++g) {
    if (g >= a.group) break;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int t = 0; t < 8; ++t) acc = fmaf(k[i * 8 + t], qs[g][(i * 4 + ql) * 8 + t], acc);
    acc += __shfl_xor_sync(qmask, acc, 1);
    acc += __shfl_xor_sync(qmask, acc, 2);
    s[g] = acc * a.scale_log2;
  }
}

// (m, l) of two parts of a softmax sum merged: m the larger max, l the sums rescaled to it (an empty part has m = -inf, l = 0)
__device__ __forceinline__ void merge_ml(float& m, float& l, float m2, float l2) {
  const float mn = fmaxf(m, m2);
  if (mn == -INFINITY) return;
  l = l * exp2f(m - mn) + l2 * exp2f(m2 - mn);
  m = mn;
}

__global__ void __launch_bounds__(DTHREADS) decode_stats_kernel(const DecodeArgs a) {
  __shared__ float qs[DMAX_GROUP][HD];
  __shared__ float2 part[DTHREADS / 32][DMAX_GROUP];
  const int c = blockIdx.x, kvh = blockIdx.y, r = blockIdx.z;
  const int P = a.pos[r] + 1, j0 = c * DCHUNK;
  if (j0 >= P) return;  // decode_probs_kernel reads the chunks below P only
  load_q_group(a, qs, r, kvh);
  __syncthreads();
  const int* pt = a.page_tables + (size_t)r * a.pt_stride;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float m[DMAX_GROUP], l[DMAX_GROUP], s[DMAX_GROUP];
#pragma unroll
  for (int g = 0; g < DMAX_GROUP; ++g) m[g] = -INFINITY, l[g] = 0.f;
  const int j1 = min(P, j0 + DCHUNK);
  for (int jb = j0; jb < j1; jb += DTHREADS / 4) {
    const int j = jb + (threadIdx.x >> 2);
    if (j >= j1) break;
    key_logits(a, pt, kvh, j, qs, s);
#pragma unroll
    for (int g = 0; g < DMAX_GROUP; ++g) {
      if (g >= a.group) break;
      merge_ml(m[g], l[g], s[g], 1.f);
    }
  }
  // quads -> warp (xor 4, 8, 16), warps -> CTA in warp order
#pragma unroll
  for (int g = 0; g < DMAX_GROUP; ++g) {
    if (g >= a.group) break;
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m[g], o), l2 = __shfl_xor_sync(0xffffffffu, l[g], o);
      merge_ml(m[g], l[g], m2, l2);
    }
    if (lane == 0) part[warp][g] = make_float2(m[g], l[g]);
  }
  __syncthreads();
  if (threadIdx.x < a.group) {
    const int g = threadIdx.x;
    float mm = -INFINITY, ll = 0.f;
    for (int w = 0; w < DTHREADS / 32; ++w) merge_ml(mm, ll, part[w][g].x, part[w][g].y);
    const int n_chunks = (a.n_cols + DCHUNK - 1) / DCHUNK;
    a.ws[((size_t)r * a.n_kv_heads * a.group + kvh * a.group + g) * n_chunks + c] = make_float2(mm, ll);
  }
}

__global__ void __launch_bounds__(DTHREADS) decode_probs_kernel(const DecodeArgs a) {
  __shared__ float qs[DMAX_GROUP][HD];
  __shared__ float2 stat[DMAX_GROUP];  // (max, 1 / sum) of each head of the group
  const int c = blockIdx.x, kvh = blockIdx.y, r = blockIdx.z;
  const int P = a.pos[r] + 1, n = a.n_prompt[r], off = a.off[r];
  const int cols = min(a.T + P - n, a.n_cols);  // the row's view: T prompt columns, then the generated keys
  const int c0 = c * DCHUNK, c1 = min(cols, c0 + DCHUNK);
  if (c0 >= c1) return;
  load_q_group(a, qs, r, kvh);
  if (threadIdx.x < a.group) {
    const int g = threadIdx.x, n_chunks = (a.n_cols + DCHUNK - 1) / DCHUNK;
    const float2* w = a.ws + ((size_t)r * a.n_kv_heads * a.group + kvh * a.group + g) * n_chunks;
    float mm = -INFINITY, ll = 0.f;
    for (int k = 0; k * DCHUNK < P; ++k) merge_ml(mm, ll, w[k].x, w[k].y);
    stat[g] = make_float2(mm, ll > 0.f ? 1.f / ll : 0.f);
  }
  __syncthreads();
  const int* pt = a.page_tables + (size_t)r * a.pt_stride;
  bf16* ob = a.out + (long long)(*a.step + a.step_offset) * a.step_stride + (long long)r * a.row_stride + (long long)kvh * a.group * a.head_stride;
  const int ql = threadIdx.x & 3;
  float s[DMAX_GROUP];
  for (int cb = c0; cb < c1; cb += DTHREADS / 4) {
    const int col = cb + (threadIdx.x >> 2);
    if (col >= c1) break;
    const int j = (col >= off && col < off + n) ? col - off : (col >= a.T ? n + col - a.T : -1);
    if (j >= 0 && j < P) {  // every lane of the quad takes part in the shuffles
      key_logits(a, pt, kvh, j, qs, s);
#pragma unroll
      for (int g = 0; g < DMAX_GROUP; ++g) {
        if (g >= a.group) break;
        if ((g & 3) == ql) ob[g * a.head_stride + col] = f2e(exp2f(s[g] - stat[g].x) * stat[g].y);
      }
    } else {
      for (int g = ql; g < a.group; g += 4) ob[g * a.head_stride + col] = f2e(0.f);
    }
  }
}

int decode_probs(const void* q, int q_ld, const void* kv_pages, const int* page_tables, int pt_stride, int page_size, const int* pos, int rows,
                 int n_heads, int n_kv_heads, int head_dim, float scale, const int* off, const int* n_prompt, int T, int n_cols, const int* step,
                 int step_offset, void* out, long long step_stride, long long row_stride, long long head_stride, float* ws, void* stream) {
  SRGPT_CHECK_ARG(q && kv_pages && page_tables && pos && off && n_prompt && step && out && ws);
  SRGPT_CHECK_ARG(rows >= 1 && rows <= 65535 && n_heads > 0 && n_kv_heads > 0 && n_kv_heads <= 65535 && (n_heads % n_kv_heads) == 0);
  SRGPT_CHECK_ARG(n_heads / n_kv_heads <= DMAX_GROUP && page_size > 0 && (pt_stride > 0 || rows == 1) && q_ld >= n_heads * head_dim);
  SRGPT_CHECK_ARG(T >= 1 && n_cols >= T && head_stride >= n_cols && row_stride >= head_stride * n_heads);
  SRGPT_CHECK_ARG(((q_ld % 8) == 0) && ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(kv_pages)) & 15) == 0);
  if (head_dim != HD) {
    set_last_error("srgpt_attention_probs_decode_bf16: head_dim %d unsupported (128 only)", head_dim);
    return SRGPT_ERR_UNSUPPORTED;
  }
  const DecodeArgs a{reinterpret_cast<const bf16*>(q), q_ld, reinterpret_cast<const bf16*>(kv_pages), page_tables, pt_stride, page_size,
                     n_kv_heads, n_heads / n_kv_heads, pos, scale * 1.4426950408889634f, off, n_prompt, T, n_cols, step, step_offset,
                     reinterpret_cast<bf16*>(out), step_stride, row_stride, head_stride, reinterpret_cast<float2*>(ws)};
  const dim3 grid(ceil_div(n_cols, DCHUNK), n_kv_heads, rows);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  decode_stats_kernel<<<grid, DTHREADS, 0, st>>>(a);
  SRGPT_CHECK_LAUNCH();
  decode_probs_kernel<<<grid, DTHREADS, 0, st>>>(a);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
}  // namespace probs
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_attention_probs_bf16(const void* q, int q_ld, const void* k, int k_ld, int n_seqs,
                                                                                 const int* cu_seqlens, int max_seqlen, int n_heads, int n_kv_heads,
                                                                                 int head_dim, float scale, void* out, long long seq_stride,
                                                                                 long long head_stride, long long ld, int out_rows,
                                                                                 const int* row_off, void* stream) {
  SRGPT_CHECK_ARG(q && k && out && n_seqs >= 1 && n_seqs <= 65535 && max_seqlen >= 1 && n_heads > 0 && n_heads <= 65535 && n_kv_heads > 0);
  SRGPT_CHECK_ARG((n_heads % n_kv_heads) == 0 && (cu_seqlens != nullptr || n_seqs == 1));
  SRGPT_CHECK_ARG((q_ld % 8) == 0 && (k_ld % 8) == 0 && ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k)) & 15) == 0);
  SRGPT_CHECK_ARG(out_rows >= max_seqlen && ld >= out_rows && head_stride >= ld * out_rows && seq_stride >= head_stride * n_heads);
  if (head_dim != probs::HD) {
    set_last_error("srgpt_attention_probs_bf16: head_dim %d unsupported (128 only)", head_dim);
    return SRGPT_ERR_UNSUPPORTED;
  }
  const int smem = (int)sizeof(probs::Smem);
  static bool configured = false;
  if (!configured) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(probs::attn_probs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const dim3 grid(ceil_div(out_rows, probs::BM), n_heads, n_seqs);
  probs::attn_probs_kernel<<<grid, probs::NTHREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(q), q_ld, reinterpret_cast<const bf16*>(k), k_ld, cu_seqlens, max_seqlen, n_heads / n_kv_heads,
      scale * 1.4426950408889634f, reinterpret_cast<bf16*>(out), seq_stride, head_stride, ld, out_rows, row_off);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_attention_probs_decode_bf16(
    const void* q, int q_ld, const void* kv_pages, const int* page_tables, int pt_stride, int page_size, const int* pos, int rows, int n_heads,
    int n_kv_heads, int head_dim, float scale, const int* off, const int* n_prompt, int T, int n_cols, const int* step, int step_offset, void* out,
    long long step_stride, long long row_stride, long long head_stride, float* ws, void* stream) {
  return probs::decode_probs(q, q_ld, kv_pages, page_tables, pt_stride, page_size, pos, rows, n_heads, n_kv_heads, head_dim, scale, off, n_prompt,
                             T, n_cols, step, step_offset, out, step_stride, row_stride, head_stride, ws, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_store_step_rows_bf16(const void* x, int rows, int H, const int* step, int step_offset,
                                                                                 void* dst, long long step_stride, long long row_stride,
                                                                                 void* stream) {
  SRGPT_CHECK_ARG(step != nullptr);
  return probs::store_rows(x, rows, H, 1, nullptr, dst, 0, row_stride, nullptr, stream, step, step_offset, step_stride);
}
