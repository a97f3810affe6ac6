// Kernels behind forward(output_attentions=True, output_hidden_states=True) (DESIGN.md §4, §7):
//   * attn_probs_kernel : the causal attention probabilities softmax(Q K^T * scale) of one layer, written in the element type
//     straight into the caller's [n_seqs, n_heads, out_rows, out_rows] blocks - the S x S matrix the flash kernels never build.
//   * store_rows_kernel : copies the residual rows of packed sequences into a padded [n_seqs, out_rows, H] output.
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

// Row r of x [rows, H] (sequence s of the packed rows, local row r - cu[s]) -> dst + s * seq_stride + (row_off[s] + local) * ld.
__global__ void __launch_bounds__(128)
store_rows_kernel(const bf16* __restrict__ x, int H, int n_seqs, const int* __restrict__ cu_seqlens, bf16* __restrict__ dst, long long seq_stride,
                  long long ld, const int* __restrict__ row_off) {
  const int row = blockIdx.x;
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
               void* stream) {
  SRGPT_CHECK_ARG(x && dst && rows > 0 && n_seqs >= 1 && (cu_seqlens != nullptr || n_seqs == 1));
  SRGPT_CHECK_ARG((H % 8) == 0 && (ld % 8) == 0 && (seq_stride % 8) == 0 && ld >= H);
  SRGPT_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0);
  store_rows_kernel<<<rows, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const bf16*>(x), H, n_seqs, cu_seqlens,
                                                                              reinterpret_cast<bf16*>(dst), seq_stride, ld, row_off);
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
