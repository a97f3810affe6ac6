// Decode-time weight-streaming kernels (one new token): y = W · x with W [N, K] bf16 read exactly
// once from HBM.  At batch 1 the whole Llama decode step is bound by these reads (15 GB / token for
// Llama-3-8B, SURVEY.md §8d), so this kernel is written against the HBM roofline.
//
// Design (earlier persistent-warp and bulk-copy-ring + CTA-level K split versions streamed more slowly than this one):
//   * one warp = one PAIR of weight rows, read with 8 independent 16-byte streaming loads in flight per
//     lane (ld.global.nc.L1::no_allocate).  A warp is latency-bound by design (4 KB in flight), the chip
//     is saturated by having >= 2000 warps resident; CTAs are NOT persistent, so the hardware scheduler
//     balances the row pairs dynamically and no warp ever owns 2 pairs while another owns 1;
//   * the first 8 loads of every warp are issued BEFORE anything that depends on the previous kernel;
//     programmatic dependent launch (griddepcontrol.launch_dependents / .wait) lets the next kernel's
//     CTAs take the SM slots the current kernel frees in its tail, so launch latency, the first HBM
//     round trip and the RMSNorm prologue overlap the previous kernel instead of adding to the step;
//   * x (RMS-normalised in the prologue when requested) is staged once per CTA in shared memory;
//   * the pair is chosen so the fused epilogue is warp-local: (gate_i, up_i) for SwiGLU, (d, d + hd/2)
//     of one head for RoPE + KV-cache append, two vocabulary rows for lm_head + argmax.
// Rounding points follow the reference's bf16 torch ops (modeling_llama.py:429-431,186-191,221,668,682).
//
// The weights come in one of three formats (Bf16, Packed12 = the lossless 12-bit packing of pack12.cuh, Nf4 = the planes of nf4.cuh).
// A format only says how a batch of 4 chunks per lane and row is loaded and turned into the element-type chunks dot8 reads; the kernel
// around it (row pairs, x staging, the prefetch before the dependency wait, the chunk order of every lane's fma chain and the epilogue)
// is one, so the packed and NF4 kernels are bit-identical to the bf16 kernel over the same (dequantized) matrix.
#include <type_traits>

#include "common.cuh"
#include "fp8.cuh"
#include "nf4.cuh"
#include "pack12.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace gemv {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
enum { MODE_LM = 3 };

struct Params {
  const bf16* x;
  const bf16* W;
  int ldw;
  bf16* y;
  int N, K;
  const bf16* norm_weight;
  float eps;
  const bf16* residual;
  // QKV_ROPE
  int n_heads, n_kv_heads, hd;
  const bf16* cos_tab;
  const bf16* sin_tab;
  const int* pos;
  bf16* kv_pages;
  const int* page_table;
  int page_size;
  // LM
  float* logits_out;
  float* part_val;
  int* part_idx;
  unsigned long long* trace;  // optional timeline record (srgpt_trace_begin)
  // tensor parallelism (srgpt_gemv_tp_bf16): this rank's slice of the heads / of the reduction dimension
  int kv_heads_total;         // KV-cache row = kv_heads_total * hd elements (0: n_kv_heads); the rank writes heads [kv_head_off, +n_kv_heads)
  int kv_head_off;
  float* y_f32;               // PLAIN mode: un-rounded fp32 partial dot products go here instead of bf16 y (+ residual)
  srgpt_packed12 pk;          // Packed12's weights (W is unused there)
  srgpt_nf4 nf;               // Nf4's planes
};

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// stage x (optionally RMS-normalised) into shared memory as bf16.
// Fast path (K <= 2 * THREADS * 8 = 4096, the two RMSNorm-fused kernels of a layer): every thread keeps its <= 2
// chunks of x in registers between the sum of squares and the scaling, and the (static) norm weights `nw` were
// fetched before the dependency wait -> one L2 round trip on the critical path instead of three.
__device__ __forceinline__ void stage_x(const bf16* __restrict__ x, const bf16* __restrict__ norm_weight, float eps, int K,
                                        bf16* sx, float* red, const uint4* nw_pre, bool nw_pre_valid) {
  const int nchunk = K >> 3;
  if (norm_weight == nullptr) {
    for (int c = threadIdx.x; c < nchunk; c += THREADS)
      reinterpret_cast<uint4*>(sx)[c] = reinterpret_cast<const uint4*>(x)[c];
  } else if (nw_pre_valid) {
    uint4 xr[2];
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c = threadIdx.x + k * THREADS;
      xr[k] = make_uint4(0, 0, 0, 0);
      if (c < nchunk) xr[k] = reinterpret_cast<const uint4*>(x)[c];
      float f[8];
      unpack8(xr[k], f);
#pragma unroll
      for (int t = 0; t < 8; ++t) sq += f[t] * f[t];
    }
    const float rstd = rsqrtf(block_sum(sq, red) / (float)K + eps);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c = threadIdx.x + k * THREADS;
      if (c < nchunk) {
        float f[8], w[8], o[8];
        unpack8(xr[k], f);
        unpack8(nw_pre[k], w);
#pragma unroll
        for (int t = 0; t < 8; ++t) o[t] = w[t] * bf16_round(f[t] * rstd);
        reinterpret_cast<uint4*>(sx)[c] = pack8(o);
      }
    }
  } else {
    float sq = 0.f;
    for (int c = threadIdx.x; c < nchunk; c += THREADS) {
      float f[8];
      unpack8(reinterpret_cast<const uint4*>(x)[c], f);
#pragma unroll
      for (int t = 0; t < 8; ++t) sq += f[t] * f[t];
    }
    const float rstd = rsqrtf(block_sum(sq, red) / (float)K + eps);
    for (int c = threadIdx.x; c < nchunk; c += THREADS) {
      float f[8], w[8], o[8];
      unpack8(reinterpret_cast<const uint4*>(x)[c], f);
      unpack8(reinterpret_cast<const uint4*>(norm_weight)[c], w);
#pragma unroll
      for (int t = 0; t < 8; ++t) o[t] = w[t] * bf16_round(f[t] * rstd);
      reinterpret_cast<uint4*>(sx)[c] = pack8(o);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float dot8(const uint4& w, const float* xf) {
  float f[8];
  unpack8(w, f);
  float a = 0.f;
#pragma unroll
  for (int t = 0; t < 8; ++t) a = fmaf(f[t], xf[t], a);
  return a;
}

__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

template <int MODE>
__device__ __forceinline__ void pair_rows(const Params& p, int pi, int& r0, int& r1) {
  if (MODE == SRGPT_GEMV_QKV_ROPE) {
    const int half = p.hd >> 1;
    const int head = pi / half, j = pi - head * half;
    r0 = head * p.hd + j;
    r1 = r0 + half;
  } else {
    r0 = 2 * pi;
    r1 = r0 + 1;
    if (MODE == MODE_LM && r1 >= p.N) r1 = r0;  // odd vocabulary: the last pair streams row r0 twice
  }
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

// cp.async.wait_group takes an immediate: wait until at most n (0 or 1) of this thread's newest commit groups are pending
__device__ __forceinline__ void cp_async_wait_pending(int n) {
  if (n == 0) asm volatile("cp.async.wait_group 0;" ::: "memory");
  else asm volatile("cp.async.wait_group 1;" ::: "memory");
}

// ---- weight formats.  A format streams the two rows of a warp in batches: batch b holds chunks (8 weights) c = 128 b + lane + 32 i,
//      i = 0..3, of both rows for lane `lane`.  Its members:
//        setup(p, r0, r1, lane)      the rows' addresses (and per-CTA tables), before any weight is requested;
//        load_side(p, r0, r1, lane)  static per-row data the decode needs, requested after the first batches so its dependent loads
//                                    do not delay them;
//        nbatch(p, lane)             the whole batches of the lane;
//        Raw, load(b)                one batch as loaded into registers;
//        cp_async(slot, lane, b), read_slot(slot, lane)   the same batch through one SLOT-byte slot of the warp's shared memory (every
//                                    lane reads back exactly the vectors it requested, so no barrier is needed);
//        decode(raw, b, lane, w0, w1)   the element-type chunks i of rows r0 / r1;
//        tail(nb, nchunk, lane, px, a0, a1)   the lane's chunks after its nb whole batches, if a row may end inside a batch;
//        DEPTH, REFILL               batches 1..DEPTH go to the slots before the dependency wait; with REFILL a slot is refilled with
//                                    batch b + DEPTH as soon as batch b is read from it (a ring), else later batches load into registers.

// bf16: a batch is 4 x 16 bytes per row.  A row need not be whole batches (K % 1024 != 0): a lane's last chunks after its whole batches
// are taken one at a time (tail).  One slot, not refilled: a ring was not measured for this format.
struct Bf16 {
  static constexpr int SLOT = 2 * 4 * 32 * 16;  // both rows x 4 chunks x 32 lanes x 16 B = 4 KB
  static constexpr int DEPTH = 1;
  static constexpr bool REFILL = false;
  struct Raw {
    uint4 u0[4], u1[4];
  };
  const uint4 *p0, *p1;  // the lane's first chunk of rows r0 / r1

  __device__ __forceinline__ void setup(const Params& p, int r0, int r1, int lane) {
    p0 = reinterpret_cast<const uint4*>(p.W + (size_t)r0 * p.ldw) + lane;
    p1 = reinterpret_cast<const uint4*>(p.W + (size_t)r1 * p.ldw) + lane;
  }
  __device__ __forceinline__ void load_side(const Params&, int, int, int) {}
  __device__ __forceinline__ int nbatch(const Params& p, int lane) const {
    const int n = (p.K >> 3) - lane - 96;  // batch b is whole while 128 b + lane + 96 < K / 8
    return n > 0 ? (n + 127) >> 7 : 0;
  }
  __device__ __forceinline__ Raw load(int b) const {
    Raw t;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      t.u0[i] = ld_stream16(p0 + b * 128 + 32 * i);
      t.u1[i] = ld_stream16(p1 + b * 128 + 32 * i);
    }
    return t;
  }
  // the verify kernel's batches run to the end of the row: chunks past it are zero
  __device__ __forceinline__ Raw load_bounded(int b, int nchunk, int lane) const {
    Raw t;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = b * 128 + 32 * i;
      t.u0[i] = make_uint4(0, 0, 0, 0);
      t.u1[i] = make_uint4(0, 0, 0, 0);
      if (c + lane < nchunk) {
        t.u0[i] = ld_stream16(p0 + c);
        t.u1[i] = ld_stream16(p1 + c);
      }
    }
    return t;
  }
  // chunk i of row r0 at +512 i, of row r1 at +2048 + 512 i
  __device__ __forceinline__ void cp_async(uint8_t* slot, int lane, int b) const {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(slot + lane * 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      cp_async16(d + i * 512, p0 + b * 128 + 32 * i);
      cp_async16(d + 2048 + i * 512, p1 + b * 128 + 32 * i);
    }
  }
  __device__ __forceinline__ Raw read_slot(const uint8_t* slot, int lane) const {
    const uint4* s = reinterpret_cast<const uint4*>(slot + lane * 16);
    Raw t;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      t.u0[i] = s[32 * i];
      t.u1[i] = s[128 + 32 * i];
    }
    return t;
  }
  __device__ __forceinline__ void decode(const Raw& t, int, int, uint4 (&w0)[4], uint4 (&w1)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      w0[i] = t.u0[i];
      w1[i] = t.u1[i];
    }
  }
  __device__ __forceinline__ void tail(int nb, int nchunk, int lane, const uint4* px, float& a0, float& a1) const {
    for (int c = nb * 128; c + lane < nchunk; c += 32) {
      float xf[8];
      unpack8(px[c + lane], xf);
      a0 += dot8(ld_stream16(p0 + c), xf);
      a1 += dot8(ld_stream16(p1 + c), xf);
    }
  }
};

// ---- packed weights: one batch (4 chunks = 3 x 16 bytes) of one row for one lane.  Batch b of a row starts at uint4 64 b of its
//      sm plane row (chunks 0,1 then 2,3 of every lane) and at uint4 32 b of its ex plane row (pack12.cuh).
struct Raw12 {
  uint4 s01, s23, e;
};

__device__ __forceinline__ Raw12 ld_raw12(const uint4* sm_lane, const uint4* ex_lane, int b) {
  Raw12 q;
  q.s01 = ld_stream16(sm_lane + b * 64);
  q.s23 = ld_stream16(sm_lane + b * 64 + 32);
  q.e = ld_stream16(ex_lane + b * 32);
  return q;
}

__device__ __forceinline__ void decode_batch(const Raw12& q, uint32_t bp, uint4 (&w)[4]) {
  w[0] = pack12::decode_chunk(q.s01.x, q.s01.y, q.e.x, bp);
  w[1] = pack12::decode_chunk(q.s01.z, q.s01.w, q.e.y, bp);
  w[2] = pack12::decode_chunk(q.s23.x, q.s23.y, q.e.z, bp);
  w[3] = pack12::decode_chunk(q.s23.z, q.s23.w, q.e.w, bp);
}

// The exceptions of one row that fall into batch b: their exponent fields are ORed into the decoded chunks (where code 0 left 0).
// Lane k holds entry k of the row's list (exc), j is the next entry not yet applied; j and n are warp-uniform and the list is
// sorted by column, so a batch without exceptions costs one shuffle.  Selects, not indexing, keep w in registers.
__device__ __forceinline__ void patch_batch(uint4 (&w)[4], int exc, int n, int& j, int b, int lane) {
  while (j < n) {
    const int v = __shfl_sync(0xffffffffu, exc, j);
    const int col = v >> 8;
    if ((col >> 10) != b) break;
    const int cc = col >> 3, t = col & 7;
    const uint32_t bits = ((cc & 31) == lane) ? (uint32_t)(v & 0xFF) << (7 + 16 * (t & 1)) : 0u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t m = (i == ((cc >> 5) & 3)) ? bits : 0u;
      w[i].x |= (t >> 1) == 0 ? m : 0u;
      w[i].y |= (t >> 1) == 1 ? m : 0u;
      w[i].z |= (t >> 1) == 2 ? m : 0u;
      w[i].w |= (t >> 1) == 3 ? m : 0u;
    }
    ++j;
  }
}
// K % 1024 == 0.  A ring of depth 2: at K = 4096 that is 56 KB per CTA, so the 3 CTAs per SM the registers allow still fit and 3 of a
// row's 4 batches are requested before the dependency wait.  Deeper rings (2 CTAs per SM) made o_proj and down_proj stream faster but
// delayed the kernel after them by more (DESIGN.md §5).
struct Packed12 {
  static constexpr int SLOT = 2 * 3 * 32 * 16;  // both rows x 3 vectors x 32 lanes x 16 B = 3 KB
  static constexpr int DEPTH = 2;
  static constexpr bool REFILL = true;
  struct Raw {
    Raw12 q0, q1;
  };
  const uint4 *sm0, *ex0;  // this lane's vectors of row r0; row r1 is drow_ex rows further (sm: 2 drow_ex uint4 per ex uint4)
  int drow_ex;
  uint32_t bp0, bp1;  // base - 1 of the two rows
  int exc0, exc1;     // this lane's entry of each row's exception list
  int n0, n1;         // list lengths
  int j0, j1;         // next entry to apply

  __device__ __forceinline__ void setup(const Params& p, int r0, int r1, int lane) {
    sm0 = reinterpret_cast<const uint4*>(p.pk.sm) + (size_t)r0 * (p.K >> 4) + lane;
    ex0 = reinterpret_cast<const uint4*>(p.pk.ex) + (size_t)r0 * (p.K >> 5) + lane;
    drow_ex = (r1 - r0) * (p.K >> 5);
  }
  __device__ __forceinline__ void load_side(const Params& p, int r0, int r1, int lane) {
    const int e0 = p.pk.row_ptr[r0], e1 = p.pk.row_ptr[r1];
    n0 = min(p.pk.row_ptr[r0 + 1] - e0, pack12::MAX_EXC_PER_ROW);
    n1 = min(p.pk.row_ptr[r1 + 1] - e1, pack12::MAX_EXC_PER_ROW);
    if (lane < n0) exc0 = p.pk.exc[e0 + lane];
    if (lane < n1) exc1 = p.pk.exc[e1 + lane];
    bp0 = (uint32_t)p.pk.base[r0] - 1u;
    bp1 = (uint32_t)p.pk.base[r1] - 1u;
  }
  __device__ __forceinline__ int nbatch(const Params& p, int) const { return p.K >> 10; }
  __device__ __forceinline__ Raw load(int b) const { return {ld_raw12(sm0, ex0, b), ld_raw12(sm0 + 2 * drow_ex, ex0 + drow_ex, b)}; }
  __device__ __forceinline__ Raw load_bounded(int b, int, int) const { return load(b); }
  // row r0: sm 01, sm 23, ex at +0 / 512 / 1024, row r1 at +1536 ...
  __device__ __forceinline__ void cp_async(uint8_t* slot, int lane, int b) const {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(slot + lane * 16);
    const uint4 *s = sm0 + b * 64, *e = ex0 + b * 32;
    cp_async16(d, s);
    cp_async16(d + 512, s + 32);
    cp_async16(d + 1024, e);
    cp_async16(d + 1536, s + 2 * drow_ex);
    cp_async16(d + 2048, s + 2 * drow_ex + 32);
    cp_async16(d + 2560, e + drow_ex);
  }
  __device__ __forceinline__ Raw read_slot(const uint8_t* slot, int lane) const {
    const uint4* s = reinterpret_cast<const uint4*>(slot + lane * 16);
    return {{s[0], s[32], s[64]}, {s[96], s[128], s[160]}};
  }
  __device__ __forceinline__ void decode(const Raw& t, int b, int lane, uint4 (&w0)[4], uint4 (&w1)[4]) {
    decode_batch(t.q0, bp0, w0);
    decode_batch(t.q1, bp1, w1);
    patch_batch(w0, exc0, n0, j0, b, lane);
    patch_batch(w1, exc1, n1, j1, b, lane);
  }
  __device__ __forceinline__ void tail(int, int, int, const uint4*, float&, float&) const {}
};

// ---- NF4 weights (nf4.cuh): per batch a lane streams one 16-byte vector of codes per row (its 4 chunks) and lanes 0-15 / 16-31 one
//      scale each of row r0 / r1 (the row's 16 blocks of the batch, 64 bytes per row).  Lane l's chunk i lies in block 4 i + l / 8 of
//      the batch, so its two scales come from lanes 4 i + l / 8 and 16 + 4 i + l / 8 by shuffle.  K % 1024 == 0; the ring of Packed12.
__device__ __forceinline__ uint32_t word_of(const uint4& v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w)); }

struct Nf4 {
  static constexpr int SLOT = 2 * 32 * 16 + 32 * 4;  // both rows' code vectors (2 x 512 B) and the 32 scales (128 B)
  static constexpr int DEPTH = 2;
  static constexpr bool REFILL = true;
  struct Raw {
    uint4 q0, q1;
    float s;
  };
  const uint4 *q0, *q1;
  const float* s_lane;
  const float* tab;  // the 16 code values in shared memory, published by stage_x's barrier

  __device__ __forceinline__ void setup(const Params& p, int r0, int r1, int lane) {
    __shared__ float code_tab[16];
    if (threadIdx.x < 16) code_tab[threadIdx.x] = nf4::code_value(threadIdx.x);
    tab = code_tab;
    q0 = reinterpret_cast<const uint4*>(p.nf.q + (size_t)r0 * (p.K >> 1)) + lane;
    q1 = reinterpret_cast<const uint4*>(p.nf.q + (size_t)r1 * (p.K >> 1)) + lane;
    s_lane = p.nf.scale + (size_t)(lane < 16 ? r0 : r1) * (p.K >> 6) + (lane & 15);
  }
  __device__ __forceinline__ void load_side(const Params&, int, int, int) {}
  __device__ __forceinline__ int nbatch(const Params& p, int) const { return p.K >> 10; }
  __device__ __forceinline__ Raw load(int b) const { return {ld_stream16(q0 + b * 32), ld_stream16(q1 + b * 32), __ldg(s_lane + b * 16)}; }
  // the verify kernel's batches: rows are whole batches (K % 1024 == 0)
  __device__ __forceinline__ Raw load_bounded(int b, int, int) const { return load(b); }
  // codes of r0 / r1 at +0 / +512, scales at +1024
  __device__ __forceinline__ void cp_async(uint8_t* slot, int lane, int b) const {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(slot + lane * 16);
    const uint32_t ds = (uint32_t)__cvta_generic_to_shared(slot + 1024 + lane * 4);
    cp_async16(d, q0 + b * 32);
    cp_async16(d + 512, q1 + b * 32);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ds), "l"(s_lane + b * 16) : "memory");
  }
  __device__ __forceinline__ Raw read_slot(const uint8_t* slot, int lane) const {
    return {*reinterpret_cast<const uint4*>(slot + lane * 16), *reinterpret_cast<const uint4*>(slot + 512 + lane * 16),
            *reinterpret_cast<const float*>(slot + 1024 + lane * 4)};
  }
  __device__ __forceinline__ void decode(const Raw& t, int, int lane, uint4 (&w0)[4], uint4 (&w1)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float s0 = __shfl_sync(0xffffffffu, t.s, 4 * i + (lane >> 3));
      const float s1 = __shfl_sync(0xffffffffu, t.s, 16 + 4 * i + (lane >> 3));
      w0[i] = nf4::dequant8(word_of(t.q0, i), s0, tab);
      w1[i] = nf4::dequant8(word_of(t.q1, i), s1, tab);
    }
  }
  __device__ __forceinline__ void tail(int, int, int, const uint4*, float&, float&) const {}
};

// slots per warp: DEPTH, or for a ring DEPTH clamped to the batches after batch 0
template <class Fmt>
__host__ __device__ __forceinline__ int ring_slots(int K) {
  static_assert(Fmt::DEPTH <= 2, "cp_async_wait_pending waits for 0 or 1 pending groups");
  return Fmt::REFILL && (K >> 10) - 1 < Fmt::DEPTH ? (K >> 10) - 1 : Fmt::DEPTH;
}

// batch b of both rows in chunk order through dot8: every lane's fma chain is that of the bf16 kernel over the same (dequantized) weights
template <class Fmt>
__device__ __forceinline__ void consume(Fmt& f, const typename Fmt::Raw& t, int b, int lane, const uint4* px, float& a0, float& a1) {
  uint4 w0[4], w1[4];
  f.decode(t, b, lane, w0, w1);
  const int c = b * 128 + lane;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float xf[8];
    unpack8(px[c + 32 * i], xf);
    a0 += dot8(w0[i], xf);
    a1 += dot8(w1[i], xf);
  }
}

// The stores of one token's results for a row pair: the fp32 sums a0 / a1 of rows r0 / r1 with the mode's rounding points (those of the
// reference's torch ops, see the top of the file).  y and residual are the token's rows, pos its position and page_table its sequence's
// page table (QKV + RoPE), logits its row of fp32 logits (lm_head, may be null); lm_head returns the pair's best (value, row) in best / besti.
template <int MODE>
__device__ __forceinline__ void store_pair(const Params& p, bf16* y, const bf16* residual, float* logits, int pos, const int* page_table, int pi,
                                           int r0, int r1, float a0, float a1, float& best, int& besti) {
  if (MODE == SRGPT_GEMV_PLAIN && p.y_f32 != nullptr) {
    // row-parallel linear of a tensor-parallel rank: the partial sums over this rank's K slice, reduced across ranks afterwards
    *reinterpret_cast<float2*>(p.y_f32 + r0) = make_float2(a0, a1);
  } else if (MODE == SRGPT_GEMV_PLAIN) {
    float y0 = bf16_round(a0), y1 = bf16_round(a1);
    if (residual != nullptr) {
      y0 += e2f(residual[r0]);
      y1 += e2f(residual[r1]);
    }
    *reinterpret_cast<uint32_t*>(y + r0) = pack_bf16x2(y0, y1);
  } else if (MODE == SRGPT_GEMV_SWIGLU) {
    const float g = bf16_round(a0), u = bf16_round(a1);
    y[pi] = f2e(bf16_round(silu(g)) * u);
  } else if (MODE == SRGPT_GEMV_QKV_ROPE) {
    const int half = p.hd >> 1;
    const int head = pi / half, j = pi - head * half;
    float v0 = bf16_round(a0), v1 = bf16_round(a1);
    if (head < p.n_heads + p.n_kv_heads) {
      const float cs = e2f(p.cos_tab[(size_t)pos * half + j]);
      const float sn = e2f(p.sin_tab[(size_t)pos * half + j]);
      const float o0 = bf16_round(bf16_round(v0 * cs) + bf16_round(-v1 * sn));
      const float o1 = bf16_round(bf16_round(v1 * cs) + bf16_round(v0 * sn));
      v0 = o0;
      v1 = o1;
    }
    if (head < p.n_heads) {
      y[r0] = f2e(v0);
      y[r1] = f2e(v1);
    } else {
      const int page = page_table[pos / p.page_size], slot = pos % p.page_size;
      const bool is_v = head >= p.n_heads + p.n_kv_heads;
      const int kh = head - p.n_heads - (is_v ? p.n_kv_heads : 0) + p.kv_head_off;
      const int kv_row = (p.kv_heads_total > 0 ? p.kv_heads_total : p.n_kv_heads) * p.hd;
      bf16* dst = p.kv_pages + (((size_t)page * 2 + (is_v ? 1 : 0)) * p.page_size + slot) * kv_row + kh * p.hd;
      dst[j] = f2e(v0);
      dst[j + half] = f2e(v1);
    }
  } else {  // MODE_LM: logits = lm_head(h).float() -> bf16 rounding first (modeling_llama.py:1044-1045)
    a0 = bf16_round(a0);
    a1 = bf16_round(a1);
    if (logits != nullptr) {
      logits[r0] = a0;
      if (r1 != r0) logits[r1] = a1;
    }
    best = a0;
    besti = r0;
    if (r1 != r0 && better(a1, r1, best, besti)) { best = a1; besti = r1; }
  }
}

// The end of every one-token decode GEMV: the warp sums of the lane partials a0 / a1 of rows r0 / r1, the pair's stores and, for
// lm_head, the CTA's arg max partial.
template <int MODE>
__device__ __forceinline__ void epilogue(const Params& p, bool active, int pi, int r0, int r1, int warp, int lane, float a0, float a1, float* sv,
                                         int* si) {
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  float best = -INFINITY;
  int besti = 0x7fffffff;
  if (active && lane == 0)
    store_pair<MODE>(p, p.y, p.residual, p.logits_out, MODE == SRGPT_GEMV_QKV_ROPE ? *p.pos : 0, p.page_table, pi, r0, r1, a0, a1, best, besti);
  if (MODE == MODE_LM) {
    if (lane == 0) { sv[warp] = best; si[warp] = besti; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < WARPS; ++w)
        if (better(sv[w], si[w], best, besti)) { best = sv[w]; besti = si[w]; }
      p.part_val[blockIdx.x] = best;
      p.part_idx[blockIdx.x] = besti;
    }
  }
}

// The one-token decode GEMV over the weights of format Fmt.  Batch 0 goes to registers and batches 1..DEPTH to the warp's slots (one
// commit group each), all requested before the dependency wait, like the rows' side data and the RMSNorm weights.  With a ring, batch b
// sits in slot (b - 1) % depth: as soon as the lane has read its vectors of batch b back into registers it requests batch b + depth into
// the same slot (the reads precede the cp.async in the thread's program order), so depth batches stay in flight while batch b is decoded
// and consumed.  Batches are consumed in chunk order.
template <int MODE, class Fmt>
__global__ void __launch_bounds__(THREADS, 3) decode_gemv_kernel(const Params p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float red[32];
  __shared__ float sv[WARPS];
  __shared__ int si[WARPS];
  bf16* sx = reinterpret_cast<bf16*>(smem_raw);
  const uint4* px = reinterpret_cast<const uint4*>(sx);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  trace_mark(p.trace, 0);
  const int npairs = (MODE == MODE_LM) ? ((p.N + 1) >> 1) : (p.N >> 1);
  const int pi = blockIdx.x * WARPS + warp;
  const bool active = pi < npairs;
  // every warp, with or without a pair (one without loads nothing): then r0 / r1 are a function of pi that the epilogue recomputes
  // instead of holding it in a register through the main loop, which keeps every format within 80 registers
  int r0, r1;
  pair_rows<MODE>(p, pi, r0, r1);

  Fmt f{};
  f.setup(p, r0, r1, lane);
  uint8_t* ring = smem_raw + (size_t)p.K * 2 + (size_t)warp * ring_slots<Fmt>(p.K) * Fmt::SLOT;
  const int nbatch = f.nbatch(p, lane);
  typename Fmt::Raw t0;
  if (active && nbatch > 0) {
    t0 = f.load(0);
#pragma unroll
    for (int b = 0; b < Fmt::DEPTH && 1 + b < nbatch; ++b) {
      f.cp_async(ring + b * Fmt::SLOT, lane, 1 + b);
      cp_async_commit();
    }
  }
  if (active) f.load_side(p, r0, r1, lane);
  // norm weights are static too: fetch them before the wait when a thread owns at most 2 chunks of x
  uint4 nw_pre[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  const bool nw_pre_valid = (p.norm_weight != nullptr) && ((p.K >> 3) <= 2 * THREADS);
  if (nw_pre_valid) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int cc = threadIdx.x + k * THREADS;
      if (cc < (p.K >> 3)) nw_pre[k] = reinterpret_cast<const uint4*>(p.norm_weight)[cc];
    }
  }
  pdl_launch_dependents();
  pdl_wait();  // activations written by earlier kernels are visible from here on
  trace_mark(p.trace, 1);

  stage_x(p.x, p.norm_weight, p.eps, p.K, sx, red, nw_pre, nw_pre_valid);

  float a0 = 0.f, a1 = 0.f;
  if (active && nbatch > 0) {
    consume(f, t0, 0, lane, px, a0, a1);
    const int depth = nbatch - 1 < Fmt::DEPTH ? nbatch - 1 : Fmt::DEPTH;  // batches in the slots
    int slot = 0;
    for (int b = 1; b < nbatch; ++b) {
      typename Fmt::Raw t;
      if (Fmt::REFILL || b <= depth) {
        // batch b sits in slot `slot`; the groups committed after its own may still be pending
        cp_async_wait_pending(Fmt::REFILL ? min(depth - 1, nbatch - 1 - b) : depth - b);
        uint8_t* s = ring + slot * Fmt::SLOT;
        t = f.read_slot(s, lane);
        if (Fmt::REFILL && b + depth < nbatch) {
          f.cp_async(s, lane, b + depth);
          cp_async_commit();
        }
        if (++slot == depth) slot = 0;
      } else {
        t = f.load(b);
      }
      consume(f, t, b, lane, px, a0, a1);
    }
  }
  if (active) f.tail(nbatch, p.K >> 3, lane, px, a0, a1);
  epilogue<MODE>(p, active, pi, r0, r1, warp, lane, a0, a1, sv, si);
  trace_mark(p.trace, 2);
}

// ---- FP8 (E4M3) W8A8 one-token GEMV (the decode step of a quantization="fp8" model; definition: include/srgpt_b200.h srgpt_fp8) ----------
// x (RMS-normalised when norm_weight is given) is staged as by the kernels above, then quantized in place by the activation quantizer's
// definition: the CTA's max |x|, inv = 448 / a, and every element replaced by its E4M3 value, held exactly as an element-type value.  A
// warp streams a row pair of codes (one 16-byte vector = 16 weights per lane and load, 4 loads per row and batch, the next batch
// requested while the current one is consumed), turns each vector into two element-type chunks (exact) and runs dot8 over them: every
// product is exact and acc is their fp32 sum.  The epilogue multiplies acc by fl32(s_x * s_w[row]) and stores through store_pair, the
// rounding points of the other formats.  K % 16 == 0.
__device__ __forceinline__ float stage_quantize_e4m3(bf16* sx, int K, float* red) {
  const int nchunk = K >> 3;
  float m = 0.f;
  for (int c = threadIdx.x; c < nchunk; c += THREADS) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(sx)[c], f);
#pragma unroll
    for (int t = 0; t < 8; ++t) m = fmaxf(m, fabsf(f[t]));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < WARPS; ++w) m = fmaxf(m, red[w]);
  float inv, scale;
  fp8::row_scales(m, inv, scale);
  for (int c = threadIdx.x; c < nchunk; c += THREADS) {  // a thread rewrites only the chunks it read
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(sx)[c], f);
    uint4 v;
    v.x = fp8::e4m3x2_to_elem2(fp8::e4m3x2(__fmul_rn(f[0], inv), __fmul_rn(f[1], inv)));
    v.y = fp8::e4m3x2_to_elem2(fp8::e4m3x2(__fmul_rn(f[2], inv), __fmul_rn(f[3], inv)));
    v.z = fp8::e4m3x2_to_elem2(fp8::e4m3x2(__fmul_rn(f[4], inv), __fmul_rn(f[5], inv)));
    v.w = fp8::e4m3x2_to_elem2(fp8::e4m3x2(__fmul_rn(f[6], inv), __fmul_rn(f[7], inv)));
    reinterpret_cast<uint4*>(sx)[c] = v;
  }
  __syncthreads();
  return scale;
}

template <int MODE>
__global__ void __launch_bounds__(THREADS, 2) fp8_gemv_kernel(const Params p, const srgpt_fp8 w8) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float red[32];
  bf16* sx = reinterpret_cast<bf16*>(smem_raw);
  const uint4* px = reinterpret_cast<const uint4*>(sx);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  trace_mark(p.trace, 0);
  const int pi = blockIdx.x * WARPS + warp;
  const bool active = pi < (p.N >> 1);
  int r0, r1;
  pair_rows<MODE>(p, pi, r0, r1);
  const int nvec = p.K >> 4;  // 16-byte code vectors per row
  const uint4* q0 = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(w8.q) + (size_t)r0 * p.K);
  const uint4* q1 = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(w8.q) + (size_t)r1 * p.K);
  // batch b: vectors v = 128 b + lane + 32 i, i = 0..3, of both rows (zero past the row's end)
  auto load = [&](int b, uint4 (&u0)[4], uint4 (&u1)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int v = b * 128 + lane + 32 * i;
      u0[i] = make_uint4(0, 0, 0, 0);
      u1[i] = make_uint4(0, 0, 0, 0);
      if (active && v < nvec) {
        u0[i] = ld_stream16(q0 + v);
        u1[i] = ld_stream16(q1 + v);
      }
    }
  };
  uint4 c0[4], c1[4];
  load(0, c0, c1);  // static weights: requested before the dependency wait, like the row scales and the norm weights
  const float sw0 = active ? __ldg(w8.scale + r0) : 0.f, sw1 = active ? __ldg(w8.scale + r1) : 0.f;
  uint4 nw_pre[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  const bool nw_pre_valid = (p.norm_weight != nullptr) && ((p.K >> 3) <= 2 * THREADS);
  if (nw_pre_valid) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int cc = threadIdx.x + k * THREADS;
      if (cc < (p.K >> 3)) nw_pre[k] = reinterpret_cast<const uint4*>(p.norm_weight)[cc];
    }
  }
  pdl_launch_dependents();
  pdl_wait();
  trace_mark(p.trace, 1);

  stage_x(p.x, p.norm_weight, p.eps, p.K, sx, red, nw_pre, nw_pre_valid);
  const float s_x = stage_quantize_e4m3(sx, p.K, red);

  float a0 = 0.f, a1 = 0.f;
  const int nb = (nvec + 127) >> 7;
  for (int b = 0; b < nb; ++b) {
    uint4 n0[4], n1[4];
    if (b + 1 < nb) load(b + 1, n0, n1);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int v = b * 128 + lane + 32 * i;
      if (v < nvec) {
        uint4 w0[2], w1[2];
        fp8::e4m3x16_to_elem(c0[i], w0[0], w0[1]);
        fp8::e4m3x16_to_elem(c1[i], w1[0], w1[1]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float xf[8];
          unpack8(px[2 * v + h], xf);
          a0 += dot8(w0[h], xf);
          a1 += dot8(w1[h], xf);
        }
      }
    }
    if (b + 1 < nb) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        c0[i] = n0[i];
        c1[i] = n1[i];
      }
    }
  }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  if (active && lane == 0) {
    float best;
    int besti;
    store_pair<MODE>(p, p.y, p.residual, nullptr, MODE == SRGPT_GEMV_QKV_ROPE ? *p.pos : 0, p.page_table, pi, r0, r1, a0 * (s_x * sw0),
                     a1 * (s_x * sw1), best, besti);
  }
  trace_mark(p.trace, 2);
}

// The best (value, index) of part_val / part_idx [0, n) over a CTA of 256 threads: `better` (the larger value, the lower index on ties)
// per thread, across the warp by shuffles, then across the 8 warps by thread 0, which alone holds the result.  (-INFINITY, 0x7fffffff)
// when n = 0 or every value is NaN.  A caller that runs it again first synchronises the CTA: it reuses its shared memory.
__device__ __forceinline__ void block_argmax(const float* part_val, const int* part_idx, int n, float& best, int& bi) {
  __shared__ float sv[8];
  __shared__ int si[8];
  best = -INFINITY;
  bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (better(part_val[i], part_idx[i], best, bi)) { best = part_val[i]; bi = part_idx[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < 8; ++w)
      if (better(sv[w], si[w], best, bi)) { best = sv[w]; bi = si[w]; }
}

__global__ void __launch_bounds__(256)
lm_head_finalize_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int nparts,
                        const bf16* __restrict__ embed_table, bf16* __restrict__ next_x, int K, long long* __restrict__ out_ids,
                        int* step, int* pos) {
  __shared__ int s_tok;
  pdl_launch_dependents();
  pdl_wait();
  float best;
  int bi;
  block_argmax(part_val, part_idx, nparts, best, bi);
  if (threadIdx.x == 0) {
    if (bi == 0x7fffffff) bi = 0;  // all-NaN logits: never feed the sentinel to the embedding gather of the next step
    s_tok = bi;
    out_ids[*step] = (long long)bi;
  }
  __syncthreads();
  const int tok = s_tok;
  if (embed_table != nullptr && next_x != nullptr) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)tok * K);
    for (int c = threadIdx.x; c < (K >> 3); c += blockDim.x) reinterpret_cast<uint4*>(next_x)[c] = src[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *step += 1;
    *pos += 1;
  }
}

// ---- multi-token decode GEMV (verify pass of prompt-lookup speculative decoding) ------------------------------------------------
// The warp / row-pair layout, chunk ownership (c = lane + 32 i), dot8 chains, warp_sum, stage_x (at 256 threads, so the RMSNorm
// reduction tree is the same), format decode and stores of decode_gemv_kernel, run for MT tokens against one stream of the weights:
// for every token the fp32 operations and their order are those of the one-token kernel, so each output is bit-identical to it.
// x is staged in shared memory for all tokens.  With RMSNorm (K = hidden size) the whole row is staged; without (o_proj, down_proj:
// K up to 14336 = 28 KB per token) x is staged in tiles of MT_TILE_CH chunks, so 8 tokens take 64 KB and 2 CTAs (16 warps) stay
// resident per SM.  The next 4-chunk batch of weights is loaded into registers while the current one is consumed.
constexpr int MT_MAX = SRGPT_SPEC_T_MAX;
constexpr int MT_TILE_CH = 512;  // x chunks (of 8 elements) per staged tile without RMSNorm; a multiple of the 128-chunk batch

struct MParams {
  Params p;
  int T;        // tokens (rows of x / y)
  int ldx, ldy;  // row strides of x and y (residual) in elements
  int tile_ch;  // chunks of x per staged tile
  // QKV_ROPE: row t is at position pos_rows[t] (NULL: *p.pos + t) and appends K / V through p.page_table + t * pt_stride (0: one sequence)
  const int* pos_rows;
  int pt_stride;
};

#define SRGPT_GEMV_MULTI_KERNEL decode_gemv_multi_kernel
#include "gemv_multi_kernel.inc"
#undef SRGPT_GEMV_MULTI_KERNEL

// the NF4 planes (srgpt_gemv_multi_nf4_bf16, the verify pass of a planes-only NF4 model): the same kernel under its own name
#define SRGPT_GEMV_MULTI_KERNEL nf4_gemv_multi_kernel
#include "gemv_multi_kernel.inc"
#undef SRGPT_GEMV_MULTI_KERNEL

// ---- the two ends of a verify pass -------------------------------------------------------------------------------------------
// History of the n-gram lookup: the prompt's ids (negative = a row that is not text: never matches), then the generated ids.
struct SpecHist {
  const int* prompt;
  int P;
  const long long* out;
  __device__ __forceinline__ int operator()(int i) const { return i < P ? prompt[i] : (int)out[i - P]; }
};

__global__ void __launch_bounds__(256)
spec_draft_kernel(const int* __restrict__ prompt_ids, const int* __restrict__ prompt_len, const long long* __restrict__ out_ids, const int* __restrict__ step,
                  const int* __restrict__ pos, int* __restrict__ pos_rows, int T, int ngram, const bf16* __restrict__ embed_table,
                  bf16* __restrict__ x, int H, int* __restrict__ draft_ids, int* __restrict__ state) {
  __shared__ int s_min[8];
  __shared__ int s_draft[MT_MAX];
  const int P = prompt_len != nullptr ? *prompt_len : 0;
  const SpecHist hist{prompt_ids, P, out_ids};
  const int s = *step, L = P + s;
  int start = -1;
  for (int n = min(ngram, L - 1); n >= 1 && start < 0; --n) {
    // the earliest window i < L - n equal to the last n ids (a window at i < L - n has a non-empty continuation)
    int best = 0x7fffffff;
    for (int i = threadIdx.x; i < L - n; i += blockDim.x) {
      bool eq = true;
      for (int j = 0; j < n && eq; ++j) {
        const int v = hist(i + j);
        eq = v >= 0 && v == hist(L - n + j);
      }
      if (eq) { best = i; break; }  // i grows along the loop: the thread's first hit is its earliest
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = best;
    __syncthreads();
    int m = 0x7fffffff;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = min(m, s_min[w]);
    __syncthreads();
    if (m != 0x7fffffff) start = m + n;
  }
  if (threadIdx.x == 0) {
    int nd = 0;
    s_draft[0] = hist(L - 1);
    for (int t = 1; t < T; ++t) {
      int v = -1;
      if (start >= 0 && nd == t - 1 && start + t - 1 < L) {
        v = hist(start + t - 1);
        if (v >= 0) ++nd; else v = -1;  // a draft ends at the first non-text row
      }
      s_draft[t] = v;
    }
    state[3] = nd;
  }
  __syncthreads();
  if (threadIdx.x < T) {
    draft_ids[threadIdx.x] = s_draft[threadIdx.x];
    pos_rows[threadIdx.x] = *pos + (int)threadIdx.x;
  }
  for (int t = 0; t < T; ++t) {  // embedding rows of the pass (a missing draft takes row 0: it is never accepted)
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)max(s_draft[t], 0) * H);
    uint4* dst = reinterpret_cast<uint4*>(x + (size_t)t * H);
    for (int c = threadIdx.x; c < (H >> 3); c += blockDim.x) dst[c] = src[c];
  }
}
// The arg max of every token reduces its partials exactly as lm_head_finalize_kernel does; then the acceptance rule.
__global__ void __launch_bounds__(256)
spec_accept_kernel(const float* __restrict__ ws, int nparts, int T, const int* __restrict__ draft_ids, long long* __restrict__ out_ids, int out_cap,
                   int* step, int* pos, int* state) {
  __shared__ int s_tok[MT_MAX];
  pdl_launch_dependents();
  pdl_wait();
  for (int t = 0; t < T; ++t) {
    const float* part_val = ws + (size_t)t * 2 * nparts;
    float best;
    int bi;
    block_argmax(part_val, reinterpret_cast<const int*>(part_val + nparts), nparts, best, bi);
    if (threadIdx.x == 0) s_tok[t] = bi == 0x7fffffff ? 0 : bi;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int a = 0;
    while (a < T - 1 && draft_ids[a + 1] == s_tok[a]) ++a;
    const int s0 = *step;
    for (int t = 0; t <= a; ++t)
      if (s0 + t < out_cap) out_ids[s0 + t] = (long long)s_tok[t];
    state[0] += 1;
    state[1] += state[3];
    state[2] += a;
    state[4] = s0;
    state[5] = a + 1;
    state[6] = s0 + a + 1;
    *step = s0 + a + 1;
    *pos += a + 1;
  }
}

// One decode step of B sequences (srgpt_llama_decode_rows_*): row b's token is its arg max, reduced from its partials exactly as
// lm_head_finalize_kernel does (lowest index on ties), or ids[b] when given (a draw).  It goes to out_ids[*step * B + b], row b of x
// becomes its embedding, pos_rows[b] advances; then *step.
__global__ void __launch_bounds__(256)
rows_advance_kernel(const float* __restrict__ ws, int nparts, const long long* __restrict__ ids, int B, const bf16* __restrict__ embed_table,
                    bf16* __restrict__ x, int H, long long* __restrict__ out_ids, int* step, int* pos_rows) {
  __shared__ int s_tok[MT_MAX];
  pdl_launch_dependents();
  pdl_wait();
  for (int b = 0; b < B; ++b) {
    if (ids != nullptr) {
      if (threadIdx.x == 0) s_tok[b] = (int)ids[b];
      continue;
    }
    const float* part_val = ws + (size_t)b * 2 * nparts;
    float best;
    int bi;
    block_argmax(part_val, reinterpret_cast<const int*>(part_val + nparts), nparts, best, bi);
    if (threadIdx.x == 0) s_tok[b] = bi == 0x7fffffff ? 0 : bi;
    __syncthreads();
  }
  __syncthreads();
  const int s = *step;
  if (threadIdx.x < B) {
    out_ids[(size_t)s * B + threadIdx.x] = (long long)s_tok[threadIdx.x];
    pos_rows[threadIdx.x] += 1;
  }
  for (int b = 0; b < B; ++b) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)s_tok[b] * H);
    uint4* dst = reinterpret_cast<uint4*>(x + (size_t)b * H);
    for (int c = threadIdx.x; c < (H >> 3); c += blockDim.x) dst[c] = src[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) *step = s + 1;
}

// output_logits: the accepted rows of the pass's logits [T, V] go to rows state[4] .. state[4] + state[5] - 1
__global__ void __launch_bounds__(256) spec_copy_logits_kernel(const float* __restrict__ rows, float* __restrict__ all, int V, const int* __restrict__ state,
                                                               int out_cap) {
  const int t = blockIdx.y;
  if (t >= state[5] || state[4] + t >= out_cap) return;
  const float* src = rows + (size_t)t * V;
  float* dst = all + (size_t)(state[4] + t) * V;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < V; j += gridDim.x * blockDim.x) dst[j] = src[j];
}

// ---- tensor-parallel helpers ------------------------------------------------------------------------
// vocabulary-parallel lm_head: this rank's best (bf16-rounded logit, GLOBAL row index) -> best[0] = value bits, best[1] = index
__global__ void __launch_bounds__(256)
lm_head_local_best_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int nparts, int index_base, int* __restrict__ best) {
  pdl_launch_dependents();
  pdl_wait();
  float bv;
  int bi;
  block_argmax(part_val, part_idx, nparts, bv, bi);
  if (threadIdx.x == 0) {
    best[0] = __float_as_int(bv);
    best[1] = (bi == 0x7fffffff) ? index_base : bi + index_base;
  }
}

// after the all-gather of every rank's (value, index): the global arg max (lowest index on ties, like torch.argmax), then the same
// bookkeeping as lm_head_finalize_kernel (token id, next embedding row, ++step, ++pos); identical on every rank
__global__ void __launch_bounds__(256)
tp_pick_token_kernel(const int* __restrict__ best_all, int world, const bf16* __restrict__ embed_table, bf16* __restrict__ next_x, int K,
                     long long* __restrict__ out_ids, int* step, int* pos) {
  __shared__ int s_tok;
  if (threadIdx.x == 0) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int r = 0; r < world; ++r) {
      const float v = __int_as_float(best_all[2 * r]);
      const int i = best_all[2 * r + 1];
      if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
    if (bi == 0x7fffffff) bi = 0;
    s_tok = bi;
    out_ids[*step] = (long long)bi;
  }
  __syncthreads();
  const int tok = s_tok;
  if (embed_table != nullptr && next_x != nullptr) {
    const uint4* src = reinterpret_cast<const uint4*>(embed_table + (size_t)tok * K);
    for (int c = threadIdx.x; c < (K >> 3); c += blockDim.x) reinterpret_cast<uint4*>(next_x)[c] = src[c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *step += 1;
    *pos += 1;
  }
}

// h = bf16(bf16(sum of the ranks' partial dot products) + h): the rounding points of `residual + o_proj(x)` (modeling_llama.py:668,682)
__global__ void __launch_bounds__(256) tp_residual_add_kernel(bf16* __restrict__ h, const float* __restrict__ partial, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) h[i] = f2e(bf16_round(partial[i]) + e2f(h[i]));
}

// ---- host side ------------------------------------------------------------------------------------
static int grid_for(int npairs) { return ceil_div(npairs, WARPS); }

static void pdl_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attr, int grid, int block, int smem, cudaStream_t st) {
  cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
}

template <int MODE, class Fmt>
static int launch(const Params& p, int npairs, cudaStream_t st) {
  const int smem = p.K * 2 + WARPS * ring_slots<Fmt>(p.K) * Fmt::SLOT;
  static int configured_smem = 0;
  if (smem > 48 * 1024 && smem > configured_smem) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(decode_gemv_kernel<MODE, Fmt>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  Params q = p;
  q.trace = trace_next_slot();
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, decode_gemv_kernel<MODE, Fmt>, q));
  return SRGPT_OK;
}

template <int MODE>
static int launch_fp8(const Params& p, const srgpt_fp8& w8, int npairs, cudaStream_t st) {
  const int smem = p.K * 2;
  static int configured_smem = 0;
  if (smem > 48 * 1024 && smem > configured_smem) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(fp8_gemv_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  Params q = p;
  q.trace = trace_next_slot();
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, fp8_gemv_kernel<MODE>, q, w8));
  return SRGPT_OK;
}

// the FP8 planes are not a decode_gemv_kernel format: their kernel is fp8_gemv_kernel, which takes them beside Params
struct Fp8 {};

template <int MODE, class Fmt>
static int launch_format(const Params& p, const srgpt_fp8* w8, int npairs, cudaStream_t st) {
  if constexpr (std::is_same<Fmt, Fp8>::value)
    return launch_fp8<MODE>(p, *w8, npairs, st);
  else
    return launch<MODE, Fmt>(p, npairs, st);
}

}  // namespace gemv
}  // namespace srgpt

using namespace srgpt;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a packed matrix the kernel can stream: every array present, vector-aligned planes, K a whole number of batches
static bool packed_ok(const srgpt_packed12* P, int K) {
  return P != nullptr && P->sm && P->ex && P->base && P->row_ptr && P->exc && aligned16(P->sm) && aligned16(P->ex) && (K % pack12::BATCH) == 0;
}

#ifdef SRGPT_ELEM_F16
// the fp16 build exports the packed entry points and refuses them
static int packed_needs_bf16(const char* fn) {
  set_last_error("%s: the 12-bit packing is defined for bfloat16 weights only", fn);
  return SRGPT_ERR_UNSUPPORTED;
}
#endif

// the fields every decode GEMV entry point sets; the weights and the fields of a mode are the caller's
static void set_io(gemv::Params& p, const void* x, void* y, int N, int K, const void* norm_weight, float eps, const void* residual) {
  p.x = reinterpret_cast<const bf16*>(x);
  p.y = reinterpret_cast<bf16*>(y);
  p.N = N;
  p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.residual = reinterpret_cast<const bf16*>(residual);
}

// QKV + RoPE + KV append
static void set_rope(gemv::Params& p, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos,
                     void* kv_pages, const int* page_table, int page_size) {
  p.n_heads = n_heads;
  p.n_kv_heads = n_kv_heads;
  p.hd = head_dim;
  p.cos_tab = reinterpret_cast<const bf16*>(cos_tab);
  p.sin_tab = reinterpret_cast<const bf16*>(sin_tab);
  p.pos = pos;
  p.kv_pages = reinterpret_cast<bf16*>(kv_pages);
  p.page_table = page_table;
  p.page_size = page_size;
}

// checks and mode dispatch of srgpt_gemv_bf16, srgpt_gemv_packed_bf16, srgpt_gemv_nf4_bf16 and srgpt_gemv_fp8_bf16; p's weights are set by
// the caller
template <class Fmt>
static int gemv_modes(gemv::Params& p, const void* x, void* y, int N, int K, const void* norm_weight, float eps, const void* residual, int mode,
                      int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages,
                      const int* page_table, int page_size, void* stream, const srgpt_fp8* w8 = nullptr) {
  SRGPT_CHECK_ARG(x && y && N > 0 && K > 0);
  SRGPT_CHECK_ARG((N % 2) == 0 && (K % 8) == 0);
  SRGPT_CHECK_ARG(K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && (reinterpret_cast<uintptr_t>(y) & 3) == 0);
  SRGPT_CHECK_ARG(norm_weight == nullptr || aligned16(norm_weight));
  SRGPT_CHECK_ARG(mode >= SRGPT_GEMV_PLAIN && mode <= SRGPT_GEMV_QKV_ROPE);
  SRGPT_CHECK_ARG(x != y);  // x is read by late CTAs while early ones already write y
  set_io(p, x, y, N, K, norm_weight, eps, residual);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (mode) {
    case SRGPT_GEMV_PLAIN:
      return gemv::launch_format<SRGPT_GEMV_PLAIN, Fmt>(p, w8, N / 2, st);
    case SRGPT_GEMV_SWIGLU:
      SRGPT_CHECK_ARG(residual == nullptr);
      return gemv::launch_format<SRGPT_GEMV_SWIGLU, Fmt>(p, w8, N / 2, st);
    case SRGPT_GEMV_QKV_ROPE:
      SRGPT_CHECK_ARG(residual == nullptr && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0);
      SRGPT_CHECK_ARG(N == (n_heads + 2 * n_kv_heads) * head_dim);
      SRGPT_CHECK_ARG(cos_tab && sin_tab && pos && kv_pages && page_table && page_size > 0);
      set_rope(p, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages, page_table, page_size);
      return gemv::launch_format<SRGPT_GEMV_QKV_ROPE, Fmt>(p, w8, N / 2, st);
  }
  return SRGPT_ERR_INVALID;
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_nf4_bf16(const void* x, const srgpt_nf4* nf4, void* y, int N, int K, const void* norm_weight,
                                                                          float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim,
                                                                          const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages,
                                                                          const int* page_table, int page_size, void* stream) {
  SRGPT_CHECK_ARG(nf4 && nf4->q && nf4->scale && aligned16(nf4->q) && (reinterpret_cast<uintptr_t>(nf4->scale) & 3) == 0);
  SRGPT_CHECK_ARG(K > 0 && (K % nf4::BLOCK) == 0);
  SRGPT_CHECK_ARG((K % nf4::BATCH) == 0);
  SRGPT_CHECK_ARG(K * 2 + gemv::WARPS * 4 * gemv::Nf4::SLOT <= 227 * 1024);  // K <= 95 x 1024, the range this entry has always accepted
  gemv::Params p = {};
  p.nf = *nf4;
  return gemv_modes<gemv::Nf4>(p, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                               page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_fp8_bf16(const void* x, const srgpt_fp8* w, void* y, int N, int K, const void* norm_weight,
                                                                          float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim,
                                                                          const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages,
                                                                          const int* page_table, int page_size, void* stream) {
  SRGPT_CHECK_ARG(w && w->q && w->scale && aligned16(w->q) && (reinterpret_cast<uintptr_t>(w->scale) & 3) == 0);
  SRGPT_CHECK_ARG(K > 0 && (K % 16) == 0);
  gemv::Params p = {};
  return gemv_modes<gemv::Fp8>(p, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                               page_table, page_size, stream, w);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_bf16(const void* x, const void* W, int ldw, void* y, int N, int K, const void* norm_weight, float eps,
                               const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                               const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size,
                               void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::Params p = {};
  p.W = reinterpret_cast<const bf16*>(W);
  p.ldw = ldw;
  return gemv_modes<gemv::Bf16>(p, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                                page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_packed_bf16(const void* x, const srgpt_packed12* packed, void* y, int N, int K,
                                                                               const void* norm_weight, float eps, const void* residual, int mode, int n_heads,
                                                                               int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                                                                               const int* pos, void* kv_pages, const int* page_table, int page_size,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  return packed_needs_bf16("srgpt_gemv_packed_bf16");
#else
  gemv::Params p = {};
  p.pk = *packed;
  return gemv_modes<gemv::Packed12>(p, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                                    page_table, page_size, stream);
#endif
}

// Tensor-parallel variants of the decode GEMV (SURVEY.md §8e "optional TP", BASELINE config c5): a rank owns n_heads q heads and
// n_kv_heads kv heads of the fused qkv projection (column parallel; K/V rows land in the FULL-layout cache at kv_head_off), and a K
// slice of o_proj / down_proj (row parallel): PLAIN mode with partial_f32 != NULL writes the un-rounded fp32 partial sums that the
// ranks then all-reduce.  Everything else is srgpt_gemv_bf16.
extern "C" __attribute__((visibility("default"))) int srgpt_gemv_tp_bf16(const void* x, const void* W, int ldw, void* y, int N, int K, const void* norm_weight, float eps,
                                                                         int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                                                                         const int* pos, void* kv_pages, const int* page_table, int page_size, int kv_heads_total,
                                                                         int kv_head_off, float* partial_f32, void* stream) {
  SRGPT_CHECK_ARG(x && W && N > 0 && K > 0 && (y != nullptr || partial_f32 != nullptr));
  SRGPT_CHECK_ARG((N % 2) == 0 && (K % 8) == 0 && (ldw % 8) == 0 && ldw >= K && K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && aligned16(W) && (norm_weight == nullptr || aligned16(norm_weight)));
  SRGPT_CHECK_ARG(mode == SRGPT_GEMV_PLAIN || mode == SRGPT_GEMV_QKV_ROPE);
  gemv::Params p = {};
  p.W = reinterpret_cast<const bf16*>(W);
  p.ldw = ldw;
  set_io(p, x, y, N, K, norm_weight, eps, nullptr);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == SRGPT_GEMV_PLAIN) {
    SRGPT_CHECK_ARG(partial_f32 != nullptr && (reinterpret_cast<uintptr_t>(partial_f32) & 7) == 0);
    p.y_f32 = partial_f32;
    return gemv::launch<SRGPT_GEMV_PLAIN, gemv::Bf16>(p, N / 2, st);
  }
  SRGPT_CHECK_ARG(y != nullptr && (reinterpret_cast<uintptr_t>(y) & 3) == 0 && x != y);
  SRGPT_CHECK_ARG(n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0 && N == (n_heads + 2 * n_kv_heads) * head_dim);
  SRGPT_CHECK_ARG(cos_tab && sin_tab && pos && kv_pages && page_table && page_size > 0);
  SRGPT_CHECK_ARG(kv_heads_total >= n_kv_heads && kv_head_off >= 0 && kv_head_off + n_kv_heads <= kv_heads_total);
  set_rope(p, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages, page_table, page_size);
  p.kv_heads_total = kv_heads_total;
  p.kv_head_off = kv_head_off;
  return gemv::launch<SRGPT_GEMV_QKV_ROPE, gemv::Bf16>(p, N / 2, st);
}

extern "C" __attribute__((visibility("default"))) int srgpt_tp_residual_add_bf16(void* h, const float* partial, int n, void* stream) {
  SRGPT_CHECK_ARG(h && partial && n > 0);
  gemv::tp_residual_add_kernel<<<ceil_div(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<bf16*>(h), partial, n);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// Vocabulary-parallel lm_head of one rank: rows [index_base, index_base + V_local) of the table.  best = device int[2]
// {bf16-rounded best logit (float bits), its GLOBAL row index}; all-gather the pairs, then srgpt_tp_pick_token.
extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_local_best_bf16(const void* x, const void* W_local, int ldw, int V_local, int K, const void* norm_weight,
                                                                                    float eps, void* workspace, int index_base, int* best, void* stream) {
  SRGPT_CHECK_ARG(x && W_local && workspace && best && V_local > 0 && K > 0 && index_base >= 0);
  SRGPT_CHECK_ARG((K % 8) == 0 && (ldw % 8) == 0 && ldw >= K && K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && aligned16(W_local) && (norm_weight == nullptr || aligned16(norm_weight)));
  const int npairs = (V_local + 1) / 2;
  const int g = gemv::grid_for(npairs);
  gemv::Params p = {};
  p.W = reinterpret_cast<const bf16*>(W_local);
  p.ldw = ldw;
  set_io(p, x, nullptr, V_local, K, norm_weight, eps, nullptr);
  p.part_val = reinterpret_cast<float*>(workspace);
  p.part_idx = reinterpret_cast<int*>(p.part_val + g);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = gemv::launch<gemv::MODE_LM, gemv::Bf16>(p, npairs, st);
  if (rc != SRGPT_OK) return rc;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  gemv::pdl_config(cfg, attr, 1, 256, 0, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemv::lm_head_local_best_kernel, (const float*)p.part_val, (const int*)p.part_idx, g, index_base, best));
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_tp_pick_token(const int* best_all, int world, const void* embed_table, void* next_x, int K, long long* out_ids,
                                                                          int* step, int* pos, void* stream) {
  SRGPT_CHECK_ARG(best_all && world > 0 && out_ids && step && pos);
  SRGPT_CHECK_ARG((embed_table == nullptr) == (next_x == nullptr));
  SRGPT_CHECK_ARG(embed_table == nullptr || ((K % 8) == 0 && aligned16(embed_table) && aligned16(next_x)));
  gemv::tp_pick_token_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(best_all, world, reinterpret_cast<const bf16*>(embed_table),
                                                                                  reinterpret_cast<bf16*>(next_x), K, out_ids, step, pos);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) long long srgpt_lm_head_workspace(int V) {
  if (V <= 0) return -1;
  const int g = gemv::grid_for((V + 1) / 2);
  return (long long)g * (long long)(sizeof(float) + sizeof(int));
}

// srgpt_lm_head_argmax_bf16 and its packed form; p's weights are set by the caller
template <class Fmt>
static int lm_head_argmax(gemv::Params& p, const void* x, int V, int K, const void* norm_weight, float eps, float* logits_out, void* workspace,
                          const void* embed_table, void* next_x, long long* out_ids, int* step, int* pos, void* stream) {
  SRGPT_CHECK_ARG(x && workspace && out_ids && step && pos && V > 0 && K > 0);
  SRGPT_CHECK_ARG((K % 8) == 0 && K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && (norm_weight == nullptr || aligned16(norm_weight)));
  SRGPT_CHECK_ARG((embed_table == nullptr) == (next_x == nullptr));
  SRGPT_CHECK_ARG(embed_table == nullptr || (aligned16(embed_table) && aligned16(next_x)));
  const int npairs = (V + 1) / 2;
  const int g = gemv::grid_for(npairs);
  set_io(p, x, nullptr, V, K, norm_weight, eps, nullptr);
  p.logits_out = logits_out;
  p.part_val = reinterpret_cast<float*>(workspace);
  p.part_idx = reinterpret_cast<int*>(p.part_val + g);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = gemv::launch<gemv::MODE_LM, Fmt>(p, npairs, st);
  if (rc != SRGPT_OK) return rc;
  // finalize: also a programmatic dependent (its launch latency hides behind the lm_head kernel)
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  gemv::pdl_config(cfg, attr, 1, 256, 0, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemv::lm_head_finalize_kernel, (const float*)p.part_val, (const int*)p.part_idx, g,
                                      reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(next_x), K, out_ids, step, pos));
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_argmax_bf16(const void* x, const void* W, int ldw, int V, int K, const void* norm_weight, float eps,
                                         float* logits_out, void* workspace, const void* embed_table, void* next_x,
                                         long long* out_ids, int* step, int* pos, void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::Params p = {};
  p.W = reinterpret_cast<const bf16*>(W);
  p.ldw = ldw;
  return lm_head_argmax<gemv::Bf16>(p, x, V, K, norm_weight, eps, logits_out, workspace, embed_table, next_x, out_ids, step, pos, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_argmax_packed_bf16(const void* x, const srgpt_packed12* packed, int V, int K,
                                                                                         const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                                         const void* embed_table, void* next_x, long long* out_ids, int* step,
                                                                                         int* pos, void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  return packed_needs_bf16("srgpt_lm_head_argmax_packed_bf16");
#else
  gemv::Params p = {};
  p.pk = *packed;
  return lm_head_argmax<gemv::Packed12>(p, x, V, K, norm_weight, eps, logits_out, workspace, embed_table, next_x, out_ids, step, pos, stream);
#endif
}

// ---- prompt-lookup speculative decoding: multi-token GEMV, lm_head, draft and accept ------------------------------------------
namespace srgpt {
namespace gemv {

template <int MODE, class Fmt>
static auto multi_kernel() {
  if constexpr (std::is_same<Fmt, Nf4>::value)
    return &nf4_gemv_multi_kernel<MODE, Nf4>;
  else
    return &decode_gemv_multi_kernel<MODE, Fmt>;
}

template <int MODE, class Fmt>
static int launch_multi(MParams& mp, int npairs, cudaStream_t st) {
  const int smem = mp.T * mp.tile_ch * 16;
  static int configured_smem = 0;
  if (smem > configured_smem) {  // the opt-in counts static shared memory too, so it is set for every size, not only above 48 KB
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(multi_kernel<MODE, Fmt>(), cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, multi_kernel<MODE, Fmt>(), mp));
  return SRGPT_OK;
}

// x staged per token: the whole row with RMSNorm, tiles of MT_TILE_CH chunks without
static int multi_tile(int K, bool norm) { return norm ? (K >> 3) : ((K >> 3) < MT_TILE_CH ? (K >> 3) : MT_TILE_CH); }

}  // namespace gemv
}  // namespace srgpt

template <class Fmt>
static int gemv_multi_modes(gemv::MParams& mp, const void* x, int ldx, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                            const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                            const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream, const int* pos_rows = nullptr,
                            int pt_stride = 0) {
  SRGPT_CHECK_ARG(x && y && N > 0 && K > 0 && T >= 1 && T <= gemv::MT_MAX);
  SRGPT_CHECK_ARG((N % 2) == 0 && (K % 8) == 0 && (ldx % 8) == 0 && ldx >= K && (ldy % 2) == 0);
  SRGPT_CHECK_ARG(aligned16(x) && (reinterpret_cast<uintptr_t>(y) & 3) == 0);
  SRGPT_CHECK_ARG(norm_weight == nullptr || aligned16(norm_weight));
  SRGPT_CHECK_ARG(mode >= SRGPT_GEMV_PLAIN && mode <= SRGPT_GEMV_QKV_ROPE);
  SRGPT_CHECK_ARG(x != y);
  const int tile = gemv::multi_tile(K, norm_weight != nullptr);
  SRGPT_CHECK_ARG(T * tile * 16 <= 200 * 1024);
  set_io(mp.p, x, y, N, K, norm_weight, eps, residual);
  mp.T = T; mp.ldx = ldx; mp.ldy = ldy; mp.tile_ch = tile;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (mode) {
    case SRGPT_GEMV_PLAIN:
      SRGPT_CHECK_ARG(ldy >= N);
      return gemv::launch_multi<SRGPT_GEMV_PLAIN, Fmt>(mp, N / 2, st);
    case SRGPT_GEMV_SWIGLU:
      SRGPT_CHECK_ARG(residual == nullptr && ldy >= N / 2);
      return gemv::launch_multi<SRGPT_GEMV_SWIGLU, Fmt>(mp, N / 2, st);
    case SRGPT_GEMV_QKV_ROPE:
      SRGPT_CHECK_ARG(residual == nullptr && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0);
      SRGPT_CHECK_ARG(N == (n_heads + 2 * n_kv_heads) * head_dim && ldy >= n_heads * head_dim);
      SRGPT_CHECK_ARG(cos_tab && sin_tab && (pos || pos_rows) && kv_pages && page_table && page_size > 0 && pt_stride >= 0);
      set_rope(mp.p, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages, page_table, page_size);
      mp.pos_rows = pos_rows;
      mp.pt_stride = pt_stride;
      return gemv::launch_multi<SRGPT_GEMV_QKV_ROPE, Fmt>(mp, N / 2, st);
  }
  return SRGPT_ERR_INVALID;
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_multi_bf16(const void* x, int ldx, const void* W, int ldw, void* y, int ldy, int T, int N, int K,
                                                                            const void* norm_weight, float eps, const void* residual, int mode, int n_heads,
                                                                            int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos,
                                                                            void* kv_pages, const int* page_table, int page_size, void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::MParams mp = {};
  mp.p.W = reinterpret_cast<const bf16*>(W);
  mp.p.ldw = ldw;
  return gemv_multi_modes<gemv::Bf16>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                      kv_pages, page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, void* y, int ldy, int T,
                                                                                   int N, int K, const void* norm_weight, float eps, const void* residual,
                                                                                   int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                                                                                   const void* sin_tab, const int* pos, void* kv_pages, const int* page_table,
                                                                                   int page_size, void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  return packed_needs_bf16("srgpt_gemv_multi_packed_bf16");
#else
  gemv::MParams mp = {};
  mp.p.pk = *packed;
  return gemv_multi_modes<gemv::Packed12>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab,
                                          pos, kv_pages, page_table, page_size, stream);
#endif
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_multi_nf4_bf16(const void* x, int ldx, const srgpt_nf4* nf4, void* y, int ldy, int T, int N,
                                                                                int K, const void* norm_weight, float eps, const void* residual, int mode,
                                                                                int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                                                                                const void* sin_tab, const int* pos, void* kv_pages, const int* page_table,
                                                                                int page_size, void* stream) {
  SRGPT_CHECK_ARG(nf4 && nf4->q && nf4->scale && aligned16(nf4->q) && (reinterpret_cast<uintptr_t>(nf4->scale) & 3) == 0);
  SRGPT_CHECK_ARG(K > 0 && (K % nf4::BATCH) == 0);
  gemv::MParams mp = {};
  mp.p.nf = *nf4;
  return gemv_multi_modes<gemv::Nf4>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                     kv_pages, page_table, page_size, stream);
}

// T rows of T different sequences in QKV_ROPE mode: row t rotates at pos_rows[t] and appends its K / V through page_tables + t * pt_stride.
// The arithmetic of every row is that of the one-token srgpt_gemv_*_bf16 call at that position and page table.
extern "C" __attribute__((visibility("default"))) int srgpt_gemv_rows_bf16(const void* x, int ldx, const void* W, int ldw, void* y, int ldy, int T, int N,
                                                                           int K, const void* norm_weight, float eps, int n_heads, int n_kv_heads,
                                                                           int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows,
                                                                           void* kv_pages, const int* page_tables, int pt_stride, int page_size,
                                                                           void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K && pos_rows != nullptr);
  gemv::MParams mp = {};
  mp.p.W = reinterpret_cast<const bf16*>(W);
  mp.p.ldw = ldw;
  return gemv_multi_modes<gemv::Bf16>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads, n_kv_heads, head_dim,
                                      cos_tab, sin_tab, nullptr, kv_pages, page_tables, page_size, stream, pos_rows, pt_stride);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_rows_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, void* y, int ldy,
                                                                                  int T, int N, int K, const void* norm_weight, float eps, int n_heads,
                                                                                  int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                                                                                  const int* pos_rows, void* kv_pages, const int* page_tables,
                                                                                  int pt_stride, int page_size, void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K) && pos_rows != nullptr);
#ifdef SRGPT_ELEM_F16
  return packed_needs_bf16("srgpt_gemv_rows_packed_bf16");
#else
  gemv::MParams mp = {};
  mp.p.pk = *packed;
  return gemv_multi_modes<gemv::Packed12>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads, n_kv_heads, head_dim,
                                          cos_tab, sin_tab, nullptr, kv_pages, page_tables, page_size, stream, pos_rows, pt_stride);
#endif
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_rows_nf4_bf16(const void* x, int ldx, const srgpt_nf4* nf4, void* y, int ldy, int T, int N,
                                                                               int K, const void* norm_weight, float eps, int n_heads, int n_kv_heads,
                                                                               int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows,
                                                                               void* kv_pages, const int* page_tables, int pt_stride, int page_size,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(nf4 && nf4->q && nf4->scale && aligned16(nf4->q) && (reinterpret_cast<uintptr_t>(nf4->scale) & 3) == 0 && pos_rows != nullptr);
  SRGPT_CHECK_ARG(K > 0 && (K % nf4::BATCH) == 0);
  gemv::MParams mp = {};
  mp.p.nf = *nf4;
  return gemv_multi_modes<gemv::Nf4>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads, n_kv_heads, head_dim,
                                     cos_tab, sin_tab, nullptr, kv_pages, page_tables, page_size, stream, pos_rows, pt_stride);
}

template <class Fmt>
static int lm_head_multi(gemv::MParams& mp, const void* x, int ldx, int T, int V, int K, const void* norm_weight, float eps, float* logits_out,
                         void* workspace, void* stream) {
  SRGPT_CHECK_ARG(x && workspace && V > 0 && K > 0 && T >= 1 && T <= gemv::MT_MAX);
  SRGPT_CHECK_ARG((K % 8) == 0 && (ldx % 8) == 0 && ldx >= K && aligned16(x) && (norm_weight == nullptr || aligned16(norm_weight)));
  const int tile = gemv::multi_tile(K, norm_weight != nullptr);
  SRGPT_CHECK_ARG(T * tile * 16 <= 200 * 1024);
  set_io(mp.p, x, nullptr, V, K, norm_weight, eps, nullptr);
  mp.p.logits_out = logits_out;
  mp.p.part_val = reinterpret_cast<float*>(workspace);
  mp.T = T; mp.ldx = ldx; mp.ldy = 0; mp.tile_ch = tile;
  return gemv::launch_multi<gemv::MODE_LM, Fmt>(mp, (V + 1) / 2, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_multi_bf16(const void* x, int ldx, const void* W, int ldw, int T, int V, int K,
                                                                               const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::MParams mp = {};
  mp.p.W = reinterpret_cast<const bf16*>(W);
  mp.p.ldw = ldw;
  return lm_head_multi<gemv::Bf16>(mp, x, ldx, T, V, K, norm_weight, eps, logits_out, workspace, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, int T, int V, int K,
                                                                                      const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                                      void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  return packed_needs_bf16("srgpt_lm_head_multi_packed_bf16");
#else
  gemv::MParams mp = {};
  mp.p.pk = *packed;
  return lm_head_multi<gemv::Packed12>(mp, x, ldx, T, V, K, norm_weight, eps, logits_out, workspace, stream);
#endif
}

extern "C" __attribute__((visibility("default"))) int srgpt_spec_draft(const int* prompt_ids, const int* prompt_len, const long long* out_ids, const int* step, const int* pos,
                                                                       int* pos_rows, int T, int ngram, const void* embed_table, void* x, int H, int* draft_ids,
                                                                       int* state, void* stream) {
  SRGPT_CHECK_ARG(out_ids && step && pos && pos_rows && embed_table && x && draft_ids && state && ((prompt_ids == nullptr) == (prompt_len == nullptr)));
  SRGPT_CHECK_ARG(T >= 1 && T <= gemv::MT_MAX && ngram >= 1 && H > 0 && (H % 8) == 0 && aligned16(embed_table) && aligned16(x));
  gemv::spec_draft_kernel<<<1, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(prompt_ids, prompt_len, out_ids, step, pos, pos_rows, T, ngram,
                                                                                 reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(x), H,
                                                                                 draft_ids, state);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_spec_accept(const void* workspace, int V, int T, const int* draft_ids, long long* out_ids, int out_cap,
                                                                        int* step, int* pos, int* state, const float* logits_rows, float* logits_all,
                                                                        void* stream) {
  SRGPT_CHECK_ARG(workspace && draft_ids && out_ids && step && pos && state && V > 0 && T >= 1 && T <= gemv::MT_MAX && out_cap > 0);
  SRGPT_CHECK_ARG(logits_all == nullptr || logits_rows != nullptr);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  gemv::pdl_config(cfg, attr, 1, 256, 0, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemv::spec_accept_kernel, reinterpret_cast<const float*>(workspace), gemv::grid_for((V + 1) / 2), T, draft_ids,
                                      out_ids, out_cap, step, pos, state));
  if (logits_all != nullptr) {
    gemv::spec_copy_logits_kernel<<<dim3(ceil_div(V, 256 * 8), T), 256, 0, st>>>(logits_rows, logits_all, V, state, out_cap);
    SRGPT_CHECK_LAUNCH();
  }
  return SRGPT_OK;
}

// The end of a decode step of B sequences: each row's arg max from its lm_head_multi partials in workspace (ids == NULL), or the drawn
// ids [B]; then out_ids[*step * B + b], x row b = its embedding, ++pos_rows[b], ++*step.
extern "C" __attribute__((visibility("default"))) int srgpt_rows_advance(const void* workspace, int V, const long long* ids, int B, const void* embed_table,
                                                                         void* x, int H, long long* out_ids, int* step, int* pos_rows, void* stream) {
  SRGPT_CHECK_ARG(B >= 1 && B <= gemv::MT_MAX && V > 0 && H > 0 && (H % 8) == 0);
  SRGPT_CHECK_ARG((workspace || ids) && embed_table && x && out_ids && step && pos_rows && aligned16(embed_table) && aligned16(x));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  gemv::pdl_config(cfg, attr, 1, 256, 0, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemv::rows_advance_kernel, reinterpret_cast<const float*>(workspace), gemv::grid_for((V + 1) / 2), ids, B,
                                      reinterpret_cast<const bf16*>(embed_table), reinterpret_cast<bf16*>(x), H, out_ids, step, pos_rows));
  return SRGPT_OK;
}
