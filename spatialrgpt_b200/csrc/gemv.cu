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
// The packed variant (PACKED = true) streams the 12-bit lossless packing of pack12.cuh: per batch of 4 chunks a lane loads
// 3 x 16 bytes per row instead of 4, rebuilds the bf16 pairs in registers (decode_chunk), ORs in the row's few exception
// exponents, and then runs the very same dot8 / warp_sum / epilogue, so its results are bit-identical.  Its weight stream runs through a
// per-warp ring of cp.async slots in shared memory (ring_depth), so a warp keeps several batches in flight without spending registers.
#include <stdlib.h>

#include "common.cuh"
#include "nf4.cuh"
#include "pack12.cuh"
#include "srgpt_b200.h"

namespace srgpt {
namespace gemv {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int SPRE_MAX = 2;                       // up to 2 x 4 chunks per row per lane in shared memory
constexpr int SPRE_WARP_BYTES = 2 * 4 * 32 * 16;  // per batch: 2 rows x 4 chunks x 32 lanes x 16 B = 4 KB
constexpr int SPRE_WARP_BYTES12 = 2 * 3 * 32 * 16;  // packed: 2 rows x 3 vectors x 32 lanes x 16 B = 3 KB
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
  int ring;                   // packed: 1 = the spre slots are a ring that every later batch streams through, 0 = later batches load into
                              // registers.  It sits in the padding before the next pointer, so no other member (nor MParams) moves.
  // LM
  float* logits_out;
  float* part_val;
  int* part_idx;
  unsigned long long* trace;  // optional timeline record (srgpt_trace_begin)
  int spre;                   // number of extra 4-chunk batches per row staged in shared memory before the wait (0..SPRE_MAX)
  int l2pf;                   // 1: the rest of the warp's two rows is requested into L2 (bulk prefetch) before the dependency wait
  // tensor parallelism (srgpt_gemv_tp_bf16): this rank's slice of the heads / of the reduction dimension
  int kv_heads_total;         // KV-cache row = kv_heads_total * hd elements (0: n_kv_heads); the rank writes heads [kv_head_off, +n_kv_heads)
  int kv_head_off;
  float* y_f32;               // PLAIN mode: un-rounded fp32 partial dot products go here instead of bf16 y (+ residual)
  srgpt_packed12 pk;          // the packed kernel's weights (W is unused there)
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

// Batch b of both rows into one 3 KB slot of the warp's shared memory by cp.async (row r0: sm 01, sm 23, ex at +0 / 512 / 1024, row r1 at
// +1536 ...).  slot_lane = the slot + 16 * lane: every lane later reads back exactly the 16-byte vectors it requested, so no barrier is needed.
__device__ __forceinline__ void cp_async_batch12(const uint8_t* slot_lane, const uint4* sm0, const uint4* ex0, int drow_ex, int b) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(slot_lane);
  const uint4 *s = sm0 + b * 64, *e = ex0 + b * 32;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(s) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 512), "l"(s + 32) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 1024), "l"(e) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 1536), "l"(s + 2 * drow_ex) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 2048), "l"(s + 2 * drow_ex + 32) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 2560), "l"(e + drow_ex) : "memory");
}

__device__ __forceinline__ void ld_slot12(const uint8_t* slot_lane, Raw12& t0, Raw12& t1) {
  const uint4* s = reinterpret_cast<const uint4*>(slot_lane);
  t0 = {s[0], s[32], s[64]};
  t1 = {s[96], s[128], s[160]};
}

// cp.async.wait_group takes an immediate: wait until at most n (0..RING_MAX - 1) of this thread's newest commit groups are pending
constexpr int RING_MAX = 4;
__device__ __forceinline__ void cp_async_wait_pending(int n) {
  switch (n) {
    case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
  }
}

struct Rows12 {
  uint32_t bp0, bp1;  // base - 1 of the two rows
  int exc0, exc1;     // this lane's entry of each row's exception list
  int n0, n1;         // list lengths
  int j0, j1;         // next entry to apply
};

__device__ __forceinline__ void consume12(const Raw12& q0, const Raw12& q1, Rows12& rs, int b, int lane, const uint4* px, float& a0, float& a1) {
  uint4 w0[4], w1[4];
  decode_batch(q0, rs.bp0, w0);
  decode_batch(q1, rs.bp1, w1);
  patch_batch(w0, rs.exc0, rs.n0, rs.j0, b, lane);
  patch_batch(w1, rs.exc1, rs.n1, rs.j1, b, lane);
  const int c = b * 128 + lane;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float xf[8];
    unpack8(px[c + 32 * i], xf);
    a0 += dot8(w0[i], xf);
    a1 += dot8(w1[i], xf);
  }
}

// PRE = number of 4-chunk batches (per row) requested BEFORE the dependency wait: 1 -> 8 loads per lane (3 CTAs/SM),
// 2 -> 16 loads (2 CTAs/SM), 4 -> 32 loads = a whole K=4096 row pair per warp (1 CTA/SM).  The small matrices of a
// layer (qkv 50 MB, o_proj 33 MB) run behind a kernel that leaves HBM idle (decode attention / the previous tail), so
// the more of their weights is in flight before the dependency resolves, the less of them is exposed afterwards.
// PACKED: the weights are p.pk (12-bit packing, K % 1024 == 0, PRE == 1); everything but the weight stream is shared.
template <int MODE>
__device__ __forceinline__ void epilogue(const Params& p, bool active, int pi, int r0, int r1, int warp, int lane, float a0, float a1, float* sv,
                                         int* si);

template <int MODE, int PRE, bool PACKED>
__global__ void __launch_bounds__(THREADS, PRE == 1 ? 3 : (PRE == 2 ? 2 : 1)) decode_gemv_kernel(const Params p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float red[32];
  __shared__ float sv[WARPS];
  __shared__ int si[WARPS];
  bf16* sx = reinterpret_cast<bf16*>(smem_raw);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  trace_mark(p.trace, 0);
  const int npairs = (MODE == MODE_LM) ? ((p.N + 1) >> 1) : (p.N >> 1);
  const int pi = blockIdx.x * WARPS + warp;
  const bool active = pi < npairs;
  int r0 = 0, r1 = 0;
  if (active) pair_rows<MODE>(p, pi, r0, r1);
  const uint4* p0 = reinterpret_cast<const uint4*>(p.W + (size_t)r0 * p.ldw);
  const uint4* p1 = reinterpret_cast<const uint4*>(p.W + (size_t)r1 * p.ldw);
  const uint4* px = reinterpret_cast<const uint4*>(sx);
  const int nchunk = p.K >> 3;
  const int nchunk_all = nchunk;

  // ---- first 8*PRE loads per lane: weights do not depend on the previous kernel
  constexpr int NPRE = 4 * PRE;
  uint4 u0[NPRE], u1[NPRE];
  int c = lane;
  const bool first_full = !PACKED && active && (c + 32 * (NPRE - 1) < nchunk);
  if (first_full) {
#pragma unroll
    for (int i = 0; i < NPRE; ++i) {
      u0[i] = ld_stream16(p0 + c + 32 * i);
      u1[i] = ld_stream16(p1 + c + 32 * i);
    }
  }
  // ---- a second, register-free prefetch level: the next p.spre batches of both rows go to shared memory with
  //      cp.async (every lane later reads back exactly the 16-byte slots it filled, so no barrier is needed).
  //      Occupancy stays at 3 CTAs/SM, unlike the deeper register prefetch (PRE = 2/4) that was measured and rejected.
  uint8_t* spre_base = smem_raw + (size_t)p.K * 2 + (size_t)warp * ((size_t)p.spre * (PACKED ? SPRE_WARP_BYTES12 : SPRE_WARP_BYTES));
  int n_spre = 0;
  // ---- packed: the same two levels (batch 0 in registers, the next p.spre batches in shared memory, one commit group each), plus each
  //      row's base and exception list; all of it is static, so all of it is requested before the dependency wait
  const int nbatch = p.K >> 10;
  Raw12 q0 = {}, q1 = {};
  Rows12 rs = {};
  const uint4 *sm0 = nullptr, *ex0 = nullptr;  // this lane's vectors of row r0; row r1 is drow rows further (sm: 2 drow uint4 per ex uint4)
  const int drow_ex = (r1 - r0) * (p.K >> 5);
  if (PACKED && active) {
    sm0 = reinterpret_cast<const uint4*>(p.pk.sm) + (size_t)r0 * (p.K >> 4) + lane;
    ex0 = reinterpret_cast<const uint4*>(p.pk.ex) + (size_t)r0 * (p.K >> 5) + lane;
    q0 = ld_raw12(sm0, ex0, 0);
    q1 = ld_raw12(sm0 + 2 * drow_ex, ex0 + drow_ex, 0);
    for (int b = 0; b < p.spre && 1 + b < nbatch; ++b) {
      cp_async_batch12(spre_base + b * SPRE_WARP_BYTES12 + lane * 16, sm0, ex0, drow_ex, 1 + b);
      asm volatile("cp.async.commit_group;" ::: "memory");
      ++n_spre;
    }
    const int e0 = p.pk.row_ptr[r0], e1 = p.pk.row_ptr[r1];
    rs.n0 = min(p.pk.row_ptr[r0 + 1] - e0, pack12::MAX_EXC_PER_ROW);
    rs.n1 = min(p.pk.row_ptr[r1 + 1] - e1, pack12::MAX_EXC_PER_ROW);
    if (lane < rs.n0) rs.exc0 = p.pk.exc[e0 + lane];
    if (lane < rs.n1) rs.exc1 = p.pk.exc[e1 + lane];
    rs.bp0 = (uint32_t)p.pk.base[r0] - 1u;
    rs.bp1 = (uint32_t)p.pk.base[r1] - 1u;
  }
  if (first_full) {
    for (int b = 0; b < p.spre; ++b) {
      const int cb = c + 32 * NPRE + 128 * b;
      if (cb + 96 >= nchunk) break;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t d0 = (uint32_t)__cvta_generic_to_shared(spre_base + ((b * 2 + 0) * 4 + i) * 512 + lane * 16);
        const uint32_t d1 = (uint32_t)__cvta_generic_to_shared(spre_base + ((b * 2 + 1) * 4 + i) * 512 + lane * 16);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d0), "l"(p0 + cb + 32 * i) : "memory");
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d1), "l"(p1 + cb + 32 * i) : "memory");
      }
      ++n_spre;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  // ---- third level, no registers and no shared memory: everything of the two rows that the levels above did not request goes
  //      to L2 with one bulk prefetch per row (cp.async.bulk.prefetch.L2, SASS UBLKPF).  A kernel whose CTAs are resident while
  //      its producer still runs (o_proj under the decode attention, gate/up under o_proj's tail, every kernel across the
  //      ~1 us dependency release) then keeps HBM streaming through what used to be idle gaps and later reads L2 hits.
  //      It made the step slower on the in-graph timeline of the earlier target: the prefetch and the demand loads of the same
  //      rows race and both reach DRAM.  Off by default; SRGPT_GEMV_L2PF=1 keeps the experiment reproducible.
  if (!PACKED && p.l2pf && active && lane < 2) {
    const int c_req = first_full ? (32 * NPRE + 128 * n_spre) : 0;  // chunks per row already requested above
    if (c_req < nchunk) {
      const char* rowp = reinterpret_cast<const char*>(lane == 0 ? p0 : p1) + (size_t)c_req * 16;
      uint32_t bytes = (uint32_t)(nchunk - c_req) * 16u;
      while (bytes > 0) {  // pieces of <= 16 KB
        const uint32_t n = bytes > 16384u ? 16384u : bytes;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(rowp), "r"(n) : "memory");
        rowp += n;
        bytes -= n;
      }
    }
  }
  // norm weights are static too: fetch them before the wait when a thread owns at most 2 chunks of x
  uint4 nw_pre[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  const bool nw_pre_valid = (p.norm_weight != nullptr) && (nchunk_all <= 2 * THREADS);
  if (nw_pre_valid) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int cc = threadIdx.x + k * THREADS;
      if (cc < nchunk_all) nw_pre[k] = reinterpret_cast<const uint4*>(p.norm_weight)[cc];
    }
  }
  pdl_launch_dependents();
  pdl_wait();  // activations written by earlier kernels are visible from here on
  trace_mark(p.trace, 1);

  stage_x(p.x, p.norm_weight, p.eps, p.K, sx, red, nw_pre, nw_pre_valid);

  float a0 = 0.f, a1 = 0.f;
  if constexpr (PACKED) {  // batches in chunk order: the lane's fma chain is the plain kernel's
    if (active) {
      consume12(q0, q1, rs, 0, lane, px, a0, a1);
      if (p.ring) {
        // Ring of n_spre slots: batch b sits in slot (b - 1) % n_spre.  As soon as the lane has read its vectors of batch b back into
        // registers it requests batch b + n_spre into the same slot (the reads precede the cp.async in the thread's program order), so
        // n_spre batches stay in flight while batch b is decoded and consumed.  Batches are consumed in chunk order, as above.
        int slot = 0;
        for (int b = 1; b < nbatch; ++b) {
          cp_async_wait_pending(min(n_spre - 1, nbatch - 1 - b));  // groups committed after batch b's own may still be pending
          const uint8_t* s = spre_base + slot * SPRE_WARP_BYTES12 + lane * 16;
          Raw12 t0, t1;
          ld_slot12(s, t0, t1);
          if (b + n_spre < nbatch) {
            cp_async_batch12(s, sm0, ex0, drow_ex, b + n_spre);
            asm volatile("cp.async.commit_group;" ::: "memory");
          }
          consume12(t0, t1, rs, b, lane, px, a0, a1);
          if (++slot == n_spre) slot = 0;
        }
      } else {
        if (n_spre > 0) {
          asm volatile("cp.async.wait_group 0;" ::: "memory");
          for (int b = 0; b < n_spre; ++b) {
            Raw12 t0, t1;
            ld_slot12(spre_base + b * SPRE_WARP_BYTES12 + lane * 16, t0, t1);
            consume12(t0, t1, rs, 1 + b, lane, px, a0, a1);
          }
        }
        for (int b = 1 + n_spre; b < nbatch; ++b) {
          const Raw12 t0 = ld_raw12(sm0, ex0, b), t1 = ld_raw12(sm0 + 2 * drow_ex, ex0 + drow_ex, b);
          consume12(t0, t1, rs, b, lane, px, a0, a1);
        }
      }
    }
  } else if (active) {
    if (first_full) {
#pragma unroll
      for (int i = 0; i < NPRE; ++i) {
        float xf[8];
        unpack8(px[c + 32 * i], xf);
        a0 += dot8(u0[i], xf);
        a1 += dot8(u1[i], xf);
      }
      c += 32 * NPRE;
      if (n_spre > 0) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        for (int b = 0; b < n_spre; ++b) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float xf[8];
            unpack8(px[c + 32 * i], xf);
            const uint4 w0 = *reinterpret_cast<const uint4*>(spre_base + ((b * 2 + 0) * 4 + i) * 512 + lane * 16);
            const uint4 w1 = *reinterpret_cast<const uint4*>(spre_base + ((b * 2 + 1) * 4 + i) * 512 + lane * 16);
            a0 += dot8(w0, xf);
            a1 += dot8(w1, xf);
          }
          c += 128;
        }
      }
    }
    for (; c + 96 < nchunk; c += 128) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        u0[i] = ld_stream16(p0 + c + 32 * i);
        u1[i] = ld_stream16(p1 + c + 32 * i);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float xf[8];
        unpack8(px[c + 32 * i], xf);
        a0 += dot8(u0[i], xf);
        a1 += dot8(u1[i], xf);
      }
    }
    for (; c < nchunk; c += 32) {
      float xf[8];
      unpack8(px[c], xf);
      a0 += dot8(ld_stream16(p0 + c), xf);
      a1 += dot8(ld_stream16(p1 + c), xf);
    }
  }
  epilogue<MODE>(p, active, pi, r0, r1, warp, lane, a0, a1, sv, si);
  trace_mark(p.trace, 2);
}

// The end of every one-token decode GEMV: the warp sums of the lane partials a0 / a1 of rows r0 / r1, then the mode's epilogue
// (rounding points of the reference's torch ops, see the top of the file) and, for lm_head, the CTA's arg max partial.
template <int MODE>
__device__ __forceinline__ void epilogue(const Params& p, bool active, int pi, int r0, int r1, int warp, int lane, float a0, float a1, float* sv,
                                         int* si) {
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  float best = -INFINITY;
  int besti = 0x7fffffff;
  if (active && lane == 0) {
    if (MODE == SRGPT_GEMV_PLAIN && p.y_f32 != nullptr) {
      // row-parallel linear of a tensor-parallel rank: the partial sums over this rank's K slice, reduced across ranks afterwards
      *reinterpret_cast<float2*>(p.y_f32 + r0) = make_float2(a0, a1);
    } else if (MODE == SRGPT_GEMV_PLAIN) {
      float y0 = bf16_round(a0), y1 = bf16_round(a1);
      if (p.residual != nullptr) {
        y0 += e2f(p.residual[r0]);
        y1 += e2f(p.residual[r1]);
      }
      *reinterpret_cast<uint32_t*>(p.y + r0) = pack_bf16x2(y0, y1);
    } else if (MODE == SRGPT_GEMV_SWIGLU) {
      const float g = bf16_round(a0), u = bf16_round(a1);
      p.y[pi] = f2e(bf16_round(silu(g)) * u);
    } else if (MODE == SRGPT_GEMV_QKV_ROPE) {
      const int half = p.hd >> 1;
      const int head = pi / half, j = pi - head * half;
      float v0 = bf16_round(a0), v1 = bf16_round(a1);
      const int pos = *p.pos;
      if (head < p.n_heads + p.n_kv_heads) {
        const float cs = e2f(p.cos_tab[(size_t)pos * half + j]);
        const float sn = e2f(p.sin_tab[(size_t)pos * half + j]);
        const float o0 = bf16_round(bf16_round(v0 * cs) + bf16_round(-v1 * sn));
        const float o1 = bf16_round(bf16_round(v1 * cs) + bf16_round(v0 * sn));
        v0 = o0;
        v1 = o1;
      }
      if (head < p.n_heads) {
        p.y[r0] = f2e(v0);
        p.y[r1] = f2e(v1);
      } else {
        const int page = p.page_table[pos / p.page_size], slot = pos % p.page_size;
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
      if (p.logits_out != nullptr) {
        p.logits_out[r0] = a0;
        if (r1 != r0) p.logits_out[r1] = a1;
      }
      best = a0;
      besti = r0;
      if (r1 != r0 && better(a1, r1, best, besti)) { best = a1; besti = r1; }
    }
  }
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

// ---- NF4 weights (nf4.cuh): per batch a lane streams one 16-byte vector of codes per row (its 4 chunks) and lanes 0-15 / 16-31 one
//      scale each of row r0 / r1 (the row's 16 blocks of the batch, 64 bytes per row).  Lane l's chunk i lies in block 4 i + l / 8 of
//      the batch, so its two scales come from lanes 4 i + l / 8 and 16 + 4 i + l / 8 by shuffle.
struct NParams {
  Params p;
  srgpt_nf4 nf;
};
constexpr int SLOT_NF4 = 2 * 32 * 16 + 32 * 4;  // one ring slot per warp: both rows' code vectors (2 x 512 B) and the 32 scales (128 B)

struct Raw4 {
  uint4 q0, q1;
  float s;
};

__device__ __forceinline__ Raw4 ld_raw4(const uint4* q0, const uint4* q1, const float* s_lane, int b) {
  Raw4 t;
  t.q0 = ld_stream16(q0 + b * 32);
  t.q1 = ld_stream16(q1 + b * 32);
  t.s = __ldg(s_lane + b * 16);
  return t;
}

// batch b of both rows and the scales into one slot of the warp's ring (codes of r0 / r1 at +0 / +512, scales at +1024); every lane
// later reads back exactly what it requested, so no barrier is needed
__device__ __forceinline__ void cp_async_batch4(uint8_t* slot, int lane, const uint4* q0, const uint4* q1, const float* s_lane, int b) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(slot + lane * 16);
  const uint32_t ds = (uint32_t)__cvta_generic_to_shared(slot + 1024 + lane * 4);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(q0 + b * 32) : "memory");
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 512), "l"(q1 + b * 32) : "memory");
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ds), "l"(s_lane + b * 16) : "memory");
}

__device__ __forceinline__ Raw4 ld_slot4(const uint8_t* slot, int lane) {
  Raw4 t;
  t.q0 = *reinterpret_cast<const uint4*>(slot + lane * 16);
  t.q1 = *reinterpret_cast<const uint4*>(slot + 512 + lane * 16);
  t.s = *reinterpret_cast<const float*>(slot + 1024 + lane * 4);
  return t;
}

__device__ __forceinline__ uint32_t word_of(const uint4& v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w)); }

// batch b in chunk order through the plain kernel's dot8 chain: the lane's fp32 sums are those of the element-type kernel over the
// dequantized matrix
__device__ __forceinline__ void consume_nf4(const Raw4& t, const float* tab, int b, int lane, const uint4* px, float& a0, float& a1) {
  const int c = b * 128 + lane;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float s0 = __shfl_sync(0xffffffffu, t.s, 4 * i + (lane >> 3));
    const float s1 = __shfl_sync(0xffffffffu, t.s, 16 + 4 * i + (lane >> 3));
    const uint4 w0 = nf4::dequant8(word_of(t.q0, i), s0, tab);
    const uint4 w1 = nf4::dequant8(word_of(t.q1, i), s1, tab);
    float xf[8];
    unpack8(px[c + 32 * i], xf);
    a0 += dot8(w0, xf);
    a1 += dot8(w1, xf);
  }
}

// The one-token decode GEMV over NF4 planes (PLAIN, SWIGLU, QKV_ROPE; K % 1024 == 0).  The structure of the packed kernel: batch 0 in
// registers and the next p.spre batches in the warp's shared-memory slots, all requested before the dependency wait; with p.ring the
// slots are a ring every later batch streams through, else later batches load into registers.  Same x staging, row pairs and epilogue.
template <int MODE>
__global__ void __launch_bounds__(THREADS, 3) decode_gemv_nf4_kernel(const NParams np) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float red[32];
  __shared__ float sv[WARPS];
  __shared__ int si[WARPS];
  __shared__ float tab[16];
  const Params& p = np.p;
  bf16* sx = reinterpret_cast<bf16*>(smem_raw);
  const uint4* px = reinterpret_cast<const uint4*>(sx);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  trace_mark(p.trace, 0);
  const int pi = blockIdx.x * WARPS + warp;
  const bool active = pi < (p.N >> 1);
  int r0 = 0, r1 = 0;
  if (active) pair_rows<MODE>(p, pi, r0, r1);
  if (threadIdx.x < 16) tab[threadIdx.x] = nf4::code_value(threadIdx.x);  // published by stage_x's barrier

  const int nbatch = p.K >> 10;
  uint8_t* ring = smem_raw + (size_t)p.K * 2 + (size_t)warp * p.spre * SLOT_NF4;
  const uint4 *q0 = nullptr, *q1 = nullptr;
  const float* s_lane = nullptr;
  Raw4 t0 = {};
  int n_spre = 0;
  if (active) {
    q0 = reinterpret_cast<const uint4*>(np.nf.q + (size_t)r0 * (p.K >> 1)) + lane;
    q1 = reinterpret_cast<const uint4*>(np.nf.q + (size_t)r1 * (p.K >> 1)) + lane;
    s_lane = np.nf.scale + (size_t)(lane < 16 ? r0 : r1) * (p.K >> 6) + (lane & 15);
    t0 = ld_raw4(q0, q1, s_lane, 0);
    for (int b = 0; b < p.spre && 1 + b < nbatch; ++b) {
      cp_async_batch4(ring + b * SLOT_NF4, lane, q0, q1, s_lane, 1 + b);
      asm volatile("cp.async.commit_group;" ::: "memory");
      ++n_spre;
    }
  }
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

  float a0 = 0.f, a1 = 0.f;
  if (active) {
    consume_nf4(t0, tab, 0, lane, px, a0, a1);
    int slot = 0;
    for (int b = 1; b < nbatch; ++b) {
      Raw4 t;
      if (p.ring || b <= n_spre) {
        // batch b sits in slot `slot`; the groups committed after its own may still be pending
        cp_async_wait_pending(p.ring ? min(n_spre - 1, nbatch - 1 - b) : n_spre - b);
        uint8_t* s = ring + slot * SLOT_NF4;
        t = ld_slot4(s, lane);
        if (p.ring && b + n_spre < nbatch) {
          cp_async_batch4(s, lane, q0, q1, s_lane, b + n_spre);
          asm volatile("cp.async.commit_group;" ::: "memory");
        }
        if (++slot == n_spre) slot = 0;
      } else {
        t = ld_raw4(q0, q1, s_lane, b);
      }
      consume_nf4(t, tab, b, lane, px, a0, a1);
    }
  }
  epilogue<MODE>(p, active, pi, r0, r1, warp, lane, a0, a1, sv, si);
  trace_mark(p.trace, 2);
}

__global__ void __launch_bounds__(256)
lm_head_finalize_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int nparts,
                        const bf16* __restrict__ embed_table, bf16* __restrict__ next_x, int K, long long* __restrict__ out_ids,
                        int* step, int* pos) {
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ int s_tok;
  pdl_launch_dependents();
  pdl_wait();
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x)
    if (better(part_val[i], part_idx[i], best, bi)) { best = part_val[i]; bi = part_idx[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (better(sv[w], si[w], best, bi)) { best = sv[w]; bi = si[w]; }
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
// reduction tree is the same) and epilogues of decode_gemv_kernel, run for MT tokens against one stream of the weights: for every
// token the fp32 operations and their order are those of the one-token kernel, so each output is bit-identical to it.
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
};

template <int MODE, bool PACKED>
__global__ void __launch_bounds__(THREADS, 2) decode_gemv_multi_kernel(const MParams mp) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float red[32];
  __shared__ float sv[MT_MAX][WARPS];
  __shared__ int si[MT_MAX][WARPS];
  const Params& p = mp.p;
  const int nt = mp.T, tile_ch = mp.tile_ch;
  bf16* sx = reinterpret_cast<bf16*>(smem_raw);
  const uint4* px = reinterpret_cast<const uint4*>(sx);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int npairs = (MODE == MODE_LM) ? ((p.N + 1) >> 1) : (p.N >> 1);
  const int pi = blockIdx.x * WARPS + warp;
  const bool active = pi < npairs;
  int r0 = 0, r1 = 0;
  if (active) pair_rows<MODE>(p, pi, r0, r1);
  const int nchunk = p.K >> 3;
  const int nbatch = (nchunk + 127) >> 7;

  // ---- weights: batch 0 is requested before the dependency wait
  const uint4* p0 = reinterpret_cast<const uint4*>(p.W + (size_t)r0 * p.ldw);
  const uint4* p1 = reinterpret_cast<const uint4*>(p.W + (size_t)r1 * p.ldw);
  uint4 u0[4], u1[4];
  Raw12 q0 = {}, q1 = {};
  Rows12 rs = {};
  const uint4 *sm0 = nullptr, *ex0 = nullptr;
  const int drow_ex = (r1 - r0) * (p.K >> 5);
  auto load_plain = [&](int b, uint4 (&w0)[4], uint4 (&w1)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = b * 128 + lane + 32 * i;
      w0[i] = make_uint4(0, 0, 0, 0);
      w1[i] = make_uint4(0, 0, 0, 0);
      if (c < nchunk) {
        w0[i] = ld_stream16(p0 + c);
        w1[i] = ld_stream16(p1 + c);
      }
    }
  };
  if (active) {
    if constexpr (PACKED) {
      sm0 = reinterpret_cast<const uint4*>(p.pk.sm) + (size_t)r0 * (p.K >> 4) + lane;
      ex0 = reinterpret_cast<const uint4*>(p.pk.ex) + (size_t)r0 * (p.K >> 5) + lane;
      q0 = ld_raw12(sm0, ex0, 0);
      q1 = ld_raw12(sm0 + 2 * drow_ex, ex0 + drow_ex, 0);
      const int e0 = p.pk.row_ptr[r0], e1 = p.pk.row_ptr[r1];
      rs.n0 = min(p.pk.row_ptr[r0 + 1] - e0, pack12::MAX_EXC_PER_ROW);
      rs.n1 = min(p.pk.row_ptr[r1 + 1] - e1, pack12::MAX_EXC_PER_ROW);
      if (lane < rs.n0) rs.exc0 = p.pk.exc[e0 + lane];
      if (lane < rs.n1) rs.exc1 = p.pk.exc[e1 + lane];
      rs.bp0 = (uint32_t)p.pk.base[r0] - 1u;
      rs.bp1 = (uint32_t)p.pk.base[r1] - 1u;
    } else {
      load_plain(0, u0, u1);
    }
  }
  uint4 nw_pre[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  const bool nw_pre_valid = (p.norm_weight != nullptr) && (nchunk <= 2 * THREADS);
  if (nw_pre_valid) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int cc = threadIdx.x + k * THREADS;
      if (cc < nchunk) nw_pre[k] = reinterpret_cast<const uint4*>(p.norm_weight)[cc];
    }
  }
  pdl_launch_dependents();
  pdl_wait();

  float a0[MT_MAX], a1[MT_MAX];
#pragma unroll
  for (int t = 0; t < MT_MAX; ++t) a0[t] = a1[t] = 0.f;
  int b = 0;
  for (int c0 = 0; c0 < nchunk; c0 += tile_ch) {
    const int tlen = min(tile_ch, nchunk - c0);
    if (p.norm_weight != nullptr) {  // one tile holds the whole row (tile_ch == nchunk)
      for (int t = 0; t < nt; ++t)
        stage_x(p.x + (size_t)t * mp.ldx, p.norm_weight, p.eps, p.K, sx + (size_t)t * tile_ch * 8, red, nw_pre, nw_pre_valid);
    } else {
      __syncthreads();  // the previous tile is consumed
      for (int t = 0; t < nt; ++t) {
        const uint4* src = reinterpret_cast<const uint4*>(p.x + (size_t)t * mp.ldx) + c0;
        uint4* dst = reinterpret_cast<uint4*>(sx) + (size_t)t * tile_ch;
        for (int cc = threadIdx.x; cc < tlen; cc += THREADS) dst[cc] = src[cc];
      }
      __syncthreads();
    }
    if (!active) continue;
    for (; b < nbatch && b * 128 < c0 + tlen; ++b) {
      // batch 0 was requested before the wait; every later batch is requested here (a double-buffered variant needed more than
      // the 128 registers of 2 CTAs per SM and spilled)
      uint4 w0[4], w1[4];
      if constexpr (PACKED) {
        if (b > 0) {
          q0 = ld_raw12(sm0, ex0, b);
          q1 = ld_raw12(sm0 + 2 * drow_ex, ex0 + drow_ex, b);
        }
        decode_batch(q0, rs.bp0, w0);
        decode_batch(q1, rs.bp1, w1);
        patch_batch(w0, rs.exc0, rs.n0, rs.j0, b, lane);
        patch_batch(w1, rs.exc1, rs.n1, rs.j1, b, lane);
      } else {
        if (b > 0) load_plain(b, u0, u1);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          w0[i] = u0[i];
          w1[i] = u1[i];
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = b * 128 + lane + 32 * i;
        if (c < nchunk) {
#pragma unroll
          for (int t = 0; t < MT_MAX; ++t) {
            if (t < nt) {
              float xf[8];
              unpack8(px[(size_t)t * tile_ch + (c - c0)], xf);
              a0[t] += dot8(w0[i], xf);
              a1[t] += dot8(w1[i], xf);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < MT_MAX; ++t) {
    if (t < nt) {
      a0[t] = warp_sum(a0[t]);
      a1[t] = warp_sum(a1[t]);
    }
  }
  // lane t runs token t's epilogue (every lane holds every token's sums after warp_sum)
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int t = 0; t < MT_MAX; ++t) {
    if (t == lane) {
      s0 = a0[t];
      s1 = a1[t];
    }
  }
  if (active && lane < nt) {
    {
      const int t = lane;
      bf16* y = p.y + (size_t)t * mp.ldy;
      if (MODE == SRGPT_GEMV_PLAIN) {
        float y0 = bf16_round(s0), y1 = bf16_round(s1);
        if (p.residual != nullptr) {
          const bf16* res = p.residual + (size_t)t * mp.ldy;
          y0 += e2f(res[r0]);
          y1 += e2f(res[r1]);
        }
        *reinterpret_cast<uint32_t*>(y + r0) = pack_bf16x2(y0, y1);
      } else if (MODE == SRGPT_GEMV_SWIGLU) {
        const float g = bf16_round(s0), u = bf16_round(s1);
        y[pi] = f2e(bf16_round(silu(g)) * u);
      } else if (MODE == SRGPT_GEMV_QKV_ROPE) {
        const int half = p.hd >> 1;
        const int head = pi / half, j = pi - head * half;
        float v0 = bf16_round(s0), v1 = bf16_round(s1);
        const int pos = *p.pos + t;
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
          const int page = p.page_table[pos / p.page_size], slot = pos % p.page_size;
          const bool is_v = head >= p.n_heads + p.n_kv_heads;
          const int kh = head - p.n_heads - (is_v ? p.n_kv_heads : 0);
          bf16* dst = p.kv_pages + (((size_t)page * 2 + (is_v ? 1 : 0)) * p.page_size + slot) * ((size_t)p.n_kv_heads * p.hd) + kh * p.hd;
          dst[j] = f2e(v0);
          dst[j + half] = f2e(v1);
        }
      } else {  // MODE_LM
        const float l0 = bf16_round(s0), l1 = bf16_round(s1);
        if (p.logits_out != nullptr) {
          float* lo = p.logits_out + (size_t)t * p.N;
          lo[r0] = l0;
          if (r1 != r0) lo[r1] = l1;
        }
        float best = l0;
        int besti = r0;
        if (r1 != r0 && better(l1, r1, best, besti)) { best = l1; besti = r1; }
        sv[t][warp] = best;
        si[t][warp] = besti;
      }
    }
  }
  if (MODE == MODE_LM) {
    if (!active && lane < nt) {
      sv[lane][warp] = -INFINITY;
      si[lane][warp] = 0x7fffffff;
    }
    __syncthreads();
    if (threadIdx.x < nt) {  // the CTA reduction of decode_gemv_kernel, one thread per token
      const int t = threadIdx.x;
      float best = sv[t][0];
      int besti = si[t][0];
      for (int w = 1; w < WARPS; ++w)
        if (better(sv[t][w], si[t][w], best, besti)) { best = sv[t][w]; besti = si[t][w]; }
      float* pv = p.part_val + (size_t)t * 2 * gridDim.x;
      pv[blockIdx.x] = best;
      reinterpret_cast<int*>(pv + gridDim.x)[blockIdx.x] = besti;
    }
  }
}

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
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ int s_tok[MT_MAX];
  pdl_launch_dependents();
  pdl_wait();
  for (int t = 0; t < T; ++t) {
    const float* part_val = ws + (size_t)t * 2 * nparts;
    const int* part_idx = reinterpret_cast<const int*>(part_val + nparts);
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x)
      if (better(part_val[i], part_idx[i], best, bi)) { best = part_val[i]; bi = part_idx[i]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; ++w)
        if (better(sv[w], si[w], best, bi)) { best = sv[w]; bi = si[w]; }
      if (bi == 0x7fffffff) bi = 0;
      s_tok[t] = bi;
    }
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
  __shared__ float sv[8];
  __shared__ int si[8];
  pdl_launch_dependents();
  pdl_wait();
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x)
    if (better(part_val[i], part_idx[i], bv, bi)) { bv = part_val[i]; bi = part_idx[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (better(sv[w], si[w], bv, bi)) { bv = sv[w]; bi = si[w]; }
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

static int spre_default() {
  static const int v = [] {
    const char* e = getenv("SRGPT_GEMV_SPRE");
    const int x = (e != nullptr && e[0] != 0) ? atoi(e) : 1;
    return x < 0 ? 0 : (x > SPRE_MAX ? SPRE_MAX : x);
  }();
  return v;
}

// Depth of the packed kernel's per-warp ring (slots of 3 KB per warp).  SRGPT_GEMV_RING = 0 keeps the two fixed levels (batch 0 in
// registers, spre_default() batches in shared memory, the rest loaded into registers one batch at a time); n > 0 sets the depth (default
// 2).  Read at every launch, so a captured graph keeps the depth it was captured with.  At K = 4096 a depth of 2 is 56 KB per CTA, so
// the 3 CTAs per SM the registers allow still fit and 3 of a row's 4 batches are requested before the dependency wait.  Deeper rings
// (2 CTAs per SM) made o_proj and down_proj stream faster but delayed the kernel after them by more (DESIGN.md §5).  Returns -1 for the
// fixed levels, else the depth clamped to the batches after batch 0.
static int ring_depth(int K) {
  const char* e = getenv("SRGPT_GEMV_RING");
  int d = (e != nullptr && e[0] != 0) ? atoi(e) : 2;
  if (d <= 0) return -1;
  d = d > RING_MAX ? RING_MAX : d;
  const int later = (K >> 10) - 1;
  return d < later ? d : later;
}

template <int MODE, int PRE, bool PACKED = false>
static int launch_pre(const Params& p, int npairs, cudaStream_t st) {
  const int ring = PACKED ? ring_depth(p.K) : -1;
  const int spre = ring >= 0 ? ring : spre_default();
  const int smem = p.K * 2 + WARPS * spre * (PACKED ? SPRE_WARP_BYTES12 : SPRE_WARP_BYTES);
  static int configured_smem = 0;
  if (smem > 48 * 1024 && smem > configured_smem) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(decode_gemv_kernel<MODE, PRE, PACKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  Params q = p;
  q.trace = trace_next_slot();
  q.spre = spre;
  q.ring = ring >= 0 ? 1 : 0;
  static const int l2pf = [] {
    const char* v = getenv("SRGPT_GEMV_L2PF");
    return (v != nullptr && v[0] != 0) ? atoi(v) : 0;
  }();
  // 1: every GEMV (measured slower, see the kernel); 2: only o_proj, whose CTAs are resident while the latency-bound decode
  // attention leaves HBM idle (its 33 MB fit L2 many times over); 3: o_proj and the qkv GEMV
  const bool small_plain = MODE == SRGPT_GEMV_PLAIN && p.residual != nullptr && (long long)p.N * p.K <= (32LL << 20);
  q.l2pf = (l2pf == 1 || (l2pf >= 2 && small_plain) || (l2pf == 3 && MODE == SRGPT_GEMV_QKV_ROPE)) ? 1 : 0;
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, decode_gemv_kernel<MODE, PRE, PACKED>, q));
  return SRGPT_OK;
}

// Prefetch depth.  Deeper prefetch for the small matrices (PRE 2 / 4) shortens o_proj but costs occupancy (2 / 1 CTAs per SM),
// so the NEXT kernel can no longer co-reside and start early, and the step got slower on the earlier target's in-graph timeline.
// Default 1; SRGPT_GEMV_PRE_SMALL keeps the experiment reproducible.
template <int MODE>
static int launch(const Params& p, int npairs, cudaStream_t st) {
  static const int pre_small = [] {
    const char* v = getenv("SRGPT_GEMV_PRE_SMALL");
    const int x = (v != nullptr && v[0] != 0) ? atoi(v) : 1;
    return (x == 1 || x == 2 || x == 4) ? x : 1;
  }();
  const bool small = (MODE == SRGPT_GEMV_PLAIN || MODE == SRGPT_GEMV_QKV_ROPE) && ((size_t)p.N * p.K * 2 <= (size_t)64 << 20);
  if (small && pre_small == 4 && (p.K >> 3) >= 512) return launch_pre<MODE, 4>(p, npairs, st);
  if (small && pre_small >= 2 && (p.K >> 3) >= 256) return launch_pre<MODE, 2>(p, npairs, st);
  return launch_pre<MODE, 1>(p, npairs, st);
}

// the packed kernel always runs at the default depth (PRE 1)
template <int MODE, bool PACKED>
static int launch_mode(const Params& p, int npairs, cudaStream_t st) {
  if constexpr (PACKED) return launch_pre<MODE, 1, true>(p, npairs, st);
  else return launch<MODE>(p, npairs, st);
}

// The NF4 kernel's ring: the packed kernel's depth (ring_depth, SRGPT_GEMV_RING) in slots of SLOT_NF4 bytes per warp; depth 0 keeps the
// fixed levels (spre_default() batches in shared memory, the rest loaded into registers).
template <int MODE>
static int launch_nf4(const Params& p, const srgpt_nf4& nf, int npairs, cudaStream_t st) {
  const int ring = ring_depth(p.K);
  const int spre = ring >= 0 ? ring : spre_default();
  const int smem = p.K * 2 + WARPS * spre * SLOT_NF4;
  static int configured_smem = 0;
  if (smem > 48 * 1024 && smem > configured_smem) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(decode_gemv_nf4_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  NParams q = {p, nf};
  q.p.trace = trace_next_slot();
  q.p.spre = spre;
  q.p.ring = ring >= 0 ? 1 : 0;
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, decode_gemv_nf4_kernel<MODE>, q));
  return SRGPT_OK;
}

enum { W_PLAIN = 0, W_PACKED12 = 1, W_NF4 = 2 };  // the weight stream of a one-token decode GEMV

template <int MODE, int KIND>
static int launch_kind(const Params& p, const srgpt_nf4* nf, int npairs, cudaStream_t st) {
  if constexpr (KIND == W_NF4) return launch_nf4<MODE>(p, *nf, npairs, st);
  else return launch_mode<MODE, KIND == W_PACKED12>(p, npairs, st);
}

}  // namespace gemv
}  // namespace srgpt

using namespace srgpt;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a packed matrix the kernel can stream: every array present, vector-aligned planes, K a whole number of batches
static bool packed_ok(const srgpt_packed12* P, int K) {
  return P != nullptr && P->sm && P->ex && P->base && P->row_ptr && P->exc && aligned16(P->sm) && aligned16(P->ex) && (K % pack12::BATCH) == 0;
}

// checks and mode dispatch of srgpt_gemv_bf16, srgpt_gemv_packed_bf16 and srgpt_gemv_nf4_bf16 (KIND = gemv::W_*); p.W / p.ldw, p.pk or nf
// are set by the caller
template <int KIND>
static int gemv_modes(gemv::Params& p, const srgpt_nf4* nf, const void* x, void* y, int N, int K, const void* norm_weight, float eps,
                      const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                      const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream) {
  SRGPT_CHECK_ARG(x && y && N > 0 && K > 0);
  SRGPT_CHECK_ARG((N % 2) == 0 && (K % 8) == 0);
  SRGPT_CHECK_ARG(K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && (reinterpret_cast<uintptr_t>(y) & 3) == 0);
  SRGPT_CHECK_ARG(norm_weight == nullptr || aligned16(norm_weight));
  SRGPT_CHECK_ARG(mode >= SRGPT_GEMV_PLAIN && mode <= SRGPT_GEMV_QKV_ROPE);
  SRGPT_CHECK_ARG(x != y);  // x is read by late CTAs while early ones already write y
  p.x = reinterpret_cast<const bf16*>(x);
  p.y = reinterpret_cast<bf16*>(y);
  p.N = N; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.residual = reinterpret_cast<const bf16*>(residual);
  p.n_heads = n_heads; p.n_kv_heads = n_kv_heads; p.hd = head_dim;
  p.cos_tab = reinterpret_cast<const bf16*>(cos_tab);
  p.sin_tab = reinterpret_cast<const bf16*>(sin_tab);
  p.pos = pos;
  p.kv_pages = reinterpret_cast<bf16*>(kv_pages);
  p.page_table = page_table;
  p.page_size = page_size;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (mode) {
    case SRGPT_GEMV_PLAIN:
      p.hd = 2;
      return gemv::launch_kind<SRGPT_GEMV_PLAIN, KIND>(p, nf, N / 2, st);
    case SRGPT_GEMV_SWIGLU:
      SRGPT_CHECK_ARG(residual == nullptr);
      p.hd = 2;
      return gemv::launch_kind<SRGPT_GEMV_SWIGLU, KIND>(p, nf, N / 2, st);
    case SRGPT_GEMV_QKV_ROPE:
      SRGPT_CHECK_ARG(residual == nullptr && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0);
      SRGPT_CHECK_ARG(N == (n_heads + 2 * n_kv_heads) * head_dim);
      SRGPT_CHECK_ARG(cos_tab && sin_tab && pos && kv_pages && page_table && page_size > 0);
      return gemv::launch_kind<SRGPT_GEMV_QKV_ROPE, KIND>(p, nf, N / 2, st);
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
  SRGPT_CHECK_ARG(K * 2 + gemv::WARPS * gemv::RING_MAX * gemv::SLOT_NF4 <= 227 * 1024);
  gemv::Params p = {};
  return gemv_modes<gemv::W_NF4>(p, nf4, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                                 page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_bf16(const void* x, const void* W, int ldw, void* y, int N, int K, const void* norm_weight, float eps,
                               const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                               const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size,
                               void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::Params p = {};
  p.W = reinterpret_cast<const bf16*>(W);
  p.ldw = ldw;
  return gemv_modes<gemv::W_PLAIN>(p, nullptr, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                   kv_pages, page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_packed_bf16(const void* x, const srgpt_packed12* packed, void* y, int N, int K,
                                                                               const void* norm_weight, float eps, const void* residual, int mode, int n_heads,
                                                                               int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                                                                               const int* pos, void* kv_pages, const int* page_table, int page_size,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_gemv_packed_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  gemv::Params p = {};
  p.pk = *packed;
  return gemv_modes<gemv::W_PACKED12>(p, nullptr, x, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                      kv_pages, page_table, page_size, stream);
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
  p.x = reinterpret_cast<const bf16*>(x);
  p.W = reinterpret_cast<const bf16*>(W);
  p.ldw = ldw;
  p.y = reinterpret_cast<bf16*>(y);
  p.N = N; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == SRGPT_GEMV_PLAIN) {
    SRGPT_CHECK_ARG(partial_f32 != nullptr && (reinterpret_cast<uintptr_t>(partial_f32) & 7) == 0);
    p.hd = 2;
    p.y_f32 = partial_f32;
    return gemv::launch<SRGPT_GEMV_PLAIN>(p, N / 2, st);
  }
  SRGPT_CHECK_ARG(y != nullptr && (reinterpret_cast<uintptr_t>(y) & 3) == 0 && x != y);
  SRGPT_CHECK_ARG(n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0 && N == (n_heads + 2 * n_kv_heads) * head_dim);
  SRGPT_CHECK_ARG(cos_tab && sin_tab && pos && kv_pages && page_table && page_size > 0);
  SRGPT_CHECK_ARG(kv_heads_total >= n_kv_heads && kv_head_off >= 0 && kv_head_off + n_kv_heads <= kv_heads_total);
  p.n_heads = n_heads; p.n_kv_heads = n_kv_heads; p.hd = head_dim;
  p.cos_tab = reinterpret_cast<const bf16*>(cos_tab);
  p.sin_tab = reinterpret_cast<const bf16*>(sin_tab);
  p.pos = pos;
  p.kv_pages = reinterpret_cast<bf16*>(kv_pages);
  p.page_table = page_table;
  p.page_size = page_size;
  p.kv_heads_total = kv_heads_total;
  p.kv_head_off = kv_head_off;
  return gemv::launch<SRGPT_GEMV_QKV_ROPE>(p, N / 2, st);
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
  p.x = reinterpret_cast<const bf16*>(x);
  p.W = reinterpret_cast<const bf16*>(W_local);
  p.ldw = ldw; p.N = V_local; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.hd = 2;
  p.part_val = reinterpret_cast<float*>(workspace);
  p.part_idx = reinterpret_cast<int*>(p.part_val + g);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = gemv::launch<gemv::MODE_LM>(p, npairs, st);
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

// srgpt_lm_head_argmax_bf16 and its packed form; p.W / p.ldw or p.pk are set by the caller
template <bool PACKED>
static int lm_head_argmax(gemv::Params& p, const void* x, int V, int K, const void* norm_weight, float eps, float* logits_out, void* workspace,
                          const void* embed_table, void* next_x, long long* out_ids, int* step, int* pos, void* stream) {
  SRGPT_CHECK_ARG(x && workspace && out_ids && step && pos && V > 0 && K > 0);
  SRGPT_CHECK_ARG((K % 8) == 0 && K * 2 <= 200 * 1024);
  SRGPT_CHECK_ARG(aligned16(x) && (norm_weight == nullptr || aligned16(norm_weight)));
  SRGPT_CHECK_ARG((embed_table == nullptr) == (next_x == nullptr));
  SRGPT_CHECK_ARG(embed_table == nullptr || (aligned16(embed_table) && aligned16(next_x)));
  const int npairs = (V + 1) / 2;
  const int g = gemv::grid_for(npairs);
  p.x = reinterpret_cast<const bf16*>(x);
  p.N = V; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.hd = 2;
  p.logits_out = logits_out;
  p.part_val = reinterpret_cast<float*>(workspace);
  p.part_idx = reinterpret_cast<int*>(p.part_val + g);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = gemv::launch_mode<gemv::MODE_LM, PACKED>(p, npairs, st);
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
  return lm_head_argmax<false>(p, x, V, K, norm_weight, eps, logits_out, workspace, embed_table, next_x, out_ids, step, pos, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_argmax_packed_bf16(const void* x, const srgpt_packed12* packed, int V, int K,
                                                                                         const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                                         const void* embed_table, void* next_x, long long* out_ids, int* step,
                                                                                         int* pos, void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_lm_head_argmax_packed_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  gemv::Params p = {};
  p.pk = *packed;
  return lm_head_argmax<true>(p, x, V, K, norm_weight, eps, logits_out, workspace, embed_table, next_x, out_ids, step, pos, stream);
#endif
}

// ---- prompt-lookup speculative decoding: multi-token GEMV, lm_head, draft and accept ------------------------------------------
namespace srgpt {
namespace gemv {

template <int MODE, bool PACKED>
static int launch_multi(MParams& mp, int npairs, cudaStream_t st) {
  const int smem = mp.T * mp.tile_ch * 16;
  static int configured_smem = 0;
  if (smem > configured_smem) {  // the opt-in counts static shared memory too, so it is set for every size, not only above 48 KB
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(decode_gemv_multi_kernel<MODE, PACKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured_smem = smem;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  pdl_config(cfg, attr, grid_for(npairs), THREADS, smem, st);
  SRGPT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, decode_gemv_multi_kernel<MODE, PACKED>, mp));
  return SRGPT_OK;
}

// x staged per token: the whole row with RMSNorm, tiles of MT_TILE_CH chunks without
static int multi_tile(int K, bool norm) { return norm ? (K >> 3) : ((K >> 3) < MT_TILE_CH ? (K >> 3) : MT_TILE_CH); }

}  // namespace gemv
}  // namespace srgpt

template <bool PACKED>
static int gemv_multi_modes(gemv::MParams& mp, const void* x, int ldx, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                            const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                            const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream) {
  SRGPT_CHECK_ARG(x && y && N > 0 && K > 0 && T >= 1 && T <= gemv::MT_MAX);
  SRGPT_CHECK_ARG((N % 2) == 0 && (K % 8) == 0 && (ldx % 8) == 0 && ldx >= K && (ldy % 2) == 0);
  SRGPT_CHECK_ARG(aligned16(x) && (reinterpret_cast<uintptr_t>(y) & 3) == 0);
  SRGPT_CHECK_ARG(norm_weight == nullptr || aligned16(norm_weight));
  SRGPT_CHECK_ARG(mode >= SRGPT_GEMV_PLAIN && mode <= SRGPT_GEMV_QKV_ROPE);
  SRGPT_CHECK_ARG(x != y);
  const int tile = gemv::multi_tile(K, norm_weight != nullptr);
  SRGPT_CHECK_ARG(T * tile * 16 <= 200 * 1024);
  gemv::Params& p = mp.p;
  p.x = reinterpret_cast<const bf16*>(x);
  p.y = reinterpret_cast<bf16*>(y);
  p.N = N; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.residual = reinterpret_cast<const bf16*>(residual);
  p.n_heads = n_heads; p.n_kv_heads = n_kv_heads; p.hd = head_dim;
  p.cos_tab = reinterpret_cast<const bf16*>(cos_tab);
  p.sin_tab = reinterpret_cast<const bf16*>(sin_tab);
  p.pos = pos;
  p.kv_pages = reinterpret_cast<bf16*>(kv_pages);
  p.page_table = page_table;
  p.page_size = page_size;
  mp.T = T; mp.ldx = ldx; mp.ldy = ldy; mp.tile_ch = tile;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (mode) {
    case SRGPT_GEMV_PLAIN:
      SRGPT_CHECK_ARG(ldy >= N);
      p.hd = 2;
      return gemv::launch_multi<SRGPT_GEMV_PLAIN, PACKED>(mp, N / 2, st);
    case SRGPT_GEMV_SWIGLU:
      SRGPT_CHECK_ARG(residual == nullptr && ldy >= N / 2);
      p.hd = 2;
      return gemv::launch_multi<SRGPT_GEMV_SWIGLU, PACKED>(mp, N / 2, st);
    case SRGPT_GEMV_QKV_ROPE:
      SRGPT_CHECK_ARG(residual == nullptr && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && (head_dim % 2) == 0);
      SRGPT_CHECK_ARG(N == (n_heads + 2 * n_kv_heads) * head_dim && ldy >= n_heads * head_dim);
      SRGPT_CHECK_ARG(cos_tab && sin_tab && pos && kv_pages && page_table && page_size > 0);
      return gemv::launch_multi<SRGPT_GEMV_QKV_ROPE, PACKED>(mp, N / 2, st);
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
  return gemv_multi_modes<false>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                 kv_pages, page_table, page_size, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemv_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, void* y, int ldy, int T,
                                                                                   int N, int K, const void* norm_weight, float eps, const void* residual,
                                                                                   int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                                                                                   const void* sin_tab, const int* pos, void* kv_pages, const int* page_table,
                                                                                   int page_size, void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_gemv_multi_packed_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  gemv::MParams mp = {};
  mp.p.pk = *packed;
  return gemv_multi_modes<true>(mp, x, ldx, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                                kv_pages, page_table, page_size, stream);
#endif
}

template <bool PACKED>
static int lm_head_multi(gemv::MParams& mp, const void* x, int ldx, int T, int V, int K, const void* norm_weight, float eps, float* logits_out,
                         void* workspace, void* stream) {
  SRGPT_CHECK_ARG(x && workspace && V > 0 && K > 0 && T >= 1 && T <= gemv::MT_MAX);
  SRGPT_CHECK_ARG((K % 8) == 0 && (ldx % 8) == 0 && ldx >= K && aligned16(x) && (norm_weight == nullptr || aligned16(norm_weight)));
  const int tile = gemv::multi_tile(K, norm_weight != nullptr);
  SRGPT_CHECK_ARG(T * tile * 16 <= 200 * 1024);
  gemv::Params& p = mp.p;
  p.x = reinterpret_cast<const bf16*>(x);
  p.N = V; p.K = K;
  p.norm_weight = reinterpret_cast<const bf16*>(norm_weight);
  p.eps = eps;
  p.hd = 2;
  p.logits_out = logits_out;
  p.part_val = reinterpret_cast<float*>(workspace);
  mp.T = T; mp.ldx = ldx; mp.ldy = 0; mp.tile_ch = tile;
  return gemv::launch_multi<gemv::MODE_LM, PACKED>(mp, (V + 1) / 2, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_multi_bf16(const void* x, int ldx, const void* W, int ldw, int T, int V, int K,
                                                                               const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                               void* stream) {
  SRGPT_CHECK_ARG(W && aligned16(W) && (ldw % 8) == 0 && ldw >= K);
  gemv::MParams mp = {};
  mp.p.W = reinterpret_cast<const bf16*>(W);
  mp.p.ldw = ldw;
  return lm_head_multi<false>(mp, x, ldx, T, V, K, norm_weight, eps, logits_out, workspace, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_lm_head_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, int T, int V, int K,
                                                                                      const void* norm_weight, float eps, float* logits_out, void* workspace,
                                                                                      void* stream) {
  SRGPT_CHECK_ARG(packed_ok(packed, K));
#ifdef SRGPT_ELEM_F16
  set_last_error("srgpt_lm_head_multi_packed_bf16: the 12-bit packing is defined for bfloat16 weights only");
  return SRGPT_ERR_UNSUPPORTED;
#else
  gemv::MParams mp = {};
  mp.p.pk = *packed;
  return lm_head_multi<true>(mp, x, ldx, T, V, K, norm_weight, eps, logits_out, workspace, stream);
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
