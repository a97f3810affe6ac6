// Dense GEMM for sm_90a: C[M,N] = epilogue(A[M,K] · W[N,K]^T), 16-bit operands, fp32 accumulation on the Hopper tensor cores.
//
// This is the tensor-core core of the prefill path (SURVEY.md §2c K1,K3,K5,K6,K8,K9,K12,K13,K16,
// K20,K21): every nn.Linear / Conv2d(k=s) / ConvTranspose2d(k=s) the reference runs through
// cuBLAS/cuDNN (e.g. modeling_llama.py:429-431,498,221; base_extractor.py:92-97,158;
// base_projector.py:76-79) is one instantiation of this kernel with a fused epilogue.
//
// Design (Hopper-native, no library code):
//   * persistent kernel, one CTA per SM, 128 x 128 output tiles, K in blocks of 64;
//   * warpgroup 0 : TMA producer (one thread; cp.async.bulk.tensor 2D, 128B-swizzled K-major boxes, 6-stage ring);
//   * warpgroups 1, 2 : consumers, 64 rows of the tile each: wgmma.mma_async m64n128k16 straight from shared memory into
//     registers, then the fused bias / activation / residual epilogue from those registers to global memory;
//   * mbarrier pipeline: full (TMA -> wgmma, transaction bytes) and empty (wgmma retired -> TMA may refill).
// Out-of-bounds rows/cols/K are zero-filled by TMA, so M, N need no padding and K only has to
// be a multiple of 8 elements (16-byte global strides).
//
// FP8: gemm_fp8_kernel runs the same body over E4M3 operands (K blocks of 128 one-byte elements, the same 128-byte rows, wgmma
// m64n128k32.e4m3) and scales the accumulators by the row scales of both operands before the epilogue (W8A8 decoder linears, fp8.cu).
//
// NF4: gemm_nf4_kernel runs the same body over the decode GEMV's NF4 planes (nf4.cuh) instead of a 16-bit weight matrix.  The A operand
// still comes by TMA; the producer warpgroup builds each B stage itself: every thread loads its code words and block scales two stages
// ahead, dequantizes them with nf4::dequant8 into the 16-byte chunks TMA would have written (128B swizzle), then fences the generic-proxy
// stores against the wgmma reads (fence.proxy.async) and arrives on the stage's full barrier.  The consumers, the tile order and stream-K
// are those of the 16-bit kernel over the dequantized matrix, so the results are bit-identical to it.
//
// Short problems (M <= 128 rows: the projections and the lm_head of a batched decode step) have N / 128 tiles, too few to
// fill 132 SMs.  With a registered workspace they run "stream-K": the (n-tile, k-block) units are cut into gridDim.x equal
// contiguous ranges, one per SM.  A tile whose k-range is split is owned by the CTA holding its first k-block; the other CTAs
// write fp32 partial accumulators to a workspace slot (at most one per CTA: only the FIRST segment of a range can start
// mid-tile) and raise an epoch flag; the owner adds the partials in CTA order (deterministic) and runs the epilogue.  Owners
// only wait on first segments of higher CTAs, which wait on nothing: no cycles; all CTAs are co-resident (grid <= SMs).
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "nf4.cuh"
#include "srgpt_b200.h"
#include "tma.cuh"

namespace srgpt {
namespace gemm {

using namespace tma;  // mbarrier / TMA / wgmma wrappers shared with attention_wgmma.cu and region.cu

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int WG_K = 16;                      // K of one wgmma
constexpr int STAGES = 6;                     // 6 x 32 KB in flight
constexpr int A_BYTES = BM * BK * 2;
constexpr int B_BYTES = BN * BK * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NUM_THREADS = 3 * 128;          // producer warpgroup + two consumer warpgroups
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int TSK_MAX_CTAS = 256;
constexpr int TSK_FLAG_BYTES = TSK_MAX_CTAS * 4;
constexpr long long TSK_SLOT_FLOATS = (long long)BM * BN;

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// One wgmma consumes 16 elements = 32 bytes of K inside the 128B swizzle atom: +2 in the descriptor start field per step.
// d[64] (+)= A[64 x 16] · B[128 x 16]^T, both operands K-major in shared memory.  Accumulator layout (per warpgroup thread t,
// warp w = t / 32, lane l): d[4j + 2i + c] is row 16 w + l / 4 + 8 i, column 8 j + 2 (l % 4) + c.
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." SRGPT_ELEM_PTX "." SRGPT_ELEM_PTX " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}

// The E4M3 form (FP8 operands, gemm_fp8_kernel): one wgmma consumes 32 one-byte elements = the same 32 bytes of K, so the descriptor
// step and the accumulator layout are those of wgmma_m64n128k16.
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}

// per-row / per-column fp32 scales of the FP8 operands: y[m, n] = acc[m, n] * (sx[m] * sw[n])
struct Fp8Scales {
  const float* sx;  // [M]
  const float* sw;  // [N]
};

struct Params {
  int M, N, K;
  int ldc;                 // elements
  const bf16* bias;        // [N] or null
  const bf16* residual;    // [*, ldr] or null
  int ldr;
  int res_row_mod;         // >0: residual row = row % res_row_mod (broadcast position embeddings)
  void* C;
  int out_fp32;
  int gm;                  // rasterisation: m-tiles per group (see unit_to_tile)
};

struct TskWs {
  float* partial;          // [gridDim.x][BM * BN] fp32, in the consumer threads' register order
  unsigned int* flags;     // [gridDim.x], == epoch once CTA c's partial is complete
  unsigned int epoch;
};

// Tile order.  Units are walked group by group; a group is `gm` vertically adjacent m-tiles x ALL n-tiles, inside a group the
// m-tile varies fastest.  The CTAs (unit = blockIdx.x, + gridDim.x, ...) therefore work on ~132 neighbouring m-tiles of one
// weight tile, and a group's activation rows (gm * 128 * K * 2 bytes, sized to fit L2) are re-read from L2 - not HBM - for
// every n-tile.  gm = all m-tiles is the plain "m fastest" order, right when the whole activation fits L2 (Llama prompts); the
// ViT tower's activations (65536 x 4304 = 564 MB) do not.
__device__ __forceinline__ void unit_to_tile(int unit, int tiles_m, int tiles_n, int gm, int& mt, int& nt) {
  const int per_group = gm * tiles_n;
  const int g = unit / per_group;
  const int rem = unit - g * per_group;
  const int g0 = g * gm;
  const int gsz = min(gm, tiles_m - g0);
  nt = rem / gsz;
  mt = g0 + rem - nt * gsz;
}

// Fused epilogue of one consumer thread's accumulators; row0 / col0 locate d[0].  Rounding points mirror the reference's
// sequence of 16-bit torch ops (linear -> activation -> residual add), see DESIGN.md.
template <int EPI>
__device__ __forceinline__ void store_acc(const float (&d)[64], const Params& p, int row0, int col0) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = row0 + 8 * i;
    if (row >= p.M) continue;
    const int rrow = p.res_row_mod > 0 ? row % p.res_row_mod : row;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = col0 + 8 * j;
      if (col >= p.N) continue;
      const bool two = col + 1 < p.N;
      float v0 = d[4 * j + 2 * i], v1 = d[4 * j + 2 * i + 1];
      if (EPI == SRGPT_EPI_SWIGLU) {
        // interleaved weight rows: column 2c = gate_c, 2c + 1 = up_c -> out[:, c] (N is even)
        const float g = bf16_round(v0), u = bf16_round(v1);
        reinterpret_cast<bf16*>(p.C)[(size_t)row * p.ldc + (col >> 1)] = f2e(bf16_round(silu(g)) * u);
        continue;
      }
      if (EPI != SRGPT_EPI_NONE && p.bias != nullptr) {
        if (two) {
          const uint32_t b = *reinterpret_cast<const uint32_t*>(p.bias + col);
          v0 += bf16_lo(b);
          v1 += bf16_hi(b);
        } else {
          v0 += e2f(p.bias[col]);
        }
      }
      if (EPI == SRGPT_EPI_BIAS_GELU_TANH) {
        v0 = gelu_tanh(bf16_round(v0)); v1 = gelu_tanh(bf16_round(v1));
      } else if (EPI == SRGPT_EPI_BIAS_GELU_ERF) {
        v0 = gelu_erf(bf16_round(v0)); v1 = gelu_erf(bf16_round(v1));
      } else if (EPI == SRGPT_EPI_BIAS_QUICK_GELU) {
        v0 = quick_gelu(bf16_round(v0)); v1 = quick_gelu(bf16_round(v1));
      } else if (EPI == SRGPT_EPI_BIAS_RESIDUAL && p.residual != nullptr) {
        const bf16* rp = p.residual + (size_t)rrow * p.ldr + col;
        if (two) {
          const uint32_t r = *reinterpret_cast<const uint32_t*>(rp);
          v0 = bf16_round(v0) + bf16_lo(r);
          v1 = bf16_round(v1) + bf16_hi(r);
        } else {
          v0 = bf16_round(v0) + e2f(rp[0]);
        }
      }
      if (p.out_fp32) {
        float* cp = reinterpret_cast<float*>(p.C) + (size_t)row * p.ldc + col;
        if (two && (p.ldc & 1) == 0) {
          *reinterpret_cast<float2*>(cp) = make_float2(v0, v1);
        } else {
          cp[0] = v0;
          if (two) cp[1] = v1;
        }
      } else {
        bf16* cp = reinterpret_cast<bf16*>(p.C) + (size_t)row * p.ldc + col;
        if (two) {
          *reinterpret_cast<uint32_t*>(cp) = pack_bf16x2(v0, v1);
        } else {
          cp[0] = f2e(v0);
        }
      }
    }
  }
}

// FP8: the fp32 accumulators of one consumer thread times sx[row] * sw[col], before the epilogue rounds them (rows / columns past M / N
// are never stored and keep their value)
__device__ __forceinline__ void scale_acc(float (&d)[64], const Fp8Scales& sc, const Params& p, int row0, int col0) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = row0 + 8 * i;
    if (row >= p.M) continue;
    const float sx = sc.sx[row];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = col0 + 8 * j;
#pragma unroll
      for (int c = 0; c < 2; ++c)
        if (col + c < p.N) d[4 * j + 2 * i + c] *= sx * sc.sw[col + c];
    }
  }
}

__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// NF4 B operand: the code words and block scales of one k-block for one producer thread.  Thread pt fills 16-byte slot j = pt % 8 (the
// chunk of weights 8 j .. 8 j + 7 of the k-block) of tile rows pt / 8 + 16 i, i = 0..7: a warp's load covers 4 rows x 8 chunks.  A k-block
// is one scale block (BK == nf4::BLOCK), so a row's 8 chunks share one scale.
struct Nf4Raw {
  uint32_t w[8];
  float s[8];
};

// Load i of the producer's sequence: the same (m-tile, n-tile, k-block) order as the TMA producer of gemm_body
__device__ __forceinline__ void nf4_coords(bool sk, int i, int u_begin, int num_kb, int cta, int G, int tiles_m, int tiles_n, int gm, int& m0,
                                           int& n0, int& kb) {
  if (sk) {
    const int u = u_begin + i, tile = u / num_kb;
    m0 = 0;
    n0 = tile * BN;
    kb = u - tile * num_kb;
  } else {
    const int ui = i / num_kb;
    int mt, nt;
    unit_to_tile(cta + ui * G, tiles_m, tiles_n, gm, mt, nt);
    m0 = mt * BM;
    n0 = nt * BN;
    kb = i - ui * num_kb;
  }
}

// code word of chunk 8 kb + j of a row at nf4::lane_offset(8 kb + j); rows at or beyond N are not read and hold code 7 (the value +0)
__device__ __forceinline__ void nf4_fetch(const srgpt_nf4& w4, const Params& p, int n0, int kb, int r0, int j, Nf4Raw& c) {
  const size_t row_bytes = (size_t)(p.K >> 1);
  const int row_scales = p.K / nf4::BLOCK;
  const uint8_t* q = w4.q + (size_t)(n0 + r0) * row_bytes + nf4::lane_offset(8 * kb + j);
  const float* s = w4.scale + (size_t)(n0 + r0) * row_scales + kb;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    c.w[i] = 0x77777777u;
    c.s[i] = 0.f;
    if (n0 + r0 + 16 * i < p.N) {
      c.w[i] = __ldg(reinterpret_cast<const uint32_t*>(q + (size_t)(16 * i) * row_bytes));
      c.s[i] = __ldg(s + (size_t)(16 * i) * row_scales);
    }
  }
}

// SK = false: persistent over whole 128 x 128 tiles.  SK = true: stream-K over the (n-tile, k-block) units of an M <= 128
// problem (see the file comment).  FP8 = true: E4M3 operands, a K block of 128 one-byte elements (the same 128-byte rows, so the
// stage size, swizzle, ring and tile order are those of the 16-bit kernel), and the accumulators scaled by `sc` before the epilogue.
// NF4 = true: the B stages are dequantized from the planes `w4` by the producer warpgroup (tmap_b unused); everything else is the
// 16-bit kernel.
template <int EPI, bool SK, bool FP8, bool NF4 = false>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, const Params& p, const TskWs& ws, const Fp8Scales& sc,
                                          const srgpt_nf4& w4 = srgpt_nf4{nullptr, nullptr}) {
  constexpr int KB = FP8 ? 128 : BK;  // elements per k-block
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms need 1024-byte aligned stage buffers
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_kb = (p.K + KB - 1) / KB;
  const int num_units = tiles_m * tiles_n;
  const int G = (int)gridDim.x, cta = (int)blockIdx.x;
  const long long total = (long long)tiles_n * num_kb;  // stream-K units (M <= 128: one m-tile)
  auto range_begin = [&](int c) { return (int)(total * c / G); };
  const int u_begin = SK ? range_begin(cta) : 0, u_end = SK ? range_begin(cta + 1) : 0;

  // NF4: the 16 code values, behind the barriers (the 256 bytes reserved for them hold both)
  float* nf4_tab = reinterpret_cast<float*>(empty_bar + STAGES);
  if constexpr (NF4) {
    if (threadIdx.x < 16) nf4_tab[threadIdx.x] = nf4::code_value(threadIdx.x);
  }
  if (threadIdx.x == 0) {
    prefetch_tmap(tmap_a);
    if constexpr (!NF4) prefetch_tmap(tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), NF4 ? 1 + 128 : 1);  // NF4: the A transaction plus one arrive per producer thread
      mbar_init(smem_u32(&empty_bar[s]), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  if constexpr (NF4) {
    if (wg == 0) {
      // ===================== NF4 producer: A by TMA, B dequantized by the whole warpgroup =====================
      const int pt = threadIdx.x, j = pt & 7, r0 = pt >> 3;
      const int n_loads = SK ? u_end - u_begin : (cta < num_units ? (num_units - 1 - cta) / G + 1 : 0) * num_kb;
      uint32_t stage = 0, phase = 0;
      auto fetch = [&](int i, Nf4Raw& c) {
        int m0, n0, kb;
        nf4_coords(SK, i, u_begin, num_kb, cta, G, tiles_m, tiles_n, p.gm, m0, n0, kb);
        nf4_fetch(w4, p, n0, kb, r0, j, c);
      };
      auto put = [&](int i, const Nf4Raw& c) {
        int m0, n0, kb;
        nf4_coords(SK, i, u_begin, num_kb, cta, G, tiles_m, tiles_n, p.gm, m0, n0, kb);
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
        const uint32_t fb = smem_u32(&full_bar[stage]);
        uint8_t* sa = smem + stage * STAGE_BYTES;
        if (pt == 0) {
          mbar_expect_tx(fb, A_BYTES);
          tma_load_2d(smem_u32(sa), tmap_a, fb, kb * BK, m0);
        }
        // row r, 16-byte chunk c of a 128B-swizzled K-major tile sits at r * 128 + ((c ^ (r & 7)) << 4); r & 7 == r0 & 7 for all 8 rows
        uint8_t* sb = sa + A_BYTES + r0 * 128 + ((j ^ (r0 & 7)) << 4);
#pragma unroll
        for (int i2 = 0; i2 < 8; ++i2) *reinterpret_cast<uint4*>(sb + i2 * 16 * 128) = nf4::dequant8(c.w[i2], c.s[i2], nf4_tab);
        fence_proxy_async_shared();  // the generic-proxy stores before the wgmma (async proxy) reads them
        mbar_arrive(fb);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      };
      // three register buffers: the loads of a stage are issued two stages before it is dequantized
      Nf4Raw b0, b1, b2;
      if (n_loads > 0) fetch(0, b0);
      if (n_loads > 1) fetch(1, b1);
      if (n_loads > 2) fetch(2, b2);
      for (int i = 0; i < n_loads; i += 3) {
        put(i, b0);
        if (i + 3 < n_loads) fetch(i + 3, b0);
        if (i + 1 < n_loads) {
          put(i + 1, b1);
          if (i + 4 < n_loads) fetch(i + 4, b1);
        }
        if (i + 2 < n_loads) {
          put(i + 2, b2);
          if (i + 5 < n_loads) fetch(i + 5, b2);
        }
      }
      return;
    }
  }
  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      auto load = [&](int m0, int n0, int kb) {
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
        const uint32_t fb = smem_u32(&full_bar[stage]);
        mbar_expect_tx(fb, STAGE_BYTES);  // out-of-bounds rows / columns are zero-filled and still counted
        uint8_t* sa = smem + stage * STAGE_BYTES;
        tma_load_2d(smem_u32(sa), tmap_a, fb, kb * KB, m0);
        tma_load_2d(smem_u32(sa + A_BYTES), tmap_b, fb, kb * KB, n0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      };
      if (SK) {
        for (int u = u_begin; u < u_end; ++u) {
          const int tile = u / num_kb;
          load(0, tile * BN, u - tile * num_kb);
        }
      } else {
        for (int unit = cta; unit < num_units; unit += G) {
          int mt, nt;
          unit_to_tile(unit, tiles_m, tiles_n, p.gm, mt, nt);
          for (int kb = 0; kb < num_kb; ++kb) load(mt * BM, nt * BN, kb);
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup 1 -> tile rows [0, 64), warpgroup 2 -> [64, 128) =====================
  const int t = threadIdx.x & 127, ct = threadIdx.x - 128;
  const int r_in_tile = (wg - 1) * 64 + ((t >> 5) << 4) + ((t & 31) >> 2);  // row of d[0] inside the tile
  const int c_in_tile = (t & 3) * 2;                                        // column of d[0] inside the tile
  uint32_t stage = 0, phase = 0;
  float d[64];
  // accumulate `n` k-blocks into d; every stage is released as soon as the wgmma reading it has retired
  auto mainloop = [&](int n) {
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    uint32_t prev = 0;
    for (int kb = 0; kb < n; ++kb) {
      mbar_wait(smem_u32(&full_bar[stage]), phase);
      const uint32_t a_addr = smem_u32(smem + stage * STAGE_BYTES) + (wg - 1) * 64 * 128;
      const uint32_t b_addr = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
      const uint64_t a_desc = make_desc_sw128(a_addr), b_desc = make_desc_sw128(b_addr);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WG_K; ++k) {
        if constexpr (FP8)
          wgmma_m64n128k32_e4m3(d, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k));
        else
          wgmma_m64n128k16(d, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k));
      }
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();  // the previous k-block's wgmma has read its stage
        if (t == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (t == 0 && n > 0) mbar_arrive(smem_u32(&empty_bar[prev]));
  };

  if (!SK) {
    for (int unit = cta; unit < num_units; unit += G) {
      int mt, nt;
      unit_to_tile(unit, tiles_m, tiles_n, p.gm, mt, nt);
      mainloop(num_kb);
      if constexpr (FP8) scale_acc(d, sc, p, mt * BM + r_in_tile, nt * BN + c_in_tile);
      store_acc<EPI>(d, p, mt * BM + r_in_tile, nt * BN + c_in_tile);
    }
    return;
  }

  int u = u_begin;
  while (u < u_end) {
    const int tile = u / num_kb;
    const int seg_end = min(u_end, (tile + 1) * num_kb);
    const bool owner = u == tile * num_kb;
    // contributors of an owned, split tile: the CTAs after this one up to the one holding the tile's last k-block
    int c_last = cta;
    if (owner && seg_end < (tile + 1) * num_kb) {
      const int last_unit = (tile + 1) * num_kb - 1;
      while (c_last + 1 < G && range_begin(c_last + 1) <= last_unit) ++c_last;
    }
    mainloop(seg_end - u);
    float* slot = ws.partial + (size_t)cta * (BM * BN);
    if (!owner) {
      // publish the partial: every consumer thread's stores, then one release store of the epoch
#pragma unroll
      for (int i = 0; i < 64; ++i) __stcg(slot + i * 256 + ct, d[i]);
      __threadfence();
      named_bar_sync(1, 256);
      if (ct == 0) st_release_u32(ws.flags + cta, ws.epoch);
    } else {
      for (int cc = cta + 1; cc <= c_last; ++cc) {  // partials complete?  (lane 0 polls, the warp follows)
        if ((t & 31) == 0) {
          uint32_t spins = 0;
          while (ld_acquire_u32(ws.flags + cc) != ws.epoch) {
            __nanosleep(64);
            if (++spins > (1u << 24)) __trap();  // deadlock breaker
          }
        }
        __syncwarp();
        const float* src = ws.partial + (size_t)cc * (BM * BN);  // fixed order: deterministic sums
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] += __ldcg(src + i * 256 + ct);
      }
      if constexpr (FP8) scale_acc(d, sc, p, r_in_tile, tile * BN + c_in_tile);
      store_acc<EPI>(d, p, r_in_tile, tile * BN + c_in_tile);
      if (c_last > cta) {
        // every consumer has read the contributors' partials: clear their flags, so that a CUDA-graph REPLAY of this launch
        // (same baked epoch) starts from zeroed flags again
        named_bar_sync(1, 256);
        if (ct == 0)
          for (int cc = cta + 1; cc <= c_last; ++cc) st_release_u32(ws.flags + cc, 0u);
      }
    }
    u = seg_end;
  }
}

template <int EPI, bool SK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Params p, const TskWs ws) {
  gemm_body<EPI, SK, false>(&tmap_a, &tmap_b, p, ws, Fp8Scales{nullptr, nullptr});
}

template <int EPI, bool SK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const Params p, const TskWs ws,
                const Fp8Scales sc) {
  gemm_body<EPI, SK, true>(&tmap_a, &tmap_b, p, ws, sc);
}

template <int EPI, bool SK>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_nf4_kernel(const __grid_constant__ CUtensorMap tmap_a, const Params p, const TskWs ws, const srgpt_nf4 w4) {
  gemm_body<EPI, SK, false, true>(&tmap_a, nullptr, p, ws, Fp8Scales{nullptr, nullptr}, w4);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// [rows, k] row-major matrix with `ld` elements between rows -> box {128 bytes, 128 rows}, 128B swizzle; 16-bit elements, or E4M3
// bytes when fp8
static int make_tmap(CUtensorMap* tm, const void* ptr, int rows, int k, int ld, bool fp8 = false) {
  const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * (fp8 ? 1 : 2)};
  const cuuint32_t box[2] = {fp8 ? 128u : (cuuint32_t)BK, 128u};
  const int r = fp8 ? encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)
                    : encode_tmap_bf16(tm, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
  if (r != 0) {
    set_last_error("cuTensorMapEncodeTiled failed: %d (rows=%d k=%d ld=%d ptr=%p)", r, rows, k, ld, ptr);
    return SRGPT_ERR_CUDA;
  }
  return SRGPT_OK;
}

static int env_int(const char* name) {
  const char* v = getenv(name);
  return (v != nullptr && v[0] != 0) ? atoi(v) : 0;
}

struct TskState {
  void* base = nullptr;
  long long bytes = 0;
  unsigned int epoch = 0;
};
static TskState g_tsk;

static long long tsk_workspace_bytes(int ctas) { return TSK_FLAG_BYTES + (long long)ctas * TSK_SLOT_FLOATS * 4; }

template <int EPI, bool SK, bool FP8, bool NF4>
static int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const Params& p, const TskWs& ws, const Fp8Scales& sc, const srgpt_nf4& w4,
                         int grid, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    if constexpr (NF4)
      SRGPT_CHECK_CUDA(cudaFuncSetAttribute(gemm_nf4_kernel<EPI, SK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    else if constexpr (FP8)
      SRGPT_CHECK_CUDA(cudaFuncSetAttribute(gemm_fp8_kernel<EPI, SK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    else
      SRGPT_CHECK_CUDA(cudaFuncSetAttribute(gemm_kernel<EPI, SK>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  if constexpr (NF4)
    gemm_nf4_kernel<EPI, SK><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ta, p, ws, w4);
  else if constexpr (FP8)
    gemm_fp8_kernel<EPI, SK><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ta, tb, p, ws, sc);
  else
    gemm_kernel<EPI, SK><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ta, tb, p, ws);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}

// FP8: A and W hold E4M3 bytes (lda / ldw in bytes) and `sc` their scales.  NF4: W is unused and the weights are the planes `w4`, a 16-bit
// [N, K] matrix for every choice made here (stream-K or not, grid, rasterisation), so the partition is the 16-bit kernel's.
template <int EPI, bool FP8 = false, bool NF4 = false>
static int launch(const void* A, int lda, const void* W, int ldw, const Params& p, cudaStream_t stream, const Fp8Scales& sc = Fp8Scales{nullptr, nullptr},
                  const srgpt_nf4& w4 = srgpt_nf4{nullptr, nullptr}) {
  constexpr int EB = FP8 ? 1 : 2;           // bytes per element
  constexpr int KB = FP8 ? 128 : BK;        // elements per k-block
  CUtensorMap ta, tb;
  int rc = make_tmap(&ta, A, p.M, p.K, lda, FP8);
  if (rc != SRGPT_OK) return rc;
  if (!NF4) {
    rc = make_tmap(&tb, W, p.N, p.K, ldw, FP8);
    if (rc != SRGPT_OK) return rc;
  }
  const int sms = sm_count();
  TskWs ws = {nullptr, nullptr, 0};
  // one-tile-high problems whose weights are worth streaming (>= 4 MB) take the stream-K split when the caller registered a
  // workspace (srgpt_gemm_set_workspace); SRGPT_GEMM_TSK=-1 turns it off
  static const int tsk_env = env_int("SRGPT_GEMM_TSK");
  const long long sk_units = (long long)ceil_div(p.N, BN) * ceil_div(p.K, KB);
  if (tsk_env >= 0 && g_tsk.base != nullptr && p.M <= BM && (long long)p.N * p.K * EB >= (4LL << 20) &&
      g_tsk.bytes >= tsk_workspace_bytes(8)) {
    int grid = sms < TSK_MAX_CTAS ? sms : TSK_MAX_CTAS;
    if ((long long)grid > sk_units) grid = (int)sk_units;
    while (tsk_workspace_bytes(grid) > g_tsk.bytes && grid > 1) --grid;  // a small workspace only narrows the grid
    ws.flags = reinterpret_cast<unsigned int*>(g_tsk.base);
    ws.partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(g_tsk.base) + TSK_FLAG_BYTES);
    if (++g_tsk.epoch == 0) g_tsk.epoch = 1;  // flags start at 0 (zeroed workspace) and never equal a future epoch
    ws.epoch = g_tsk.epoch;
    return launch_kernel<EPI, true, FP8, NF4>(ta, tb, p, ws, sc, w4, grid, stream);
  }
  // rasterisation group: the whole M when the activation fits L2 (50 MB), else as many m-tiles as keep a group's rows <= 20 MB;
  // SRGPT_GEMM_GM forces the group size
  static const int gm_env = env_int("SRGPT_GEMM_GM");
  const int tiles_m = ceil_div(p.M, BM);
  Params pg = p;
  pg.gm = tiles_m;
  if ((double)EB * p.M * p.K > 40e6) {
    const int g = (int)(20e6 / ((double)EB * BM * p.K));
    pg.gm = g < 1 ? 1 : (g < tiles_m ? g : tiles_m);
  }
  if (gm_env > 0) pg.gm = gm_env < tiles_m ? gm_env : tiles_m;
  const long long units = (long long)tiles_m * ceil_div(p.N, BN);
  const int grid = (int)(units < sms ? units : sms);
  return launch_kernel<EPI, false, FP8, NF4>(ta, tb, pg, ws, sc, w4, grid, stream);
}

}  // namespace gemm
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) long long srgpt_gemm_workspace_bytes(void) {
  int n = sm_count();
  if (n <= 0 || n > gemm::TSK_MAX_CTAS) n = gemm::TSK_MAX_CTAS;
  return gemm::tsk_workspace_bytes(n);
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemm_set_workspace(void* workspace, long long bytes) {
  if (workspace == nullptr || bytes <= 0) {  // unregister
    gemm::g_tsk = gemm::TskState{};
    return SRGPT_OK;
  }
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 1023) == 0 && bytes >= gemm::tsk_workspace_bytes(8));
  gemm::g_tsk.base = workspace;
  gemm::g_tsk.bytes = bytes;
  gemm::g_tsk.epoch = 0;  // the caller hands over ZEROED memory
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemm_bf16(const void* A, int lda, const void* W, int ldw, void* C, int ldc, int M, int N, int K,
                               const void* bias, const void* residual, int ldr, int res_row_mod, int epilogue,
                               int out_fp32, void* stream) {
  SRGPT_CHECK_ARG(A != nullptr && W != nullptr && C != nullptr);
  SRGPT_CHECK_ARG(M > 0 && N > 0 && K > 0);
  SRGPT_CHECK_ARG(lda >= K && ldw >= K);
  SRGPT_CHECK_ARG((lda % 8) == 0 && (ldw % 8) == 0);  // 16-byte global strides for TMA
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(C) & 15) == 0);
  SRGPT_CHECK_ARG(epilogue >= SRGPT_EPI_NONE && epilogue <= SRGPT_EPI_BIAS_QUICK_GELU);
  if (epilogue == SRGPT_EPI_SWIGLU) {
    SRGPT_CHECK_ARG((N % 2) == 0 && !out_fp32 && ldc >= N / 2 && (ldc % 8) == 0);
  } else {
    SRGPT_CHECK_ARG(ldc >= N);
    SRGPT_CHECK_ARG(out_fp32 || (ldc % 8) == 0);
  }
  if (residual != nullptr) {
    SRGPT_CHECK_ARG(epilogue == SRGPT_EPI_BIAS_RESIDUAL && ldr >= N && (ldr % 8) == 0);
    SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(residual) & 15) == 0);
  }
  if (bias != nullptr) SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(bias) & 15) == 0);

  gemm::Params p;
  p.gm = 1;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.bias = reinterpret_cast<const bf16*>(bias);
  p.residual = reinterpret_cast<const bf16*>(residual);
  p.ldr = ldr; p.res_row_mod = res_row_mod;
  p.C = C; p.out_fp32 = out_fp32;

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case SRGPT_EPI_NONE: return gemm::launch<SRGPT_EPI_NONE>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_BIAS: return gemm::launch<SRGPT_EPI_BIAS>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_BIAS_GELU_TANH: return gemm::launch<SRGPT_EPI_BIAS_GELU_TANH>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_BIAS_GELU_ERF: return gemm::launch<SRGPT_EPI_BIAS_GELU_ERF>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_BIAS_RESIDUAL: return gemm::launch<SRGPT_EPI_BIAS_RESIDUAL>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_SWIGLU: return gemm::launch<SRGPT_EPI_SWIGLU>(A, lda, W, ldw, p, st);
    case SRGPT_EPI_BIAS_QUICK_GELU: return gemm::launch<SRGPT_EPI_BIAS_QUICK_GELU>(A, lda, W, ldw, p, st);
  }
  return SRGPT_ERR_INVALID;
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemm_fp8_bf16(const void* A, int lda, const float* sx, const void* W, int ldw, const float* sw,
                                                                            void* C, int ldc, int M, int N, int K, const void* residual, int ldr,
                                                                            int epilogue, void* stream) {
  SRGPT_CHECK_ARG(A != nullptr && W != nullptr && C != nullptr && sx != nullptr && sw != nullptr);
  SRGPT_CHECK_ARG(M > 0 && N > 0 && K > 0 && (K % 16) == 0);
  SRGPT_CHECK_ARG(lda >= K && ldw >= K && (lda % 16) == 0 && (ldw % 16) == 0);  // 16-byte global strides for TMA
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(C) & 15) == 0);
  SRGPT_CHECK_ARG(epilogue == SRGPT_EPI_NONE || epilogue == SRGPT_EPI_BIAS_RESIDUAL || epilogue == SRGPT_EPI_SWIGLU);
  if (epilogue == SRGPT_EPI_SWIGLU) {
    SRGPT_CHECK_ARG((N % 2) == 0 && ldc >= N / 2 && (ldc % 8) == 0);
  } else {
    SRGPT_CHECK_ARG(ldc >= N && (ldc % 8) == 0);
  }
  if (residual != nullptr) {
    SRGPT_CHECK_ARG(epilogue == SRGPT_EPI_BIAS_RESIDUAL && ldr >= N && (ldr % 8) == 0);
    SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(residual) & 15) == 0);
  }

  gemm::Params p;
  p.gm = 1;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.bias = nullptr;
  p.residual = reinterpret_cast<const bf16*>(residual);
  p.ldr = ldr; p.res_row_mod = 0;
  p.C = C; p.out_fp32 = 0;
  const gemm::Fp8Scales sc = {sx, sw};

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case SRGPT_EPI_NONE: return gemm::launch<SRGPT_EPI_NONE, true>(A, lda, W, ldw, p, st, sc);
    case SRGPT_EPI_BIAS_RESIDUAL: return gemm::launch<SRGPT_EPI_BIAS_RESIDUAL, true>(A, lda, W, ldw, p, st, sc);
    case SRGPT_EPI_SWIGLU: return gemm::launch<SRGPT_EPI_SWIGLU, true>(A, lda, W, ldw, p, st, sc);
  }
  return SRGPT_ERR_INVALID;
}

extern "C" __attribute__((visibility("default"))) int srgpt_gemm_nf4_bf16(const void* A, int lda, const srgpt_nf4* w, void* C, int ldc, int M, int N, int K,
                                                                            const void* residual, int ldr, int epilogue, void* stream) {
  SRGPT_CHECK_ARG(A != nullptr && w != nullptr && w->q != nullptr && w->scale != nullptr && C != nullptr);
  SRGPT_CHECK_ARG(M > 0 && N > 0 && K > 0 && (K % nf4::BATCH) == 0);
  SRGPT_CHECK_ARG(lda >= K && (lda % 8) == 0);  // 16-byte global strides for TMA
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(w->q) & 15) == 0 && (reinterpret_cast<uintptr_t>(w->scale) & 3) == 0);
  SRGPT_CHECK_ARG(epilogue == SRGPT_EPI_NONE || epilogue == SRGPT_EPI_BIAS_RESIDUAL || epilogue == SRGPT_EPI_SWIGLU);
  if (epilogue == SRGPT_EPI_SWIGLU) {
    SRGPT_CHECK_ARG((N % 2) == 0 && ldc >= N / 2 && (ldc % 8) == 0);
  } else {
    SRGPT_CHECK_ARG(ldc >= N && (ldc % 8) == 0);
  }
  if (residual != nullptr) {
    SRGPT_CHECK_ARG(epilogue == SRGPT_EPI_BIAS_RESIDUAL && ldr >= N && (ldr % 8) == 0);
    SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(residual) & 15) == 0);
  }

  gemm::Params p;
  p.gm = 1;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc;
  p.bias = nullptr;
  p.residual = reinterpret_cast<const bf16*>(residual);
  p.ldr = ldr; p.res_row_mod = 0;
  p.C = C; p.out_fp32 = 0;
  const gemm::Fp8Scales none = {nullptr, nullptr};

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case SRGPT_EPI_NONE: return gemm::launch<SRGPT_EPI_NONE, false, true>(A, lda, nullptr, K, p, st, none, *w);
    case SRGPT_EPI_BIAS_RESIDUAL: return gemm::launch<SRGPT_EPI_BIAS_RESIDUAL, false, true>(A, lda, nullptr, K, p, st, none, *w);
    case SRGPT_EPI_SWIGLU: return gemm::launch<SRGPT_EPI_SWIGLU, false, true>(A, lda, nullptr, K, p, st, none, *w);
  }
  return SRGPT_ERR_INVALID;
}
