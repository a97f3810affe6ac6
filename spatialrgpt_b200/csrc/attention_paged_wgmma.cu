// Causal prefill attention of new query rows over the paged KV cache (chunked prefill), sm_90a: TMA-fed K/V ring with mbarriers,
// S = Q K^T and O = P V on wgmma, online softmax in registers - the same family as attention_wgmma.cu.
//
// Replaces flash_attn_varlen_func over the past_key_value concatenation of the reference (modeling_llama.py:451-456,540-566):
// a chunk of new prompt rows at positions start_pos .. start_pos + rows - 1 attends to every cached position of its sequence.
// The chunk's own K/V are already in the cache (srgpt_rope_kv_append_varlen_bf16 runs first), so K/V come from the pages
// only and Q from the rotated fused qkv buffer.
//
// GQA packing: a CTA serves ONE kv head and all `group` query heads that share it.  The 128 rows of its M tile are
// (query row, head in group) pairs, packed m = row * group + h; a follow-up chunk of 30 rows with group 4 then fills a tile
// (instead of a quarter of one), and K/V are read once per group rather than once per head.  The Q tile is one 3-D TMA box
// {64 channels, group heads, BM / group rows} per channel half: the heads of a group are adjacent in the qkv row, so the box
// lands in shared memory as exactly that packed [128, 64] tile.
//
// One CTA per (q tile, kv head, sequence):
//   warpgroup 0     one TMA thread: the Q tile once, then K / V tiles of 64 positions = 4 pages through a 3-stage ring.  Every
//                   page is one box {64 channels, 1 kv head, 16 tokens} of a rank-5 tensor map over the layer's whole page array
//                   [n_pages, 2 (k|v), 16, nkv, hd]; four of them at 2 KB strides form the same 128B-swizzled smem tile as one
//                   64-row box.  The producer reads the page ids from the page table; logical pages past the last visible
//                   position repeat the last one (finite data, masked to p = 0, and the transaction count stays fixed).
//   warpgroups 1, 2 64 packed rows each.  Scores masked causally at position start_pos + row; P rounded to the element type in
//                   registers is the A operand of O += P V with the V tile as an MN-major B operand.
#include <math.h>

#include "common.cuh"
#include "srgpt_b200.h"
#include "tma.cuh"

namespace srgpt {
namespace attn_paged {

using namespace tma;

constexpr int HD = 128, PAGE = 16, BM = 128, BN = 64, STAGES = 3;
constexpr int NTHREADS = 3 * 128;                           // TMA warpgroup + two consumer warpgroups
constexpr int Q_C0 = BM * 128, Q_BYTES = 2 * Q_C0;          // two 64-channel halves, 128 B per packed row
constexpr int KV_C0 = BN * 128, KV_BYTES = 2 * KV_C0;       // per K (or V) tile: two 64-channel halves
constexpr int PAGE_BOX_BYTES = PAGE * 128;                  // one page, one channel half
constexpr int STAGE_BYTES = 2 * KV_BYTES;                   // K tile + V tile
constexpr int SMEM_BYTES = Q_BYTES + STAGES * STAGE_BYTES + 1024 /*align slack*/ + 64 /*barriers*/;

struct Params {
  const int* cu_seqlens;   // [n_seqs + 1]
  const int* start_pos;    // [n_seqs]
  const int* page_tables;  // [n_seqs, pt_stride]
  int pt_stride;
  int group, rpt, nqt;     // query heads per kv head, query rows per tile (BM / group), q tiles per sequence
  float scale_log2;
  bf16* out;
  int o_ld;
};

__device__ __forceinline__ void tma_load_5d(uint32_t smem_dst, const CUtensorMap* tmap, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// d[32] (+)= A[64 x 16] · B[64 x 16]^T, both operands K-major in shared memory; scale_d = 0 overwrites d
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." SRGPT_ELEM_PTX "." SRGPT_ELEM_PTX " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d)
      : "memory");
}
// d[32] += A[64 x 16] (registers, P) · B[16 x 64], B MN-major in shared memory (a V tile as loaded: kv rows, channels)
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." SRGPT_ELEM_PTX "." SRGPT_ELEM_PTX " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db)
      : "memory");
}

__global__ void __launch_bounds__(NTHREADS, 1) attn_prefill_paged_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kvmap,
                                                                         const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + STAGES * STAGE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* full_bar = bars + 1;
  uint64_t* empty_bar = bars + 1 + STAGES;

  const int qt = (int)blockIdx.x;
  const int kv_head = (int)blockIdx.y;
  const int b = (int)blockIdx.z;
  const int row_base = p.cu_seqlens[b];
  const int rows = p.cu_seqlens[b + 1] - row_base;
  const int row0 = qt * p.rpt;  // first chunk row of this tile
  if (row0 >= rows) return;     // whole CTA: q tile past the end of a shorter chunk
  const int pos0 = p.start_pos[b];
  const int last_row = min(rows, row0 + p.rpt) - 1;
  const int kv_end = pos0 + last_row + 1;  // positions [0, kv_end) are visible to some row of the tile
  const int n_tiles = (kv_end + BN - 1) / BN;

  if (threadIdx.x == 0) {
    prefetch_tmap(&qmap);
    prefetch_tmap(&kvmap);
    mbar_init(smem_u32(q_full), 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      const uint32_t qb = smem_u32(q_full);
      mbar_expect_tx(qb, 2 * 128 * p.group * p.rpt);  // rows past total_rows are zero-filled and still counted
      tma_load_3d(smem_u32(sQ), &qmap, qb, 0, kv_head * p.group, row_base + row0);
      tma_load_3d(smem_u32(sQ + Q_C0), &qmap, qb, 64, kv_head * p.group, row_base + row0);
      const int* pt = p.page_tables + (size_t)b * p.pt_stride;
      const int last_page = (kv_end - 1) / PAGE;
      uint32_t stage = 0, phase = 0;
      for (int t = 0; t < n_tiles; ++t) {
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
        const uint32_t fb = smem_u32(&full_bar[stage]);
        mbar_expect_tx(fb, STAGE_BYTES);
        uint8_t* sK = sKV + stage * STAGE_BYTES;
        uint8_t* sV = sK + KV_BYTES;
#pragma unroll
        for (int j = 0; j < BN / PAGE; ++j) {
          const int page = __ldg(pt + min(t * (BN / PAGE) + j, last_page));
          const uint32_t off = j * PAGE_BOX_BYTES;
          tma_load_5d(smem_u32(sK + off), &kvmap, fb, 0, kv_head, 0, 0, page);
          tma_load_5d(smem_u32(sK + KV_C0 + off), &kvmap, fb, 64, kv_head, 0, 0, page);
          tma_load_5d(smem_u32(sV + off), &kvmap, fb, 0, kv_head, 0, 1, page);
          tma_load_5d(smem_u32(sV + KV_C0 + off), &kvmap, fb, 64, kv_head, 0, 1, page);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup 1 -> packed rows [0, 64), warpgroup 2 -> [64, 128) =====================
  // accumulator layout (thread t of the warpgroup, warp w = t / 32, lane l): d[4j + 2i + c] is packed row 16 w + l / 4 + 8 i,
  // column 8 j + 2 (l % 4) + c
  const int t = threadIdx.x & 127, lane = t & 31;
  const int wr = (wg - 1) * 64;
  const int m0 = wr + ((t >> 5) << 4) + (lane >> 2);  // packed row of d[4j + 0/1]; d[4j + 2/3] is m0 + 8
  const int c0 = (lane & 3) * 2;
  const int m_valid = p.rpt * p.group;                // packed rows the Q box filled
  int row_of[2], pos_of[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + 8 * i;
    row_of[i] = m < m_valid ? row0 + m / p.group : rows;  // rows == "not a row of this chunk"
    pos_of[i] = pos0 + row_of[i];
  }
  const uint64_t qa0 = make_desc_sw128(smem_u32(sQ + wr * 128));
  const uint64_t qa1 = make_desc_sw128(smem_u32(sQ + Q_C0 + wr * 128));

  float o0[32], o1[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { o0[i] = 0.f; o1[i] = 0.f; }
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

  mbar_wait(smem_u32(q_full), 0);
  uint32_t stage = 0, phase = 0;
  for (int tile = 0; tile < n_tiles; ++tile) {
    mbar_wait(smem_u32(&full_bar[stage]), phase);
    uint8_t* sK = sKV + stage * STAGE_BYTES;
    uint8_t* sV = sK + KV_BYTES;
    const uint32_t k_addr = smem_u32(sK), v_addr = smem_u32(sV);

    // ---- S = Q K^T over the 128 channels (16 per wgmma)
    float s[32];
    wgmma_fence();
    const uint64_t kb0 = make_desc_sw128(k_addr), kb1 = make_desc_sw128(k_addr + KV_C0);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n64(s, qa0 + 2 * k, kb0 + 2 * k, k);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n64(s, qa1 + 2 * k, kb1 + 2 * k, 1);
    wgmma_commit();
    wgmma_wait<0>();

    // ---- causal mask at the row's position, scale to base 2, online softmax (a row's 64 scores sit in the 4 lanes of a quad)
    const int kv0 = tile * BN;
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int col = kv0 + 8 * j + c0 + c;
          float& v = s[4 * j + 2 * i + c];
          v = col <= pos_of[i] ? v * p.scale_log2 : -INFINITY;
          mx = fmaxf(mx, v);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[i], mx);
      const float m_use = m_new == -INFINITY ? 0.f : m_new;  // no visible column yet: keep p = 0, no NaN
      alpha[i] = exp2f(m[i] - m_use);
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          float& v = s[4 * j + 2 * i + c];
          v = exp2f(v - m_use);
          sum += v;
        }
      }
      l[i] = l[i] * alpha[i] + sum;
      m[i] = m_new;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o0[4 * j] *= alpha[0]; o0[4 * j + 1] *= alpha[0];
      o0[4 * j + 2] *= alpha[1]; o0[4 * j + 3] *= alpha[1];
      o1[4 * j] *= alpha[0]; o1[4 * j + 1] *= alpha[0];
      o1[4 * j + 2] *= alpha[1]; o1[4 * j + 3] *= alpha[1];
    }

    // ---- O += P V: P (element type) as the register A operand, 16 kv rows per wgmma; V tile MN-major as loaded
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                             pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
      wgmma_rs_n64(o0, a, make_desc_sw128(v_addr + kk * 16 * 128));
      wgmma_rs_n64(o1, a, make_desc_sw128(v_addr + KV_C0 + kk * 16 * 128));
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (t == 0) mbar_arrive(smem_u32(&empty_bar[stage]));  // both operand tiles of this stage have been read
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }

  // ---- O / l, rounded to the element type; packed rows outside the chunk are not stored
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float sum = l[i];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const float inv = 1.f / sum;
    if (row_of[i] >= rows) continue;
    const int head = kv_head * p.group + (m0 + 8 * i) % p.group;
    bf16* orow = p.out + (size_t)(row_base + row_of[i]) * p.o_ld + head * HD;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(orow + 8 * j + c0) = pack_bf16x2(o0[4 * j + 2 * i] * inv, o0[4 * j + 2 * i + 1] * inv);
      *reinterpret_cast<uint32_t*>(orow + 64 + 8 * j + c0) = pack_bf16x2(o1[4 * j + 2 * i] * inv, o1[4 * j + 2 * i + 1] * inv);
    }
  }
}

}  // namespace attn_paged
}  // namespace srgpt

using namespace srgpt;

extern "C" __attribute__((visibility("default"))) int srgpt_attention_prefill_paged_bf16(
    const void* q, int q_ld, void* out, int o_ld, const void* kv_pages, int n_pages, const int* page_tables, int page_table_stride, int page_size,
    const int* start_pos, const int* cu_seqlens, int n_seqs, int max_rows, int total_rows, int n_heads, int n_kv_heads, int head_dim, float scale,
    void* stream) {
  using namespace attn_paged;
  SRGPT_CHECK_ARG(q && out && kv_pages && page_tables && start_pos && cu_seqlens);
  SRGPT_CHECK_ARG(head_dim == HD && page_size == PAGE);
  SRGPT_CHECK_ARG(n_pages > 0 && page_table_stride > 0 && n_seqs > 0 && n_seqs <= 65535 && max_rows > 0 && total_rows >= max_rows);
  SRGPT_CHECK_ARG(n_heads > 0 && n_kv_heads > 0 && (n_heads % n_kv_heads) == 0 && n_heads / n_kv_heads <= BM && n_kv_heads <= 65535);
  SRGPT_CHECK_ARG((q_ld % 8) == 0 && q_ld >= n_heads * HD && (o_ld % 2) == 0 && o_ld >= n_heads * HD);
  SRGPT_CHECK_ARG((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(kv_pages) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0);
  static bool configured = false;
  if (!configured) {
    SRGPT_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_paged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  Params p;
  p.cu_seqlens = cu_seqlens;
  p.start_pos = start_pos;
  p.page_tables = page_tables;
  p.pt_stride = page_table_stride;
  p.group = n_heads / n_kv_heads;
  p.rpt = BM / p.group;
  p.nqt = ceil_div(max_rows, p.rpt);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = reinterpret_cast<bf16*>(out);
  p.o_ld = o_ld;

  CUtensorMap qmap, kvmap;
  {  // (channel, head, row) view of the q columns of the fused qkv activation; a box is a group's heads over rpt rows
    const cuuint64_t dims[3] = {(cuuint64_t)HD, (cuuint64_t)n_heads, (cuuint64_t)total_rows};
    const cuuint64_t strides[2] = {(cuuint64_t)HD * 2, (cuuint64_t)q_ld * 2};
    const cuuint32_t box[3] = {64, (cuuint32_t)p.group, (cuuint32_t)p.rpt};
    const int rc = tma::encode_tmap_bf16(&qmap, q, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc != 0) {
      set_last_error("attention (paged): cuTensorMapEncodeTiled failed (%d) for q=%p heads=%d ld=%d rows=%d", rc, q, n_heads, q_ld, total_rows);
      return SRGPT_ERR_CUDA;
    }
  }
  {  // (channel, kv head, token, k|v, page) view of one layer's page array [n_pages, 2, page_size, nkv, hd]; a box is one page
    const cuuint64_t tok = (cuuint64_t)n_kv_heads * HD * 2;
    const cuuint64_t dims[5] = {(cuuint64_t)HD, (cuuint64_t)n_kv_heads, (cuuint64_t)PAGE, 2, (cuuint64_t)n_pages};
    const cuuint64_t strides[4] = {(cuuint64_t)HD * 2, tok, tok * PAGE, tok * PAGE * 2};
    const cuuint32_t box[5] = {64, 1, (cuuint32_t)PAGE, 1, 1};
    const int rc = tma::encode_tmap_bf16(&kvmap, kv_pages, 5, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc != 0) {
      set_last_error("attention (paged): cuTensorMapEncodeTiled failed (%d) for pages=%p n_pages=%d nkv=%d", rc, kv_pages, n_pages, n_kv_heads);
      return SRGPT_ERR_CUDA;
    }
  }
  const dim3 grid((unsigned)p.nqt, (unsigned)n_kv_heads, (unsigned)n_seqs);
  attn_prefill_paged_kernel<<<grid, NTHREADS, SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(qmap, kvmap, p);
  SRGPT_CHECK_LAUNCH();
  return SRGPT_OK;
}
