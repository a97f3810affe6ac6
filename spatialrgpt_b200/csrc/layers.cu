// Composite entry points: whole transformer stacks behind ONE C-ABI call each, so the host does a single ctypes
// call per tower pass / prompt / decode step instead of ~8 per layer (the Python launch path costs more per
// kernel than several of the kernels themselves take).  Pure sequencing of the kernels in this library on the
// caller's stream; no allocation (workspaces are passed in), no synchronisation.
#include "common.cuh"
#include "srgpt_b200.h"

using namespace srgpt;

#define SRGPT_TRY(call)            \
  do {                             \
    int _rc = (call);              \
    if (_rc != SRGPT_OK) return _rc; \
  } while (0)

static inline const char* cptr(const void* p, size_t byte_off) { return reinterpret_cast<const char*>(p) + byte_off; }
static inline char* mptr(void* p, size_t byte_off) { return reinterpret_cast<char*>(p) + byte_off; }

namespace srgpt {
namespace probs {  // attention_probs.cu
int store_rows(const void* x, int rows, int H, int n_seqs, const int* cu_seqlens, void* dst, long long seq_stride, long long ld, const int* row_off,
               void* stream, const int* step = nullptr, int step_offset = 0, long long step_stride = 0);
}
}  // namespace srgpt

extern "C" __attribute__((visibility("default"))) int srgpt_vit_layers_bf16(void* x, const srgpt_siglip_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                                                              void* ws_attn, void* ws_mlp, int n_img, int T, int D, int heads, int I, float eps,
                                                                              int fc1_epilogue, void* stream) {
  SRGPT_CHECK_ARG(x && layers && ws_h && ws_qkv && ws_attn && ws_mlp && n_layers >= 0 && n_img > 0 && T > 0 && D > 0 && heads > 0 && I > 0);
  SRGPT_CHECK_ARG(D % heads == 0);
  SRGPT_CHECK_ARG(fc1_epilogue == SRGPT_EPI_BIAS_GELU_TANH || fc1_epilogue == SRGPT_EPI_BIAS_GELU_ERF || fc1_epilogue == SRGPT_EPI_BIAS_QUICK_GELU);
  const int M = n_img * T, hd = D / heads;
  const float scale = 1.0f / sqrtf((float)hd);
  for (int l = 0; l < n_layers; ++l) {
    const srgpt_siglip_layer_weights& w = layers[l];
    SRGPT_TRY(srgpt_layernorm_bf16(x, D, w.ln1_w, w.ln1_b, ws_h, D, M, D, eps, 0, stream));
    SRGPT_TRY(srgpt_gemm_bf16(ws_h, D, w.qkv_w, D, ws_qkv, 3 * D, M, 3 * D, D, w.qkv_b, nullptr, 0, 0, SRGPT_EPI_BIAS, 0, stream));
    SRGPT_TRY(srgpt_attention_prefill_bf16(ws_qkv, cptr(ws_qkv, (size_t)D * 2), cptr(ws_qkv, (size_t)2 * D * 2), ws_attn, 3 * D, 3 * D, D, n_img, T,
                                           heads, heads, hd, scale, 0, stream));
    SRGPT_TRY(srgpt_gemm_bf16(ws_attn, D, w.out_w, D, x, D, M, D, D, w.out_b, x, D, 0, SRGPT_EPI_BIAS_RESIDUAL, 0, stream));
    SRGPT_TRY(srgpt_layernorm_bf16(x, D, w.ln2_w, w.ln2_b, ws_h, D, M, D, eps, 0, stream));
    SRGPT_TRY(srgpt_gemm_bf16(ws_h, D, w.fc1_w, D, ws_mlp, I, M, I, D, w.fc1_b, nullptr, 0, 0, fc1_epilogue, 0, stream));
    SRGPT_TRY(srgpt_gemm_bf16(ws_mlp, I, w.fc2_w, I, x, D, M, D, I, w.fc2_b, x, D, 0, SRGPT_EPI_BIAS_RESIDUAL, 0, stream));
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_siglip_layers_bf16(void* x, const srgpt_siglip_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                                                                 void* ws_attn, void* ws_mlp, int n_img, int T, int D, int heads, int I, float eps,
                                                                                 void* stream) {
  return srgpt_vit_layers_bf16(x, layers, n_layers, ws_h, ws_qkv, ws_attn, ws_mlp, n_img, T, D, heads, I, eps, SRGPT_EPI_BIAS_GELU_TANH, stream);
}

// ---- Llama decoder stacks: every entry point's arrays become one LayerRef per layer, and one body per stack runs them ----------

// One decoder-layer matrix [N, K]: the element-type weight and whichever format replaces it - the 12-bit packing, NF4 planes or FP8
// codes.  A packing with sm == NULL and planes with q == NULL are held as absent (the element-type matrix is used).
struct MatRef {
  const void* w;
  const srgpt_packed12* pk;
  const srgpt_nf4* nf;
  const srgpt_fp8* f8;
};

struct LayerRef {
  const void* in_norm;
  const void* post_norm;
  void* kv_pages;
  MatRef m[4];  // qkv, o, gateup, down
};

static const srgpt_packed12* packed_or_null(const srgpt_packed12* p) { return p != nullptr && p->sm != nullptr ? p : nullptr; }
static const srgpt_nf4* planes_or_null(const srgpt_nf4& p) { return p.q != nullptr ? &p : nullptr; }

// layer l of the FP8 array when there is one, else of the element-type array with the packed or NF4 matrices of their arrays
static LayerRef layer_ref(int l, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                          const srgpt_llama_layer_fp8* fp8) {
  if (fp8 != nullptr) {
    const srgpt_llama_layer_fp8& w = fp8[l];
    LayerRef r{w.in_norm, w.post_norm, w.kv_pages, {}};
    const srgpt_fp8* f8[4] = {&w.qkv, &w.o, &w.gateup, &w.down};
    for (int i = 0; i < 4; ++i) r.m[i].f8 = f8[i];
    return r;
  }
  const srgpt_llama_layer_weights& w = layers[l];
  LayerRef r{w.in_norm, w.post_norm, w.kv_pages, {{w.qkv_w}, {w.o_w}, {w.gateup_w}, {w.down_w}}};
  if (packed != nullptr) {
    const srgpt_packed12* pk[4] = {&packed[l].qkv, &packed[l].o, &packed[l].gateup, &packed[l].down};
    for (int i = 0; i < 4; ++i) r.m[i].pk = packed_or_null(pk[i]);
  }
  if (nf4 != nullptr) {
    const srgpt_nf4* nf[4] = {&nf4[l].qkv, &nf4[l].o, &nf4[l].gateup, &nf4[l].down};
    for (int i = 0; i < 4; ++i) r.m[i].nf = planes_or_null(*nf[i]);
  }
  return r;
}

// y = epilogue(x [M, K] · W [N, K]^T): the NF4 GEMM over the planes, else the activation quantizer (into q8 [M, K], s [M]) and the FP8
// GEMM, else the element-type GEMM
static int linear(const MatRef& W, const void* x, int ldx, void* q8, float* s, void* y, int ldy, int M, int N, int K, const void* residual, int ldr,
                  int epilogue, void* stream) {
  if (W.nf != nullptr) return srgpt_gemm_nf4_bf16(x, ldx, W.nf, y, ldy, M, N, K, residual, ldr, epilogue, stream);
  if (W.f8 == nullptr) return srgpt_gemm_bf16(x, ldx, W.w, K, y, ldy, M, N, K, nullptr, residual, ldr, 0, epilogue, 0, stream);
  SRGPT_TRY(srgpt_fp8_quantize_act_bf16(x, ldx, M, K, q8, K, s, stream));
  return srgpt_gemm_fp8_bf16(q8, K, s, W.f8->q, K, W.f8->scale, y, ldy, M, N, K, residual, ldr, epilogue, stream);
}

// The prefill stacks over S rows: one prompt (cu_seqlens == NULL), prompts packed back to back (cu_seqlens), or chunks that continue
// their sequences in the paged cache (chunk; attention reads the earlier positions from the pages).  max_rows = the longest prompt / chunk.
static int prefill_layers(bool chunk, void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, const srgpt_llama_layer_fp8* fp8,
                          int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_s, int S, int H, int n_heads,
                          int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
                          const int* page_table, int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows,
                          void* stream, const srgpt_prefill_probe* probe = nullptr) {
  SRGPT_CHECK_ARG(x && (layers || fp8) && ws_h && ws_qkv && ws_attn && ws_act && n_layers >= 0 && S > 0 && H > 0 && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && I > 0);
  SRGPT_CHECK_ARG(fp8 == nullptr || (ws_q8 && ws_s));
  SRGPT_CHECK_ARG(cu_seqlens != nullptr ? (n_seqs >= 1 && max_rows >= 1 && max_rows <= S && page_table_stride > 0) : (n_seqs == 1));
  SRGPT_CHECK_ARG(!chunk || (start_pos && page_table && cu_seqlens && n_pages > 0));
  SRGPT_CHECK_ARG(probe == nullptr || (!chunk && probe->out_rows >= max(max_rows, cu_seqlens != nullptr ? 1 : S)));
  const int qd = n_heads * head_dim, kd = n_kv_heads * head_dim, nqkv = qd + 2 * kd;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const LayerRef w = layer_ref(l, layers, nullptr, nf4, fp8);
    if (probe != nullptr && probe->hidden != nullptr)  // hidden_states[l]: the rows layer l reads
      SRGPT_TRY(probs::store_rows(x, S, H, n_seqs, cu_seqlens, mptr(probe->hidden, (size_t)l * probe->hidden_layer_stride * 2), probe->hidden_seq_stride,
                                  probe->hidden_ld, probe->row_off, stream));
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.in_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(w.m[0], ws_h, H, ws_q8, ws_s, ws_qkv, nqkv, S, nqkv, H, nullptr, 0, SRGPT_EPI_NONE, stream));
    if (cu_seqlens != nullptr)
      SRGPT_TRY(srgpt_rope_kv_append_varlen_bf16(ws_qkv, S, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, start_pos, w.kv_pages, page_table,
                                                 page_table_stride, page_size, n_seqs, cu_seqlens, stream));
    else
      SRGPT_TRY(srgpt_rope_kv_append_bf16(ws_qkv, S, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, start_pos, w.kv_pages, page_table, page_size, stream));
    if (probe != nullptr && probe->attn != nullptr)  // RoPE rotated q and k in place in ws_qkv, where the attention below reads them
      SRGPT_TRY(srgpt_attention_probs_bf16(ws_qkv, nqkv, cptr(ws_qkv, (size_t)qd * 2), nqkv, n_seqs, cu_seqlens, cu_seqlens != nullptr ? max_rows : S,
                                           n_heads, n_kv_heads, head_dim, scale, mptr(probe->attn, (size_t)l * probe->attn_layer_stride * 2),
                                           probe->attn_seq_stride, probe->attn_head_stride, probe->attn_ld, probe->out_rows, probe->row_off, stream));
    if (chunk)
      SRGPT_TRY(srgpt_attention_prefill_paged_bf16(ws_qkv, nqkv, ws_attn, qd, w.kv_pages, n_pages, page_table, page_table_stride, page_size, start_pos,
                                                   cu_seqlens, n_seqs, max_rows, S, n_heads, n_kv_heads, head_dim, scale, stream));
    else if (cu_seqlens != nullptr)
      SRGPT_TRY(srgpt_attention_prefill_varlen_bf16(ws_qkv, cptr(ws_qkv, (size_t)qd * 2), cptr(ws_qkv, (size_t)(qd + kd) * 2), ws_attn, nqkv, nqkv, qd, n_seqs,
                                                    cu_seqlens, max_rows, S, n_heads, n_kv_heads, head_dim, scale, 1, stream));
    else
      SRGPT_TRY(srgpt_attention_prefill_bf16(ws_qkv, cptr(ws_qkv, (size_t)qd * 2), cptr(ws_qkv, (size_t)(qd + kd) * 2), ws_attn, nqkv, nqkv, qd, 1, S, n_heads,
                                             n_kv_heads, head_dim, scale, 1, stream));
    SRGPT_TRY(linear(w.m[1], ws_attn, qd, ws_q8, ws_s, x, H, S, H, qd, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.post_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(w.m[2], ws_h, H, ws_q8, ws_s, ws_act, I, S, 2 * I, H, nullptr, 0, SRGPT_EPI_SWIGLU, stream));
    SRGPT_TRY(linear(w.m[3], ws_act, I, ws_q8, ws_s, x, H, S, H, I, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_bf16(void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                                                                        void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads,
                                                                                        int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
                                                                                        const int* start_pos, const int* page_table, int page_size, int n_seqs, const int* cu_seqlens,
                                                                                        int max_seqlen, int page_table_stride, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(false, x, layers, nullptr, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_table, page_table_stride, page_size, 0, n_seqs, cu_seqlens, max_seqlen, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_fp8_bf16(
    void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_scale, int S,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_table,
    int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(false, x, nullptr, nullptr, layers, n_layers, ws_h, ws_qkv, ws_attn, ws_act, ws_q8, ws_scale, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_table, page_table_stride, page_size, 0, n_seqs, cu_seqlens, max_seqlen, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_nf4_bf16(
    void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
    void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
    const int* start_pos, const int* page_table, int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride,
    void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr && nf4 != nullptr);
  return prefill_layers(false, x, layers, nf4, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_table, page_table_stride, page_size, 0, n_seqs, cu_seqlens, max_seqlen, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_probe_bf16(
    void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, const srgpt_llama_layer_fp8* fp8, int n_layers, void* ws_h,
    void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_scale, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
    const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables, int page_size, int n_seqs, const int* cu_seqlens,
    int max_seqlen, int page_table_stride, const srgpt_prefill_probe* probe, void* stream) {
  SRGPT_CHECK_ARG(probe != nullptr);
  return prefill_layers(false, x, layers, nf4, fp8, n_layers, ws_h, ws_qkv, ws_attn, ws_act, ws_q8, ws_scale, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, 0, n_seqs, cu_seqlens, max_seqlen, stream, probe);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_bf16(
    void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, int S, int H, int n_heads,
    int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables,
    int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(true, x, layers, nullptr, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_fp8_bf16(
    void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_scale, int S,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
    const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(true, x, nullptr, nullptr, layers, n_layers, ws_h, ws_qkv, ws_attn, ws_act, ws_q8, ws_scale, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_nf4_bf16(
    void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
    void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
    const int* start_pos, const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows,
    void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr && nf4 != nullptr);
  return prefill_layers(true, x, layers, nf4, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows, stream);
}

// the one-token GEMV of W: over the NF4 planes, else the packing, else the FP8 codes, else the element-type weight
static int gemv(const MatRef& W, const void* x, void* y, int N, int K, const void* norm_weight, float eps, const void* residual, int mode, int n_heads,
                int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages, const int* page_table,
                int page_size, void* stream) {
  if (W.nf != nullptr)
    return srgpt_gemv_nf4_bf16(x, W.nf, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                               page_table, page_size, stream);
  if (W.pk != nullptr)
    return srgpt_gemv_packed_bf16(x, W.pk, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                                  page_table, page_size, stream);
  if (W.f8 != nullptr)
    return srgpt_gemv_fp8_bf16(x, W.f8, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                               page_table, page_size, stream);
  return srgpt_gemv_bf16(x, W.w, K, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages, page_table,
                         page_size, stream);
}

static int decode_step(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       const srgpt_llama_layer_fp8* fp8, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads,
                       int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
                       const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                       float* logits_out, long long* out_ids, int* step, void* stream, const srgpt_decode_probe* probe = nullptr) {
  SRGPT_CHECK_ARG(h && (layers || fp8) && q_buf && attn_buf && act_buf && pos && page_table && final_norm && lm_head && lm_workspace && out_ids && step);
  SRGPT_CHECK_ARG(probe == nullptr || probe->hidden == nullptr || I >= H);  // act_buf holds the final norm row
  const int qd = n_heads * head_dim, nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const LayerRef w = layer_ref(l, layers, packed, nf4, fp8);
    if (probe != nullptr && probe->hidden != nullptr)  // hidden_states[l] of this step: the row layer l reads
      SRGPT_TRY(probs::store_rows(h, 1, H, 1, nullptr, mptr(probe->hidden, (size_t)l * probe->hidden_layer_stride * 2), 0, probe->hidden_row_stride,
                                  nullptr, stream, step, probe->step_offset, probe->hidden_step_stride));
    SRGPT_TRY(gemv(w.m[0], h, q_buf, nqkv, H, w.in_norm, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                   w.kv_pages, page_table, page_size, stream));
    SRGPT_TRY(srgpt_attention_decode_bf16(q_buf, attn_buf, w.kv_pages, page_table, page_size, pos, n_heads, n_kv_heads, head_dim, scale, stream));
    if (probe != nullptr && probe->attn != nullptr)  // the rotated q of this step and the K pages the attention above just read
      SRGPT_TRY(srgpt_attention_probs_decode_bf16(q_buf, qd, w.kv_pages, page_table, 0, page_size, pos, 1, n_heads, n_kv_heads, head_dim, scale,
                                                  probe->off, probe->n_prompt, probe->T, probe->n_cols, step, probe->step_offset,
                                                  mptr(probe->attn, (size_t)l * probe->attn_layer_stride * 2), probe->attn_step_stride,
                                                  probe->attn_row_stride, probe->attn_head_stride, probe->ws, stream));
    SRGPT_TRY(gemv(w.m[1], attn_buf, h, H, qd, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(gemv(w.m[2], h, act_buf, 2 * I, H, w.post_norm, eps, nullptr, SRGPT_GEMV_SWIGLU, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                   stream));
    SRGPT_TRY(gemv(w.m[3], act_buf, h, H, I, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, stream));
  }
  if (probe != nullptr && probe->hidden != nullptr) {  // hidden_states[L]: the final norm of the last residual row (LlamaDecoder.final_norm)
    SRGPT_TRY(srgpt_rmsnorm_bf16(h, H, final_norm, act_buf, H, 1, H, eps, stream));
    SRGPT_TRY(probs::store_rows(act_buf, 1, H, 1, nullptr, mptr(probe->hidden, (size_t)n_layers * probe->hidden_layer_stride * 2), 0,
                                probe->hidden_row_stride, nullptr, stream, step, probe->step_offset, probe->hidden_step_stride));
  }
  if (packed_or_null(lm_packed) != nullptr)
    return srgpt_lm_head_argmax_packed_bf16(h, lm_packed, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
  return srgpt_lm_head_argmax_bf16(h, lm_head, H, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_bf16(void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf,
                                                                                     void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                                                                     const void* cos_tab, const void* sin_tab, int* pos, const int* page_table,
                                                                                     int page_size, const void* final_norm, const void* lm_head, int V,
                                                                                     const void* embed_table, void* lm_workspace, float* logits_out,
                                                                                     long long* out_ids, int* step, void* stream) {
  return decode_step(h, layers, nullptr, nullptr, nullptr, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, nullptr, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_packed_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table,
    int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
    float* logits_out, long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(packed != nullptr);
  return decode_step(h, layers, packed, nullptr, nullptr, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_nf4_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H,
    int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
    const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out,
    long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(nf4 != nullptr);
  return decode_step(h, layers, nullptr, nf4, nullptr, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_fp8_bf16(
    void* h, const srgpt_llama_layer_fp8* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads,
    int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size, const void* final_norm,
    const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out, long long* out_ids,
    int* step, void* stream) {
  return decode_step(h, nullptr, nullptr, nullptr, layers, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

// The decode step of any weight format (packed / nf4 / fp8 as the _packed / _nf4 / _fp8 entries take them; at most one given) with the
// probes of `probe` recorded ahead of the lm_head that advances step and pos; h, the KV cache, the ids and the logits are those of the
// unprobed entry.
extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_probe_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
    const srgpt_llama_layer_fp8* fp8, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I,
    float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size, const void* final_norm, const void* lm_head,
    const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out, long long* out_ids, int* step,
    const srgpt_decode_probe* probe, void* stream) {
  SRGPT_CHECK_ARG(probe != nullptr && (probe->hidden != nullptr || probe->attn != nullptr));
  SRGPT_CHECK_ARG((packed != nullptr) + (nf4 != nullptr) + (fp8 != nullptr) <= 1 && (fp8 != nullptr || layers != nullptr));
  return decode_step(h, fp8 != nullptr ? nullptr : layers, packed, nf4, fp8, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps,
                     cos_tab, sin_tab, pos, page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids,
                     step, stream, probe);
}

// ---- T-row passes: T rows through the layer stack, every weight streamed once, each row with the arithmetic of a one-token step ------
// the T-row GEMV of W: over the NF4 planes, else the packing, else the element-type weight
static int gemv_multi(const MatRef& W, const void* x, int ldx, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                      const void* residual, int mode, void* stream) {
  if (W.nf != nullptr)
    return srgpt_gemv_multi_nf4_bf16(x, ldx, W.nf, y, ldy, T, N, K, norm_weight, eps, residual, mode, 0, 0, 0, nullptr, nullptr, nullptr, nullptr,
                                     nullptr, 0, stream);
  if (W.pk != nullptr)
    return srgpt_gemv_multi_packed_bf16(x, ldx, W.pk, y, ldy, T, N, K, norm_weight, eps, residual, mode, 0, 0, 0, nullptr, nullptr, nullptr, nullptr,
                                        nullptr, 0, stream);
  return srgpt_gemv_multi_bf16(x, ldx, W.w, K, y, ldy, T, N, K, norm_weight, eps, residual, mode, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                               stream);
}

// the T-row QKV + RoPE + KV-append GEMV of W: row t at pos_rows[t], through page_tables + t * pt_stride
static int gemv_rows(const MatRef& W, const void* x, int ldx, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps, int n_heads,
                     int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows, void* kv_pages, const int* page_tables,
                     int pt_stride, int page_size, void* stream) {
  if (W.nf != nullptr)
    return srgpt_gemv_rows_nf4_bf16(x, ldx, W.nf, y, ldy, T, N, K, norm_weight, eps, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos_rows, kv_pages,
                                    page_tables, pt_stride, page_size, stream);
  if (W.pk != nullptr)
    return srgpt_gemv_rows_packed_bf16(x, ldx, W.pk, y, ldy, T, N, K, norm_weight, eps, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos_rows,
                                       kv_pages, page_tables, pt_stride, page_size, stream);
  return srgpt_gemv_rows_bf16(x, ldx, W.w, K, y, ldy, T, N, K, norm_weight, eps, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos_rows, kv_pages,
                              page_tables, pt_stride, page_size, stream);
}

// The layers over the T rows of h [T, H]: row t is at position pos_rows[t] of the sequence whose page table is page_tables + t * pt_stride
// (pt_stride = 0: T consecutive positions of one sequence, the verify pass).  5 kernels per layer.
static int rows_layers(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       int n_layers, void* q_buf, void* attn_buf, void* act_buf, int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                       const void* cos_tab, const void* sin_tab, const int* pos_rows, const int* page_tables, int pt_stride, int page_size,
                       void* stream) {
  const int qd = n_heads * head_dim, nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const LayerRef w = layer_ref(l, layers, packed, nf4, nullptr);
    SRGPT_TRY(gemv_rows(w.m[0], h, H, q_buf, qd, T, nqkv, H, w.in_norm, eps, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos_rows, w.kv_pages,
                        page_tables, pt_stride, page_size, stream));
    SRGPT_TRY(srgpt_attention_decode_rows_bf16(q_buf, qd, attn_buf, qd, w.kv_pages, page_tables, pt_stride, page_size, pos_rows, T, n_heads, n_kv_heads,
                                               head_dim, scale, stream));
    SRGPT_TRY(gemv_multi(w.m[1], attn_buf, qd, h, H, T, H, qd, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, stream));
    SRGPT_TRY(gemv_multi(w.m[2], h, H, act_buf, I, T, 2 * I, H, w.post_norm, eps, nullptr, SRGPT_GEMV_SWIGLU, stream));
    SRGPT_TRY(gemv_multi(w.m[3], act_buf, I, h, H, T, H, I, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, stream));
  }
  return SRGPT_OK;
}

// final norm + lm_head over the T rows: fp32 logits [T, V] (optional) and every row's arg max partials in lm_workspace
static int lm_head_rows(const void* h, int T, int H, float eps, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
                        float* logits_rows, void* lm_workspace, void* stream) {
  if (packed_or_null(lm_packed) != nullptr)
    return srgpt_lm_head_multi_packed_bf16(h, H, lm_packed, T, V, H, final_norm, eps, logits_rows, lm_workspace, stream);
  return srgpt_lm_head_multi_bf16(h, H, lm_head, H, T, V, H, final_norm, eps, logits_rows, lm_workspace, stream);
}

// verify pass of prompt-lookup speculative decoding: the draft writes pos_rows[t] = *pos + t, the rows pass runs over the one page table
static int verify_step(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       int n_layers, void* q_buf, void* attn_buf, void* act_buf, int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                       const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows, const int* page_table, int page_size, const void* final_norm,
                       const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                       float* logits_rows, float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram, int* draft_ids, long long* out_ids,
                       int out_cap, int* step, int* state, void* stream) {
  SRGPT_CHECK_ARG(h && layers && q_buf && attn_buf && act_buf && pos && pos_rows && page_table && final_norm && lm_head && lm_workspace && out_ids &&
                  step && state && draft_ids);
  SRGPT_CHECK_ARG(logits_all == nullptr || logits_rows != nullptr);
  SRGPT_TRY(srgpt_spec_draft(prompt_ids, prompt_len, out_ids, step, pos, pos_rows, T, ngram, embed_table, h, H, draft_ids, state, stream));
  SRGPT_TRY(rows_layers(h, layers, packed, nf4, n_layers, q_buf, attn_buf, act_buf, T, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos_rows,
                        page_table, 0, page_size, stream));
  SRGPT_TRY(lm_head_rows(h, T, H, eps, final_norm, lm_head, lm_packed, V, logits_rows, lm_workspace, stream));
  return srgpt_spec_accept(lm_workspace, V, T, draft_ids, out_ids, out_cap, step, pos, state, logits_rows, logits_all, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_verify_step_bf16(
    void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int T, int H, int n_heads,
    int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows, const int* page_table,
    int page_size, const void* final_norm, const void* lm_head, int V, const void* embed_table, void* lm_workspace, float* logits_rows,
    float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram, int* draft_ids, long long* out_ids, int out_cap, int* step, int* state, void* stream) {
  return verify_step(h, layers, nullptr, nullptr, n_layers, q_buf, attn_buf, act_buf, T, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos, pos_rows,
                     page_table, page_size, final_norm, lm_head, nullptr, V, embed_table, lm_workspace, logits_rows, logits_all, prompt_ids, prompt_len, ngram,
                     draft_ids, out_ids, out_cap, step, state, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_verify_step_packed_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows,
    const int* page_table, int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table,
    void* lm_workspace, float* logits_rows, float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram, int* draft_ids, long long* out_ids, int out_cap,
    int* step, int* state, void* stream) {
  SRGPT_CHECK_ARG(packed != nullptr);
  return verify_step(h, layers, packed, nullptr, n_layers, q_buf, attn_buf, act_buf, T, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos, pos_rows,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows, logits_all, prompt_ids, prompt_len, ngram,
                     draft_ids, out_ids, out_cap, step, state, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_verify_step_nf4_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows,
    const int* page_table, int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table,
    void* lm_workspace, float* logits_rows, float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram, int* draft_ids, long long* out_ids,
    int out_cap, int* step, int* state, void* stream) {
  SRGPT_CHECK_ARG(nf4 != nullptr);
  return verify_step(h, layers, nullptr, nf4, n_layers, q_buf, attn_buf, act_buf, T, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     pos_rows, page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows, logits_all, prompt_ids,
                     prompt_len, ngram, draft_ids, out_ids, out_cap, step, state, stream);
}

// ---- decode step of B sequences, each with exactly the arithmetic of its one-token step ---------------------------------------------
// Row b of h [B, H] is the newest token of the sequence at position pos_rows[b] with page table page_tables + b * pt_stride.  The rows
// pass, then lm_head over the B rows and the advance: greedy (seeds == NULL) the arg max of each row; sampled, row b draws from its fp32
// logits row with seeds[b] at counter *step (srgpt_sample_rows into ids [B]).  Token b goes to out_ids[*step * B + b], h row b becomes its
// embedding, pos_rows[b] and then *step advance.
static int decode_rows(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       int n_layers, void* q_buf, void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                       const void* cos_tab, const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride, int page_size,
                       const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                       float* logits_rows, const float* sample_params, const unsigned long long* seeds, long long* ids, long long* out_ids, int* step,
                       const srgpt_guidance* guidance, void* stream, bool warped = false) {
  // warped: sample_params is the float[6] of srgpt_sample_rows_warped (typical / epsilon / eta after top-p)
  auto sample_rows = warped ? srgpt_sample_rows_warped : srgpt_sample_rows;
  SRGPT_CHECK_ARG(B >= 1 && B <= SRGPT_SPEC_T_MAX && pt_stride > 0);
  SRGPT_CHECK_ARG(guidance == nullptr || ((B % 2) == 0 && guidance->scale && guidance->guided_rows && ids && logits_rows));
  SRGPT_CHECK_ARG(h && layers && q_buf && attn_buf && act_buf && pos_rows && page_tables && final_norm && lm_head && embed_table && lm_workspace &&
                  out_ids && step);
  SRGPT_CHECK_ARG(seeds == nullptr || (sample_params && ids && logits_rows));
  SRGPT_TRY(rows_layers(h, layers, packed, nf4, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                        pos_rows, page_tables, pt_stride, page_size, stream));
  SRGPT_TRY(lm_head_rows(h, B, H, eps, final_norm, lm_head, lm_packed, V, logits_rows, lm_workspace, stream));
  if (guidance != nullptr) {  // rows B/2 .. B-1 are the unconditional branches of rows 0 .. B/2-1; each pair takes the guided choice
    const int P = B / 2;
    SRGPT_TRY(srgpt_guidance_rows(logits_rows, V, P, guidance->scale, guidance->guided_rows, nullptr, seeds == nullptr ? ids : nullptr, stream));
    if (seeds != nullptr) {
      SRGPT_TRY(sample_rows(guidance->guided_rows, 1, V, P, V, sample_params, seeds, step, 0, ids, stream));
      SRGPT_TRY(srgpt_guidance_pair_ids(ids, P, stream));
    }
    return srgpt_rows_advance(lm_workspace, V, ids, B, embed_table, h, H, out_ids, step, pos_rows, stream);
  }
  if (seeds != nullptr) SRGPT_TRY(sample_rows(logits_rows, 1, V, B, V, sample_params, seeds, step, 0, ids, stream));
  return srgpt_rows_advance(lm_workspace, V, seeds != nullptr ? ids : nullptr, B, embed_table, h, H, out_ids, step, pos_rows, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_rows_bf16(
    void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads,
    int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride, int page_size,
    const void* final_norm, const void* lm_head, int V, const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params,
    const unsigned long long* seeds, long long* ids, long long* out_ids, int* step, void* stream) {
  return decode_rows(h, layers, nullptr, nullptr, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                     pos_rows, page_tables, pt_stride, page_size, final_norm, lm_head, nullptr, V, embed_table, lm_workspace, logits_rows, sample_params,
                     seeds, ids, out_ids, step, nullptr, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_rows_packed_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos_rows,
    const int* page_tables, int pt_stride, int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
    const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params, const unsigned long long* seeds, long long* ids,
    long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(packed != nullptr);
  return decode_rows(h, layers, packed, nullptr, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                     pos_rows, page_tables, pt_stride, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows,
                     sample_params, seeds, ids, out_ids, step, nullptr, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_rows_nf4_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos_rows,
    const int* page_tables, int pt_stride, int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
    const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params, const unsigned long long* seeds, long long* ids,
    long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(nf4 != nullptr);
  return decode_rows(h, layers, nullptr, nf4, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                     pos_rows, page_tables, pt_stride, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows,
                     sample_params, seeds, ids, out_ids, step, nullptr, stream);
}

// The rows step of B = 2P rows with classifier-free guidance: one entry point for every weight format of the step (packed / nf4 may be
// NULL, not both given), the same layer body as the three above.
extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_rows_guided_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4, int n_layers,
    void* q_buf, void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab,
    const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride, int page_size, const void* final_norm, const void* lm_head,
    const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params,
    const unsigned long long* seeds, long long* ids, long long* out_ids, int* step, const srgpt_guidance* guidance, void* stream) {
  SRGPT_CHECK_ARG(packed == nullptr || nf4 == nullptr);
  return decode_rows(h, layers, packed, nf4, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                     pos_rows, page_tables, pt_stride, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows,
                     sample_params, seeds, ids, out_ids, step, guidance, stream);
}

// The sampled rows step, plain or guided (guidance may be NULL), drawing with srgpt_sample_rows_warped: warp_params = device float[6]
// {temperature, top_p, top_k, typical_p, epsilon_cutoff, eta_cutoff}.  One entry point for every weight format of the step, as the
// guided one; the same kernels as the sampled step of srgpt_llama_decode_rows_bf16 / _guided_bf16 with the warped sampler in place of
// srgpt_sample_rows.
extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_rows_warped_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4, int n_layers,
    void* q_buf, void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab,
    const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride, int page_size, const void* final_norm, const void* lm_head,
    const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_rows, const float* warp_params,
    const unsigned long long* seeds, long long* ids, long long* out_ids, int* step, const srgpt_guidance* guidance, void* stream) {
  SRGPT_CHECK_ARG(packed == nullptr || nf4 == nullptr);
  SRGPT_CHECK_ARG(warp_params != nullptr && seeds != nullptr);
  return decode_rows(h, layers, packed, nf4, n_layers, q_buf, attn_buf, act_buf, B, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab,
                     pos_rows, page_tables, pt_stride, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_rows,
                     warp_params, seeds, ids, out_ids, step, guidance, stream, true);
}
