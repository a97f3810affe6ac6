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

// One decoder layer as the prefill stacks see it: the element-type matrices of `srgpt_llama_layer_weights`, or the FP8 planes of
// `srgpt_llama_layer_fp8` (w8 != NULL), or with `srgpt_llama_layer_nf4` the NF4 planes of every matrix whose q != NULL (w4; the others
// keep their element-type matrix).
struct LayerRef {
  const void* in_norm;
  const void* post_norm;
  void* kv_pages;
  const void* w[4];        // qkv, o, gateup, down
  const srgpt_fp8* w8[4];  // the same, FP8; NULL for element-type layers
  const srgpt_nf4* w4[4];  // the same, NF4; NULL where the element-type matrix is used
};

static const srgpt_nf4* planes_or_null(const srgpt_nf4& p) { return p.q != nullptr ? &p : nullptr; }

static LayerRef layer_ref(const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_fp8* layers8, int l,
                          const srgpt_llama_layer_nf4* layers4 = nullptr) {
  if (layers8 != nullptr) {
    const srgpt_llama_layer_fp8& w = layers8[l];
    return LayerRef{w.in_norm, w.post_norm, w.kv_pages, {nullptr, nullptr, nullptr, nullptr}, {&w.qkv, &w.o, &w.gateup, &w.down},
                    {nullptr, nullptr, nullptr, nullptr}};
  }
  const srgpt_llama_layer_weights& w = layers[l];
  LayerRef r{w.in_norm, w.post_norm, w.kv_pages, {w.qkv_w, w.o_w, w.gateup_w, w.down_w}, {nullptr, nullptr, nullptr, nullptr},
             {nullptr, nullptr, nullptr, nullptr}};
  if (layers4 != nullptr) {
    const srgpt_llama_layer_nf4& n = layers4[l];
    r.w4[0] = planes_or_null(n.qkv);
    r.w4[1] = planes_or_null(n.o);
    r.w4[2] = planes_or_null(n.gateup);
    r.w4[3] = planes_or_null(n.down);
  }
  return r;
}

// y = epilogue(x [M, K] · W [N, K]^T): the element-type GEMM, with w4 the NF4 GEMM over its planes, or with w8 the activation quantizer
// (into q8 [M, K], s [M]) and the FP8 GEMM
static int linear(const void* x, int ldx, const void* W, const srgpt_fp8* w8, const srgpt_nf4* w4, void* q8, float* s, void* y, int ldy, int M,
                  int N, int K, const void* residual, int ldr, int epilogue, void* stream) {
  if (w4 != nullptr) return srgpt_gemm_nf4_bf16(x, ldx, w4, y, ldy, M, N, K, residual, ldr, epilogue, stream);
  if (w8 == nullptr) return srgpt_gemm_bf16(x, ldx, W, K, y, ldy, M, N, K, nullptr, residual, ldr, 0, epilogue, 0, stream);
  SRGPT_TRY(srgpt_fp8_quantize_act_bf16(x, ldx, M, K, q8, K, s, stream));
  return srgpt_gemm_fp8_bf16(q8, K, s, w8->q, K, w8->scale, y, ldy, M, N, K, residual, ldr, epilogue, stream);
}

static int prefill_layers(void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_fp8* layers8, const srgpt_llama_layer_nf4* layers4, int n_layers, void* ws_h,
                          void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_s, int S, int H, int n_heads, int n_kv_heads,
                          int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_table,
                          int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride, void* stream) {
  SRGPT_CHECK_ARG(x && (layers || layers8) && ws_h && ws_qkv && ws_attn && ws_act && n_layers >= 0 && S > 0 && H > 0 && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && I > 0);
  SRGPT_CHECK_ARG(layers8 == nullptr || (ws_q8 && ws_s));
  const bool packed = cu_seqlens != nullptr;
  SRGPT_CHECK_ARG(packed ? (n_seqs >= 1 && max_seqlen >= 1 && max_seqlen <= S && page_table_stride > 0) : (n_seqs == 1));
  const int qd = n_heads * head_dim, kd = n_kv_heads * head_dim, nqkv = qd + 2 * kd;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const LayerRef w = layer_ref(layers, layers8, l, layers4);
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.in_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(ws_h, H, w.w[0], w.w8[0], w.w4[0], ws_q8, ws_s, ws_qkv, nqkv, S, nqkv, H, nullptr, 0, SRGPT_EPI_NONE, stream));
    if (packed) {
      SRGPT_TRY(srgpt_rope_kv_append_varlen_bf16(ws_qkv, S, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, start_pos, w.kv_pages, page_table, page_table_stride,
                                                 page_size, n_seqs, cu_seqlens, stream));
      SRGPT_TRY(srgpt_attention_prefill_varlen_bf16(ws_qkv, cptr(ws_qkv, (size_t)qd * 2), cptr(ws_qkv, (size_t)(qd + kd) * 2), ws_attn, nqkv, nqkv, qd, n_seqs,
                                                    cu_seqlens, max_seqlen, S, n_heads, n_kv_heads, head_dim, scale, 1, stream));
    } else {
      SRGPT_TRY(srgpt_rope_kv_append_bf16(ws_qkv, S, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, start_pos, w.kv_pages, page_table, page_size, stream));
      SRGPT_TRY(srgpt_attention_prefill_bf16(ws_qkv, cptr(ws_qkv, (size_t)qd * 2), cptr(ws_qkv, (size_t)(qd + kd) * 2), ws_attn, nqkv, nqkv, qd, 1, S, n_heads,
                                             n_kv_heads, head_dim, scale, 1, stream));
    }
    SRGPT_TRY(linear(ws_attn, qd, w.w[1], w.w8[1], w.w4[1], ws_q8, ws_s, x, H, S, H, qd, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.post_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(ws_h, H, w.w[2], w.w8[2], w.w4[2], ws_q8, ws_s, ws_act, I, S, 2 * I, H, nullptr, 0, SRGPT_EPI_SWIGLU, stream));
    SRGPT_TRY(linear(ws_act, I, w.w[3], w.w8[3], w.w4[3], ws_q8, ws_s, x, H, S, H, I, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_bf16(void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                                                                        void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads,
                                                                                        int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
                                                                                        const int* start_pos, const int* page_table, int page_size, int n_seqs, const int* cu_seqlens,
                                                                                        int max_seqlen, int page_table_stride, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(x, layers, nullptr, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab,
                        sin_tab, start_pos, page_table, page_size, n_seqs, cu_seqlens, max_seqlen, page_table_stride, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_fp8_bf16(
    void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_scale, int S,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_table,
    int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_layers(x, nullptr, layers, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, ws_q8, ws_scale, S, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab,
                        sin_tab, start_pos, page_table, page_size, n_seqs, cu_seqlens, max_seqlen, page_table_stride, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_layers_nf4_bf16(
    void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
    void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
    const int* start_pos, const int* page_table, int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride,
    void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr && nf4 != nullptr);
  return prefill_layers(x, layers, nullptr, nf4, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                        cos_tab, sin_tab, start_pos, page_table, page_size, n_seqs, cu_seqlens, max_seqlen, page_table_stride, stream);
}

static int prefill_chunk_layers(void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_fp8* layers8, const srgpt_llama_layer_nf4* layers4,
                                int n_layers, void* ws_h,
                                void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_s, int S, int H, int n_heads, int n_kv_heads,
                                int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables,
                                int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows, void* stream) {
  SRGPT_CHECK_ARG(x && (layers || layers8) && ws_h && ws_qkv && ws_attn && ws_act && n_layers >= 0 && S > 0 && H > 0 && n_heads > 0 && n_kv_heads > 0 && head_dim > 0 && I > 0);
  SRGPT_CHECK_ARG(layers8 == nullptr || (ws_q8 && ws_s));
  SRGPT_CHECK_ARG(start_pos && page_tables && cu_seqlens && n_seqs >= 1 && max_rows >= 1 && max_rows <= S && page_table_stride > 0 && n_pages > 0);
  const int qd = n_heads * head_dim, kd = n_kv_heads * head_dim, nqkv = qd + 2 * kd;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const LayerRef w = layer_ref(layers, layers8, l, layers4);
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.in_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(ws_h, H, w.w[0], w.w8[0], w.w4[0], ws_q8, ws_s, ws_qkv, nqkv, S, nqkv, H, nullptr, 0, SRGPT_EPI_NONE, stream));
    SRGPT_TRY(srgpt_rope_kv_append_varlen_bf16(ws_qkv, S, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, start_pos, w.kv_pages, page_tables, page_table_stride,
                                               page_size, n_seqs, cu_seqlens, stream));
    SRGPT_TRY(srgpt_attention_prefill_paged_bf16(ws_qkv, nqkv, ws_attn, qd, w.kv_pages, n_pages, page_tables, page_table_stride, page_size, start_pos, cu_seqlens,
                                                 n_seqs, max_rows, S, n_heads, n_kv_heads, head_dim, scale, stream));
    SRGPT_TRY(linear(ws_attn, qd, w.w[1], w.w8[1], w.w4[1], ws_q8, ws_s, x, H, S, H, qd, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
    SRGPT_TRY(srgpt_rmsnorm_bf16(x, H, w.post_norm, ws_h, H, S, H, eps, stream));
    SRGPT_TRY(linear(ws_h, H, w.w[2], w.w8[2], w.w4[2], ws_q8, ws_s, ws_act, I, S, 2 * I, H, nullptr, 0, SRGPT_EPI_SWIGLU, stream));
    SRGPT_TRY(linear(ws_act, I, w.w[3], w.w8[3], w.w4[3], ws_q8, ws_s, x, H, S, H, I, x, H, SRGPT_EPI_BIAS_RESIDUAL, stream));
  }
  return SRGPT_OK;
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_bf16(
    void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, int S, int H, int n_heads,
    int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables,
    int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_chunk_layers(x, layers, nullptr, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                              cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_fp8_bf16(
    void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, void* ws_q8, float* ws_scale, int S,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
    const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows, void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr);
  return prefill_chunk_layers(x, nullptr, layers, nullptr, n_layers, ws_h, ws_qkv, ws_attn, ws_act, ws_q8, ws_scale, S, H, n_heads, n_kv_heads, head_dim, I, eps,
                              cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_prefill_chunk_layers_nf4_bf16(
    void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
    void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
    const int* start_pos, const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs, const int* cu_seqlens, int max_rows,
    void* stream) {
  SRGPT_CHECK_ARG(layers != nullptr && nf4 != nullptr);
  return prefill_chunk_layers(x, layers, nullptr, nf4, n_layers, ws_h, ws_qkv, ws_attn, ws_act, nullptr, nullptr, S, H, n_heads, n_kv_heads, head_dim,
                              I, eps, cos_tab, sin_tab, start_pos, page_tables, page_table_stride, page_size, n_pages, n_seqs, cu_seqlens, max_rows,
                              stream);
}

// one decode GEMV over the NF4 planes when there are some (nf->q != NULL), else over the packed matrix when there is one (pk->sm != NULL),
// else over the plain weight W [N, K]
static int gemv_either(const void* x, const void* W, const srgpt_packed12* pk, const srgpt_nf4* nf, void* y, int N, int K, const void* norm_weight,
                       float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                       const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream) {
  if (nf != nullptr && nf->q != nullptr)
    return srgpt_gemv_nf4_bf16(x, nf, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                               page_table, page_size, stream);
  if (pk != nullptr && pk->sm != nullptr)
    return srgpt_gemv_packed_bf16(x, pk, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages,
                                  page_table, page_size, stream);
  return srgpt_gemv_bf16(x, W, K, y, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, kv_pages, page_table,
                         page_size, stream);
}

static int decode_step(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                       const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size, const void* final_norm,
                       const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out,
                       long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(h && layers && q_buf && attn_buf && act_buf && pos && page_table && final_norm && lm_head && lm_workspace && out_ids && step);
  const int qd = n_heads * head_dim, nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const srgpt_llama_layer_weights& w = layers[l];
    const srgpt_llama_layer_packed* pk = packed != nullptr ? &packed[l] : nullptr;
    const srgpt_llama_layer_nf4* nf = nf4 != nullptr ? &nf4[l] : nullptr;
    SRGPT_TRY(gemv_either(h, w.qkv_w, pk ? &pk->qkv : nullptr, nf ? &nf->qkv : nullptr, q_buf, nqkv, H, w.in_norm, eps, nullptr, SRGPT_GEMV_QKV_ROPE,
                          n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos, w.kv_pages, page_table, page_size, stream));
    SRGPT_TRY(srgpt_attention_decode_bf16(q_buf, attn_buf, w.kv_pages, page_table, page_size, pos, n_heads, n_kv_heads, head_dim, scale, stream));
    SRGPT_TRY(gemv_either(attn_buf, w.o_w, pk ? &pk->o : nullptr, nf ? &nf->o : nullptr, h, H, qd, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr,
                          nullptr, nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(gemv_either(h, w.gateup_w, pk ? &pk->gateup : nullptr, nf ? &nf->gateup : nullptr, act_buf, 2 * I, H, w.post_norm, eps, nullptr,
                          SRGPT_GEMV_SWIGLU, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(gemv_either(act_buf, w.down_w, pk ? &pk->down : nullptr, nf ? &nf->down : nullptr, h, H, I, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0,
                          nullptr, nullptr, nullptr, nullptr, nullptr, 0, stream));
  }
  if (lm_packed != nullptr && lm_packed->sm != nullptr)
    return srgpt_lm_head_argmax_packed_bf16(h, lm_packed, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
  return srgpt_lm_head_argmax_bf16(h, lm_head, H, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_bf16(void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf,
                                                                                     void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                                                                     const void* cos_tab, const void* sin_tab, int* pos, const int* page_table,
                                                                                     int page_size, const void* final_norm, const void* lm_head, int V,
                                                                                     const void* embed_table, void* lm_workspace, float* logits_out,
                                                                                     long long* out_ids, int* step, void* stream) {
  return decode_step(h, layers, nullptr, nullptr, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, nullptr, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_packed_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
    int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table,
    int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
    float* logits_out, long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(packed != nullptr);
  return decode_step(h, layers, packed, nullptr, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_nf4_bf16(
    void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H,
    int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
    const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out,
    long long* out_ids, int* step, void* stream) {
  SRGPT_CHECK_ARG(nf4 != nullptr);
  return decode_step(h, layers, nullptr, nf4, n_layers, q_buf, attn_buf, act_buf, H, n_heads, n_kv_heads, head_dim, I, eps, cos_tab, sin_tab, pos,
                     page_table, page_size, final_norm, lm_head, lm_packed, V, embed_table, lm_workspace, logits_out, out_ids, step, stream);
}

extern "C" __attribute__((visibility("default"))) int srgpt_llama_decode_step_fp8_bf16(
    void* h, const srgpt_llama_layer_fp8* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads,
    int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size, const void* final_norm,
    const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out, long long* out_ids,
    int* step, void* stream) {
  SRGPT_CHECK_ARG(h && layers && q_buf && attn_buf && act_buf && pos && page_table && final_norm && lm_head && lm_workspace && out_ids && step);
  const int qd = n_heads * head_dim, nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
  const float scale = 1.0f / sqrtf((float)head_dim);
  for (int l = 0; l < n_layers; ++l) {
    const srgpt_llama_layer_fp8& w = layers[l];
    SRGPT_TRY(srgpt_gemv_fp8_bf16(h, &w.qkv, q_buf, nqkv, H, w.in_norm, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads, n_kv_heads, head_dim, cos_tab,
                                  sin_tab, pos, w.kv_pages, page_table, page_size, stream));
    SRGPT_TRY(srgpt_attention_decode_bf16(q_buf, attn_buf, w.kv_pages, page_table, page_size, pos, n_heads, n_kv_heads, head_dim, scale, stream));
    SRGPT_TRY(srgpt_gemv_fp8_bf16(attn_buf, &w.o, h, H, qd, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr,
                                  0, stream));
    SRGPT_TRY(srgpt_gemv_fp8_bf16(h, &w.gateup, act_buf, 2 * I, H, w.post_norm, eps, nullptr, SRGPT_GEMV_SWIGLU, 0, 0, 0, nullptr, nullptr,
                                  nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(srgpt_gemv_fp8_bf16(act_buf, &w.down, h, H, I, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr,
                                  0, stream));
  }
  if (lm_packed != nullptr && lm_packed->sm != nullptr)
    return srgpt_lm_head_argmax_packed_bf16(h, lm_packed, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
  return srgpt_lm_head_argmax_bf16(h, lm_head, H, V, H, final_norm, eps, logits_out, lm_workspace, embed_table, h, out_ids, step, pos, stream);
}

// ---- verify pass of prompt-lookup speculative decoding: T tokens through the layer stack, every weight streamed once -----------
static int gemv_multi_either(const void* x, int ldx, const void* W, const srgpt_packed12* pk, const srgpt_nf4* nf, void* y, int ldy, int T, int N,
                             int K, const void* norm_weight, float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim,
                             const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size,
                             void* stream) {
  if (nf != nullptr && nf->q != nullptr)
    return srgpt_gemv_multi_nf4_bf16(x, ldx, nf, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab,
                                     pos, kv_pages, page_table, page_size, stream);
  if (pk != nullptr && pk->sm != nullptr)
    return srgpt_gemv_multi_packed_bf16(x, ldx, pk, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab,
                                        pos, kv_pages, page_table, page_size, stream);
  return srgpt_gemv_multi_bf16(x, ldx, W, K, y, ldy, T, N, K, norm_weight, eps, residual, mode, n_heads, n_kv_heads, head_dim, cos_tab, sin_tab, pos,
                               kv_pages, page_table, page_size, stream);
}

static int verify_step(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, const srgpt_llama_layer_nf4* nf4,
                       int n_layers, void* q_buf,
                       void* attn_buf, void* act_buf, int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab,
                       const void* sin_tab, int* pos, int* pos_rows, const int* page_table, int page_size, const void* final_norm,
                       const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                       float* logits_rows, float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram, int* draft_ids, long long* out_ids,
                       int out_cap, int* step, int* state, void* stream) {
  SRGPT_CHECK_ARG(h && layers && q_buf && attn_buf && act_buf && pos && pos_rows && page_table && final_norm && lm_head && lm_workspace && out_ids &&
                  step && state && draft_ids);
  SRGPT_CHECK_ARG(logits_all == nullptr || logits_rows != nullptr);
  const int qd = n_heads * head_dim, nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
  const float scale = 1.0f / sqrtf((float)head_dim);
  SRGPT_TRY(srgpt_spec_draft(prompt_ids, prompt_len, out_ids, step, pos, pos_rows, T, ngram, embed_table, h, H, draft_ids, state, stream));
  for (int l = 0; l < n_layers; ++l) {
    const srgpt_llama_layer_weights& w = layers[l];
    const srgpt_llama_layer_packed* pk = packed != nullptr ? &packed[l] : nullptr;
    const srgpt_llama_layer_nf4* nf = nf4 != nullptr ? &nf4[l] : nullptr;
    SRGPT_TRY(gemv_multi_either(h, H, w.qkv_w, pk ? &pk->qkv : nullptr, nf ? &nf->qkv : nullptr, q_buf, qd, T, nqkv, H, w.in_norm, eps, nullptr, SRGPT_GEMV_QKV_ROPE, n_heads,
                                n_kv_heads, head_dim, cos_tab, sin_tab, pos, w.kv_pages, page_table, page_size, stream));
    SRGPT_TRY(srgpt_attention_decode_multi_bf16(q_buf, qd, attn_buf, qd, w.kv_pages, page_table, page_size, pos_rows, T, n_heads, n_kv_heads, head_dim,
                                                scale, stream));
    SRGPT_TRY(gemv_multi_either(attn_buf, qd, w.o_w, pk ? &pk->o : nullptr, nf ? &nf->o : nullptr, h, H, T, H, qd, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr, nullptr,
                                nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(gemv_multi_either(h, H, w.gateup_w, pk ? &pk->gateup : nullptr, nf ? &nf->gateup : nullptr, act_buf, I, T, 2 * I, H, w.post_norm, eps, nullptr, SRGPT_GEMV_SWIGLU, 0, 0,
                                0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, stream));
    SRGPT_TRY(gemv_multi_either(act_buf, I, w.down_w, pk ? &pk->down : nullptr, nf ? &nf->down : nullptr, h, H, T, H, I, nullptr, 0.f, h, SRGPT_GEMV_PLAIN, 0, 0, 0, nullptr,
                                nullptr, nullptr, nullptr, nullptr, 0, stream));
  }
  if (lm_packed != nullptr && lm_packed->sm != nullptr)
    SRGPT_TRY(srgpt_lm_head_multi_packed_bf16(h, H, lm_packed, T, V, H, final_norm, eps, logits_rows, lm_workspace, stream));
  else
    SRGPT_TRY(srgpt_lm_head_multi_bf16(h, H, lm_head, H, T, V, H, final_norm, eps, logits_rows, lm_workspace, stream));
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
