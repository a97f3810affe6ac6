/* srgpt_b200 — C-ABI of the H100 (sm_90a) kernels behind SpatialRGPT's multimodal generate() path.
 *
 * The reference (AnjieCheng/SpatialRGPT) has no FFI / plugin layer: every op below replaces a
 * PyTorch library call on the path  LlavaLlamaModel.generate -> prepare_inputs_labels_for_multimodal
 * -> llm.generate  (llava/model/language_model/llava_llama.py:194-213).  Each entry cites the
 * reference call site it replaces (paths relative to the reference checkout;
 * "modeling_llama.py" = llava/train/transformers_replace/models/llama/modeling_llama.py).
 *
 * Conventions
 *   - plain C: device pointers as void*, sizes as int / long long, CUDA stream as void* (cudaStream_t).
 *   - all tensors are row-major; strides (ld*) are in ELEMENTS.
 *   - element type: the library is built twice from the same sources.  libsrgpt_b200.so computes in bfloat16 (the dtype the
 *     reference's eval scripts load the model in, llava/eval/eval_spatial.py:206-212); libsrgpt_b200_f16.so (-DSRGPT_ELEM_F16) in
 *     IEEE half, the reference loader's default (llava/model/builder.py:62, llava/eval/eval_region_cls.py:316-317).  Both export the
 *     SAME entry points: in the names and comments below "bf16" stands for "the 16-bit element type of the build" - __nv_bfloat16
 *     or __half - and srgpt_elem_type() says which.  Accumulation is fp32 and the rounding points are identical in both builds.
 *   - every function is asynchronous on `stream`, allocates nothing, and returns 0 on success or a
 *     negative srgpt error code; the message is available from srgpt_last_error().  Nothing throws.
 *   - callable from any host thread; no global state except the last-error string (thread-local).
 */
#ifndef SRGPT_B200_H_
#define SRGPT_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define SRGPT_ABI_VERSION 1

/* ---- library -------------------------------------------------------------------------------- */
int srgpt_abi_version(void);
/* 0 = bfloat16 build, 1 = IEEE half build (see "element type" above). */
int srgpt_elem_type(void);
const char* srgpt_last_error(void);
/* sm count + compute capability of the current device; fails (<0) unless it is sm_90. */
int srgpt_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* Optional in-kernel timeline for the decode-step kernels (debug / profiling aid; nsys is not available on
 * the target boxes).  Between trace_begin and trace_end every traced launch (gemv / lm_head / decode attention)
 * takes the next 4-u64 record of device_buf: {min CTA-start ns, min after-dependency-wait ns, max CTA-end ns,
 * CTA count} from %globaltimer.  The caller pre-fills records with {~0, ~0, 0, 0}.  trace_end returns the
 * number of records used.  Not thread-safe; launches captured into a CUDA graph keep their record. */
int srgpt_trace_begin(void* device_buf, int capacity_records);
int srgpt_trace_end(void);

/* ---- dense GEMM on the Hopper tensor cores (gemm_wgmma.cu: TMA + wgmma) ----------------------
 * C[M,N] = epilogue(A[M,K] · W[N,K]^T), bf16 in, fp32 accumulate.  W is the nn.Linear weight as
 * stored ([out, in]).  Replaces every F.linear / Conv2d(k=s) / ConvTranspose2d(k=s) on the path:
 * SigLIP q/k/v/out/fc1/fc2 (HF SiglipVisionModel, call site vision_encoder.py:119-130),
 * deconv refinement (base_extractor.py:92-97), rgb/depth projectors (base_extractor.py:158),
 * mm_projector (base_projector.py:76-79), Llama q/k/v/o/gate/up/down at prefill
 * (modeling_llama.py:429-431,498,221). */
enum {
  SRGPT_EPI_NONE = 0,           /* C = acc                                                        */
  SRGPT_EPI_BIAS = 1,           /* C = acc + bias[n]                                              */
  SRGPT_EPI_BIAS_GELU_TANH = 2, /* C = gelu_tanh(bf16(acc + bias))   (SigLIP fc1)                 */
  SRGPT_EPI_BIAS_GELU_ERF = 3,  /* C = gelu_erf(bf16(acc + bias))    (deconv #2, mm_projector)    */
  SRGPT_EPI_BIAS_RESIDUAL = 4,  /* C = bf16(acc + bias) + residual[row (% res_row_mod), n]        */
  SRGPT_EPI_SWIGLU = 5,         /* W rows interleaved (gate_i, up_i): C[:, i] = silu(g) * u; C has N/2 cols */
  SRGPT_EPI_BIAS_QUICK_GELU = 6 /* C = x * sigmoid(1.702 x), x = bf16(acc + bias)   (CLIP fc1, HF QuickGELUActivation) */
};
/* Optional workspace of the short-prompt ("tall stream-K") configuration: M <= 384 rows, all rows in one CTA, the (n-tile,
 * k-block) units balanced over the SMs, split tiles combined through fp32 partials in this buffer.  The caller owns the memory
 * (no hidden allocation): srgpt_gemm_workspace_bytes() bytes, 1024-byte aligned, ZEROED when registered, used by one stream at a
 * time, alive until unregistered with (NULL, 0).  Without a workspace short prompts run on the default 128-row tiles. */
long long srgpt_gemm_workspace_bytes(void);
int srgpt_gemm_set_workspace(void* workspace, long long bytes);
int srgpt_gemm_bf16(const void* A, int lda, const void* W, int ldw, void* C, int ldc, int M, int N, int K,
                    const void* bias /*bf16[N] or NULL*/, const void* residual /*bf16 or NULL*/, int ldr,
                    int res_row_mod /*0 = none*/, int epilogue, int out_fp32, void* stream);

/* ---- row-wise normalisation / elementwise (rowops.cu) ----------------------------------------
 * LayerNorm over the last dim, fp32 statistics, bf16 in/out.  act: 0 none, 1 GELU(erf) applied to
 * the bf16-rounded LN output.  Replaces nn.LayerNorm in SigLIP (eps 1e-6) and LayerNorm2d + GELU
 * (base_extractor.py:12-24,93-95; our activations are pixel-major so LN2d is a row LayerNorm). */
int srgpt_layernorm_bf16(const void* x, int ldx, const void* weight, const void* bias, void* y, int ldy, int rows,
                         int cols, float eps, int act, void* stream);
/* mm_projector front end (base_projector.py:32-52,75): DownSampleBlock (zero-pad side->even,
 * 2x2 token merge, the reference's transposed output order) fused with LayerNorm(4C).
 * x: [n_img, side*side, C] -> y: [n_img, ceil(side/2)^2, 4C]. */
int srgpt_downsample_layernorm_bf16(const void* x, const void* weight, const void* bias, void* y, int n_img, int side,
                                    int C, float eps, void* stream);
/* LlamaRMSNorm (modeling_llama.py:70-75): y = weight * bf16(x * rsqrt(mean(x^2) + eps)). */
int srgpt_rmsnorm_bf16(const void* x, int ldx, const void* weight, void* y, int ldy, int rows, int cols, float eps,
                       void* stream);
/* SigLIP patch embedding front end: Conv2d(3, D, k=14, s=14) == GEMM over this im2col
 * (HF SiglipVisionEmbeddings; call site siglip_encoder.py:11-16).  images: [n, 3, R, R] fp32 or
 * bf16 (src_is_bf16) -> A: [n*(R/ps)^2, ldk] bf16, column = c*ps*ps + ky*ps + kx, zero padded to ldk. */
int srgpt_patchify_bf16(const void* images, int src_is_bf16, void* A, int n, int R, int ps, int ldk, void* stream);
/* CLIP embeddings (HF CLIPVisionEmbeddings.forward; call site clip_encoder.py:11): out [n_img, T + 1, D] =
 * cat([class_embedding, patch_embeds[n]]) + position_embedding, one element-type add per value like torch's. */
int srgpt_clip_embed_bf16(const void* patch_embeds, const void* class_embedding, const void* position_embedding, void* out,
                          int n_img, int T, int D, void* stream);
/* Embedding splice (llava_arch.py:434-539): out[r,:] = src[src_id[r]][src_row[r],:] for the four
 * sources (0 = token embedding table, 1 = image features, 2 = mask embeds, 3 = depth embeds).
 * The (src_id,src_row) plan is built on the host from input_ids. */
int srgpt_splice_rows_bf16(const void* src0, const void* src1, const void* src2, const void* src3, const int* src_id,
                           const int* src_row, void* out, int rows, int cols, void* stream);

/* ---- region extractor HBM kernels (region.cu) -------------------------------------------------
 * MaskPooling weights (base_extractor.py:52-72): bilinear (align_corners=False, no antialias)
 * resample of masks [n_img, M, IH, IW] to the feature grid (side x side), cast to bf16, divide by
 * bf16(sum + 1e-8).  w: [n_img, M, side*side] bf16 (the reference's `mask / denorm`) in the feature
 * tensor's row order: order = 0 row-major (y*side+x); order = 2 the 2-level 2x2-nested order the deconv
 * GEMMs produce (see DESIGN.md "hres layout").  rscale = (float)(1.0 / scale_factor) exactly as ATen
 * computes it.  workspace: srgpt_mask_weights_workspace(n_img, M, side) bytes. */
long long srgpt_mask_weights_workspace(int n_img, int M, int side);
/* Layout of w (here and in srgpt_mask_pool_bf16): [n_img, M, ld] bf16 with ld = L rounded up to a multiple of 8 elements (16-byte
 * rows for the TMA view of the pooling kernel; L = side^2 is odd for odd sides); the pad elements are never read. */
int srgpt_mask_weights(const void* masks, int mask_is_bf16, void* w, void* workspace, int n_img, int M, int IH, int IW,
                       int side, float rscale, int order, void* stream);
/* Mask pooling proper (base_extractor.py:74-78): out[i,m,:] = sum_l w[i,m,l] * x[i,l,:] — bf16 tensor-core
 * product with fp32 accumulation like the reference's einsum.  x: [n_img, L, C] bf16 streamed once;
 * workspace: fp32 partials, srgpt_mask_pool_workspace() bytes. */
long long srgpt_mask_pool_workspace(int n_img, int M, int L, int C);
int srgpt_mask_pool_bf16(const void* x, const void* w, void* out, void* workspace, int n_img, int M, int L, int C,
                         void* stream);
/* AdaptiveAvgPool2d(out_side) over the (side x side) feature map (base_extractor.py:123,145).
 * x: [n_img, side*side, C] in `order` (as above) -> y: [n_img, out_side*out_side, C] row-major. */
int srgpt_adaptive_avgpool_bf16(const void* x, void* y, int n_img, int side, int out_side, int C, int order,
                                void* stream);
/* Row permutation between the nested order and row-major (tests / API parity for `hres`). */
int srgpt_reorder_rows_bf16(const void* x, void* y, int n_img, int side, int C, int from_order, int to_order,
                            void* stream);
/* Depth map preparation (llava/eval/eval_spatial.py:99-105): bilinear resize of depth [h, w] fp32 to
 * (H, W), min-max normalise * 255, truncate to u8, replicate to 3 channels -> out [H, W, 3] u8.
 * workspace: (H*W + 2) floats. */
int srgpt_depth_to_u8x3(const void* depth, int h, int w, void* out, int H, int W, void* workspace, void* stream);

/* ---- attention (attention.cu) ------------------------------------------------------------------
 * Prefill attention, softmax in fp32, flash-style (no S x S matrix in HBM).  head_dim 72 / 128
 * run on TMA + wgmma (attention_wgmma.cu), head_dim 64 on mma.sync tiles.
 * Replaces SigLIP's eager attention (non-causal, head_dim 72) and flash_attn_func(causal=True) with
 * GQA (modeling_llama.py:564-566).  q/k/v/out rows are tokens; head h of a row starts at h*head_dim.
 * Sequences are `batch` equal-length segments of `seqlen` consecutive rows. */
int srgpt_attention_prefill_bf16(const void* q, const void* k, const void* v, void* out, int q_ld, int kv_ld, int o_ld,
                                 int batch, int seqlen, int n_heads, int n_kv_heads, int head_dim, float scale,
                                 int causal, void* stream);
/* Same, for `n_seqs` variable-length sequences packed back to back: sequence b owns rows
 * [cu_seqlens[b], cu_seqlens[b+1]) (device int32 [n_seqs+1]); max_seqlen bounds the grid, total_rows =
 * cu_seqlens[n_seqs] bounds the TMA views (host value).  This is the varlen form of modeling_llama.py:540-562
 * (flash_attn_varlen_func over unpadded rows). */
int srgpt_attention_prefill_varlen_bf16(const void* q, const void* k, const void* v, void* out, int q_ld, int kv_ld,
                                        int o_ld, int n_seqs, const int* cu_seqlens, int max_seqlen, int total_rows,
                                        int n_heads, int n_kv_heads, int head_dim, float scale, int causal, void* stream);
/* RoPE + KV-cache append for `rows` new tokens of one sequence (modeling_llama.py:448-456):
 * rotates q and k in place inside the fused qkv buffer [rows, (nh + 2*nkv)*hd] using the bf16
 * cos/sin tables [max_pos, hd/2], and writes k, v into the paged cache.
 * Cache layout: pages [n_pages, 2 (k,v), page_size, nkv, hd] bf16 for ONE layer; page_table[i] =
 * physical page of logical page i of this sequence.  start_pos: device int (position of row 0). */
int srgpt_rope_kv_append_bf16(void* qkv, int rows, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                              const void* sin_tab, const int* start_pos, void* kv_pages, const int* page_table,
                              int page_size, void* stream);
/* Packed-sequence form: row r belongs to sequence b with cu_seqlens[b] <= r < cu_seqlens[b+1], its position is
 * start_pos[b] + r - cu_seqlens[b], and its page table is page_tables + b * page_table_stride. */
int srgpt_rope_kv_append_varlen_bf16(void* qkv, int rows, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                                     const void* sin_tab, const int* start_pos, void* kv_pages, const int* page_tables,
                                     int page_table_stride, int page_size, int n_seqs, const int* cu_seqlens, void* stream);
/* Causal prefill attention of new prompt rows over the paged cache (attention_paged_wgmma.cu; chunked prefill).  Replaces
 * flash_attn_varlen_func over the past_key_value concatenation (modeling_llama.py:451-456,540-566).  n_seqs chunks are packed
 * back to back: chunk b owns rows [cu_seqlens[b], cu_seqlens[b+1]) of q / out, and its row r sits at position
 * start_pos[b] + r - cu_seqlens[b] (device int32 arrays).  Row r attends to positions 0 .. its own position of sequence b, whose
 * K/V are read from kv_pages [n_pages, 2, page_size, nkv, hd] (one layer) through page_tables + b * page_table_stride; the
 * chunk's own K/V must already be in the cache (srgpt_rope_kv_append_varlen_bf16 first).  q: the rotated q columns of the fused
 * qkv buffer, row stride q_ld.  max_rows = longest chunk, total_rows = cu_seqlens[n_seqs] (host values).  head_dim 128 and
 * page_size 16 only; n_heads % n_kv_heads == 0 (the query heads of a kv head are served by one pass over its pages). */
int srgpt_attention_prefill_paged_bf16(const void* q, int q_ld, void* out, int o_ld, const void* kv_pages, int n_pages,
                                       const int* page_tables, int page_table_stride, int page_size, const int* start_pos,
                                       const int* cu_seqlens, int n_seqs, int max_rows, int total_rows, int n_heads, int n_kv_heads,
                                       int head_dim, float scale, void* stream);
/* Causal attention probabilities (attention_probs.cu; HF eager attention's softmax(Q K^T * scale + causal mask) in fp32, cast to the
 * element type), the S x S matrix the kernels above never build.  q / k: the rotated q and k columns of n_seqs sequences packed back to
 * back (cu_seqlens device int32 [n_seqs + 1]; NULL: one sequence of max_seqlen rows), row strides q_ld / k_ld; query head h reads kv head
 * h / (n_heads / n_kv_heads).  Sequence b's probabilities go to out + b * seq_stride + h * head_stride, an out_rows x out_rows block with
 * row stride ld (elements), its local row / column i at row / column row_off[b] + i (device int32 [n_seqs]; NULL: 0).  Every entry of the
 * block is written: entries above the diagonal and at rows / columns outside the sequence are 0.  head_dim 128 only. */
int srgpt_attention_probs_bf16(const void* q, int q_ld, const void* k, int k_ld, int n_seqs, const int* cu_seqlens, int max_seqlen, int n_heads,
                               int n_kv_heads, int head_dim, float scale, void* out, long long seq_stride, long long head_stride, long long ld,
                               int out_rows, const int* row_off, void* stream);
/* The attention probabilities of one-token decode steps over the paged cache (attention_probs.cu; HF generate(output_attentions=True)'s
 * decode-step entries, eager attention: softmax(q K^T * scale) in fp32, cast to the element type), which the flash-decode kernels never
 * build.  Row r: rotated q at q + r * q_ld (n_heads * 128 wide), keys 0 .. pos[r] in kv_pages through page_tables + r * pt_stride, query
 * head h reading KV head h / (n_heads / n_kv_heads) (at most 8 query heads per KV head).  The logits are srgpt_attention_probs_bf16's
 * (fp32 dot products, times scale * log2(e), exp2f, fp32 sum).  Row r, head h goes to out + (*step + step_offset) * step_stride
 * + r * row_stride + h * head_stride, in generate()'s padded columns: prompt key p (p < n_prompt[r]) at column off[r] + p, generated key
 * n_prompt[r] + j at column T + j.  Every column of [0, min(T + pos[r] + 1 - n_prompt[r], n_cols)) is written (0 where no key lands) and
 * nothing past it.  step / pos / off / n_prompt: device int32, read at run time, so one captured graph serves every step.  ws: fp32
 * workspace of 2 * rows * n_heads * ceil(n_cols / 128) floats.  Two launches.  head_dim 128 only. */
int srgpt_attention_probs_decode_bf16(const void* q, int q_ld, const void* kv_pages, const int* page_tables, int pt_stride, int page_size,
                                      const int* pos, int rows, int n_heads, int n_kv_heads, int head_dim, float scale, const int* off,
                                      const int* n_prompt, int T, int n_cols, const int* step, int step_offset, void* out, long long step_stride,
                                      long long row_stride, long long head_stride, float* ws, void* stream);
/* Rows x [rows, H] (contiguous) -> dst + (*step + step_offset) * step_stride + r * row_stride (strides in elements; step device int32):
 * generate(output_hidden_states=True)'s per-step hidden rows, written by the store kernel of the probed prefill. */
int srgpt_store_step_rows_bf16(const void* x, int rows, int H, const int* step, int step_offset, void* dst, long long step_stride,
                               long long row_stride, void* stream);
/* flags[r] = 1 when rows r of a and b ([rows, row_bytes] bytes, rows contiguous) are bitwise equal, else 0 (rowops.cu).  The
 * prompt-prefix cache of generate(prefix_cache=True) compares a request's images / depths / masks with the previous ones. */
int srgpt_rows_equal(const void* a, const void* b, int rows, long long row_bytes, int* flags, void* stream);
/* Decode attention for ONE new token over the paged cache (replaces torch.cat of the cache +
 * flash_attn_func with q_len 1, modeling_llama.py:451-456,564).  q: [nh*hd] bf16 (already rotated),
 * kv_len_minus1: device int = position of the new token (its k/v are already in the cache). */
int srgpt_attention_decode_bf16(const void* q, void* out, const void* kv_pages, const int* page_table, int page_size,
                                const int* kv_len_minus1, int n_heads, int n_kv_heads, int head_dim, float scale,
                                void* stream);

/* ---- decode-time weight-streaming kernels (gemv.cu) -------------------------------------------
 * One token: y = W · x with W [N, K] bf16 streamed once from HBM (the decode roofline).
 *   norm_weight != NULL : x is first RMS-normalised (LlamaRMSNorm) inside the kernel.
 *   mode SRGPT_GEMV_PLAIN    : y[n] = bf16(acc) (+ residual[n])            (o_proj, down_proj)
 *   mode SRGPT_GEMV_SWIGLU   : W rows interleaved (gate_i, up_i); y[i] = silu(g)*u   (gate/up)
 *   mode SRGPT_GEMV_QKV_ROPE : W = fused [q;k;v]; rotates q,k at *pos with the cos/sin tables, writes
 *                              q to y [nh*hd] and appends k,v to the paged cache      (q/k/v_proj + RoPE)
 * Replaces modeling_llama.py:429-431,448-456,498,221 at q_len == 1. */
enum { SRGPT_GEMV_PLAIN = 0, SRGPT_GEMV_SWIGLU = 1, SRGPT_GEMV_QKV_ROPE = 2 };
int srgpt_gemv_bf16(const void* x, const void* W, int ldw, void* y, int N, int K, const void* norm_weight, float eps,
                    const void* residual, int mode,
                    /* QKV_ROPE only: */ int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                    const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size,
                    void* stream);
/* Final norm + lm_head + greedy argmax (modeling_llama.py:922,1044-1045 + HF greedy search):
 * logits = float(bf16(W · rmsnorm(x))); writes argmax (lowest index on ties) to out_ids[*step],
 * copies the chosen token's embedding row to next_x, then ++*step and ++*pos.
 * logits_out (fp32 [V]) may be NULL.  workspace: srgpt_lm_head_workspace(V) bytes. */
long long srgpt_lm_head_workspace(int V);
int srgpt_lm_head_argmax_bf16(const void* x, const void* W, int ldw, int V, int K, const void* norm_weight, float eps,
                              float* logits_out, void* workspace, const void* embed_table, void* next_x,
                              long long* out_ids, int* step, int* pos, void* stream);
/* ---- 12-bit lossless packing of decode weights (pack12.cu, gemv.cu; DESIGN.md §3) --------------------------------------
 * A bf16 matrix [N, K] (K a multiple of 1024) as the batch-1 decode GEMV streams it, 12 bits per weight instead of 16:
 * sm = sign << 7 | mantissa (1 byte per weight), ex = a 4-bit exponent code per weight against the row's base
 * (code 0 = exponent field 0, code c = base + c - 1), and a CSR list of the exceptions (nonzero exponents below the window,
 * stored with code 0): exc[row_ptr[r] .. row_ptr[r+1]) = column << 8 | exponent, sorted by column, at most 32 per row.
 * The byte order inside the planes follows the GEMV's lanes (pack12.cuh).  Defined for bfloat16 only: the IEEE-half build
 * exports the same functions and they return SRGPT_ERR_UNSUPPORTED (-3). */
typedef struct {
  const void* sm;            /* [N, K] bytes */
  const void* ex;            /* [N, K / 2] bytes */
  const unsigned char* base; /* [N] */
  const int* row_ptr;        /* [N + 1] */
  const int* exc;            /* [row_ptr[N]] (a valid pointer even when empty) */
} srgpt_packed12;
/* Load time, step 1: per row base[r] and the number of exceptions n_exc[r]; *n_bad += the rows holding Inf or NaN (such a
 * matrix must stay plain bf16).  Step 2 (the caller has decided to pack and built row_ptr from n_exc): write the planes. */
int srgpt_pack12_scan_bf16(const void* W, int ldw, int N, int K, unsigned char* base, int* n_exc, int* n_bad, void* stream);
int srgpt_pack12_bf16(const void* W, int ldw, int N, int K, const unsigned char* base, const int* row_ptr, void* sm, void* ex, int* exc,
                      void* stream);
/* The inverse (W [N, ldw] bf16), through the GEMV's own decoder: the round-trip check of a packed matrix. */
int srgpt_unpack12_bf16(const srgpt_packed12* packed, int N, int K, void* W, int ldw, void* stream);
/* srgpt_gemv_bf16 / srgpt_lm_head_argmax_bf16 over a packed matrix (`packed` is a host pointer; the arrays it names are on
 * the device).  Every lane sees the same fp32 weights in the same order as the plain kernel, so the results are bit-identical. */
int srgpt_gemv_packed_bf16(const void* x, const srgpt_packed12* packed, void* y, int N, int K, const void* norm_weight, float eps,
                           const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                           const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream);
int srgpt_lm_head_argmax_packed_bf16(const void* x, const srgpt_packed12* packed, int V, int K, const void* norm_weight, float eps,
                                     float* logits_out, void* workspace, const void* embed_table, void* next_x, long long* out_ids,
                                     int* step, int* pos, void* stream);
/* ---- NF4 weight-only quantization of the decoder-layer matrices (nf4.cu, gemv.cu; DESIGN.md §3) ------------------------
 * Stands for the reference's load_pretrained_model(load_4bit=True) (llava/model/builder.py:51-60): bitsandbytes NF4 codes,
 * blocksize 64, double-quantized absmax, applied to the LLM only (llava/model/llava_arch.py:99-101).  A weight's value is
 * round_to_elem(fl32(code[q] * scale)), dequantized to the element type before the multiply as bitsandbytes' Linear4bit does.
 * Computed in the build's element type: bfloat16 in libsrgpt_b200.so, IEEE half in libsrgpt_b200_f16.so (the loader's default).
 * The decode GEMV's planes (nf4.cuh): q [N, K / 2] codes in the GEMV's lane order (K a multiple of 1024), scale [N, K / 64]
 * fp32 resolved scales in natural order. */
typedef struct {
  const unsigned char* q; /* [N, K / 2] */
  const float* scale;     /* [N, K / 64] */
} srgpt_nf4;
/* Load time, step 1 (one original [N, K] matrix, K a multiple of 64): codes [N, K / 2] in natural order (weight 2j in the high
 * nibble of byte j) chosen against the exact fp32 absmax [N, K / 64] of each block of 64; *n_bad += the blocks holding Inf or NaN. */
int srgpt_nf4_quantize_bf16(const void* W, int ldw, int N, int K, unsigned char* codes, float* absmax, int* n_bad, void* stream);
/* Step 2, double quantization of the n absmax values of one matrix: *offset = their mean (fp64 sum in index order, rounded to
 * fp32), blocks of 256 of (absmax - offset) to the nearest entry of the 256-value signed dynamic map dyn_map, and
 * scale[i] = fl32(map[c] * absmax2) + offset, the scale the weights are dequantized with. */
int srgpt_nf4_double_quant(const float* absmax, long long n, const float* dyn_map, float* offset, float* scale, void* stream);
/* Natural-order codes + scales -> the element-type matrix W [N, ldw] (the resident dequantized copy). */
int srgpt_nf4_dequantize_bf16(const unsigned char* codes, const float* scale, int N, int K, void* W, int ldw, void* stream);
/* Natural-order codes [N, K / 2] -> the GEMV's lane order (K a multiple of 1024); run on a fused matrix. */
int srgpt_nf4_lane_order(const unsigned char* codes, int N, int K, unsigned char* q, void* stream);
/* The lane-ordered planes -> W [N, ldw], through the GEMV's own dequantization: the round-trip check of the planes. */
int srgpt_nf4_unpack_bf16(const srgpt_nf4* nf4, int N, int K, void* W, int ldw, void* stream);
/* srgpt_gemv_bf16 (PLAIN + residual, SWIGLU + RMSNorm, QKV_ROPE + KV append) streaming the NF4 planes: bit-identical to
 * srgpt_gemv_bf16 over the dequantized matrix.  `nf4` is a host pointer; K a multiple of 1024. */
int srgpt_gemv_nf4_bf16(const void* x, const srgpt_nf4* nf4, void* y, int N, int K, const void* norm_weight, float eps, const void* residual,
                        int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos,
                        void* kv_pages, const int* page_table, int page_size, void* stream);
/* srgpt_gemm_bf16 (epilogue SRGPT_EPI_NONE, SRGPT_EPI_BIAS_RESIDUAL without bias, or SRGPT_EPI_SWIGLU) with the weight W [N, K] read from
 * the decode GEMV's NF4 planes `w` (a host pointer; K a multiple of 1024): the producer warpgroup dequantizes each B tile into shared
 * memory.  Tiles, tile order, stream-K and its workspace are chosen as for a 16-bit [N, K] matrix, so the result is bit-identical to
 * srgpt_gemm_bf16 over the dequantized matrix. */
int srgpt_gemm_nf4_bf16(const void* A, int lda, const srgpt_nf4* w, void* C, int ldc, int M, int N, int K, const void* residual, int ldr,
                        int epilogue, void* stream);
/* Plain argmax over fp32 rows (first index on ties), e.g. first token after prefill. */
int srgpt_argmax_f32(const float* x, int rows, int cols, long long* out, void* stream);
/* Same over bf16 rows [rows, ldx] (the bf16-rounded logits of a batched lm_head GEMM, modeling_llama.py:1044). */
int srgpt_argmax_bf16(const void* x, int ldx, int rows, int cols, long long* out, void* stream);
/* Beam-search candidates (rowops.cu): replaces log_softmax + the [num_beams x vocab] torch.topk of HF GenerationMixin.beam_search
 * (transformers 4.37.2; reached from llava_llama.py:212 when the eval scripts pass --num_beams > 1).  logits: [n_beams, ldx] in the
 * element type (the rounded lm_head output, modeling_llama.py:1044-1045).  Per row the n_cand best
 * (log_softmax(logits.float())[token] + beam_scores[row], token) in (score desc, token asc) order -> cand_scores / cand_tokens
 * [n_beams, n_cand] (token -1 / score -inf when a row has fewer finite logits). */
int srgpt_beam_candidates_bf16(const void* logits, int ldx, int n_beams, int V, const float* beam_scores, int n_cand,
                               float* cand_scores, int* cand_tokens, void* stream);
/* The same candidates and, when logprobs is given, every row's whole log_softmax (fp32, before the beam score is added) -> logprobs
 * [n_beams, ldo], ldo >= V: HF's output_scores of a beam step (next_token_scores_processed). */
int srgpt_beam_candidates_scores_bf16(const void* logits, int ldx, int n_beams, int V, const float* beam_scores, int n_cand,
                                      float* cand_scores, int* cand_tokens, float* logprobs, long long ldo, void* stream);
/* Diverse beam search's candidates (rowops.cu): per row the n_cand best (log_softmax(logits.float())[token] + beam_scores[row], token) in
 * (score desc, token asc) order of that fp32 score, which the rounding of + beam_scores can make differ from the logit order ->
 * cand_scores / cand_tokens [n_beams, n_cand], and the row's (max, log-sum-exp) of the rounded logits -> stats [n_beams][2] (8-byte
 * aligned), from which log_softmax[token] = (logit - max) - lse. */
int srgpt_beam_candidates_scored_bf16(const void* logits, int ldx, int n_beams, int V, const float* beam_scores, int n_cand,
                                      float* cand_scores, int* cand_tokens, float* stats, void* stream);
/* Score rows of a decode step (rowops.cu): HF's output_scores of a greedy step.  Row r of rows [R, ld] (fp32 when rows_f32, else the
 * element type widened exactly, as .float()) -> scores + (*step + step_offset) * step_stride + r * row_stride, for r < R.  The index is
 * read at run time, so one captured decode graph writes every step's rows.  R <= 65535, ld >= V, row_stride >= V. */
int srgpt_step_scores(const void* rows, int rows_f32, long long ld, int R, int V, const int* step, int step_offset, float* scores,
                      long long step_stride, long long row_stride, void* stream);
/* Beam search over a batch of prompts (beam.cu): merges the candidates srgpt_beam_candidates_bf16 wrote for n_groups * k rows (prompt g
 * owns rows g*k .. g*k+k-1).  Per prompt the n_cand best (score, beam within the prompt, token) in (score desc, beam asc, token asc)
 * order, candidates with token < 0 dropped -> out_scores / out_beams / out_tokens [n_groups, n_cand] (score -inf, beam and token -1 where a
 * prompt has fewer valid candidates).  One CTA per prompt; k * n_cand <= 4096. */
int srgpt_beam_select(const float* cand_scores, const int* cand_tokens, int n_groups, int k, int n_cand, float* out_scores, int* out_beams,
                      int* out_tokens, void* stream);
/* Diverse beam search over a batch of prompts (beam.cu; HF group_beam_search with HammingDiversityLogitsProcessor, transformers 4.37.2):
 * prompt p owns rows p*k .. p*k+k-1, group g of it the gs = k / n_groups rows p*k + g*gs ..  One CTA per prompt takes the groups in
 * order.  Each token of group g's rows scores fl(fl(logp - fl(diversity_penalty * c)) + beam_scores[row]), c = how often groups 0 .. g-1
 * of the prompt chose it in this step and logp = (logit - max) - lse from stats; the candidates are the L tokens per row that
 * srgpt_beam_candidates_scored_bf16 wrote (cand_tokens [rows, L]) and the earlier groups' choices, which is exact for L >= n_cand + k - gs.
 * The group's n_cand best (score, beam within the group, token) in (score desc, beam asc, token asc) order -> out_* [n_prompts,
 * n_groups, n_cand] (-inf / -1 / -1 past the valid ones); BeamSearchScorer.process's choice (EOS candidates closing no beam here) ->
 * next_beams (the parent, a beam within the prompt) and next_tokens [n_prompts * k], -1 where a group runs out of non-EOS candidates.  A
 * group with done[p * n_groups + g] != 0 writes no candidates and gives each of its beams parent g*gs and token pad_id.  Chosen and pad
 * tokens both count for the later groups.  k <= 64, n_cand <= 512, V <= 2^26, gs * (L + k - gs) <= 4096. */
int srgpt_beam_group_select(const void* logits, int ldx, int V, const float* stats, const float* beam_scores, const int* cand_tokens, int L,
                            int n_prompts, int k, int n_groups, int n_cand, const int* eos, int n_eos, int pad_id, float diversity_penalty,
                            const int* done, float* out_scores, int* out_beams, int* out_tokens, int* next_beams, int* next_tokens,
                            void* stream);
/* Bytes of the workspace srgpt_kv_copy_pages needs for n_staged pairs (-1 on invalid arguments). */
long long srgpt_kv_copy_workspace_bytes(int n_staged, int n_layers, int page_rows, int row_bytes);
/* Copies rows of KV pages for K and V of every layer (beam.cu).  pages: [n_layers, n_pages, 2 (K, V), page_rows, row_bytes] bytes, the
 * paged cache of the Llama decoder.  pairs: device int[n_pairs][4] = (src page, dst page, first row, rows); a pair outside the cache or
 * the page is skipped.  The first n_staged pairs are staged through the workspace: one pass copies them there and every other pair
 * straight to its destination, a second pass (a second launch, only when n_staged > 0) writes the staged ones.  So a pair whose
 * destination is another pair's source must be staged; then any permutation is safe.  row_bytes a multiple of 16. */
int srgpt_kv_copy_pages(void* pages, int n_layers, int n_pages, int page_rows, int row_bytes, const int* pairs, int n_pairs, int n_staged,
                        void* workspace, long long workspace_bytes, void* stream);
/* Row log-softmax at target tokens (logprob.cu): replaces the .float() + CrossEntropyLoss of LlamaForCausalLM.forward
 * (modeling_llama.py:1044-1058) and the per-token log-probabilities of likelihood scoring.  logits: [rows, ld] in the element type (the
 * rounded lm_head output), ld >= V.  lse[rows] (fp32) = m + log sum exp(x - m) over each row, every element widened to fp32 exactly; a NaN
 * in a row makes its lse NaN.  n pairs (pair_rows[i], pair_targets[i]) given in HOST memory: logprob[i] (fp32, device) = logits[row, target]
 * - lse[row], 0 for target -100 (ignored).  loss (device float, optional) = the mean of -logprob over the pairs that are not ignored, NaN
 * when every pair is.  A row outside [0, rows) or a target outside [0, V) that is not -100 is rejected (-1) before anything is read or
 * launched.  workspace: device memory of at least 8 n bytes, 8-byte aligned.  Fixed reduction orders: repeated calls are bit-identical. */
int srgpt_token_logprobs(const void* logits, long long ld, int rows, int V, const int* pair_rows, const long long* pair_targets, int n,
                         void* workspace, long long workspace_bytes, float* lse, float* logprob, float* loss, void* stream);
/* Temperature + nucleus (top-p) sampling of one token from fp32 logits [V] (sampling.cu): replaces HF's TemperatureLogitsWarper /
 * TopKLogitsWarper / TopPLogitsWarper / multinomial behind do_sample=True (llava/eval/eval_spatial.py:231-236, llava/eval/model_vqa.py:72-78).
 * params = device float[3] {temperature, top_p, top_k (0 = off)}; seed = device u64; the draw is a counter-based generator of
 * (*seed, *step + step_offset) - both read at run time, so a captured decode graph serves every request.
 * Writes out_ids[*step + step_offset] and, when given, next_x[K] = embed_table[token].  Call it right after
 * srgpt_lm_head_argmax_bf16 / srgpt_llama_decode_step_bf16 (which advanced *step) with step_offset = -1. */
int srgpt_sample_top_p_f32(const float* logits, int V, const float* params, const unsigned long long* seed, const int* step, int step_offset,
                           long long* out_ids, const void* embed_table, void* next_x, int K, void* stream);
/* The same draw for R rows in one launch (sampling.cu, one 1024-thread CTA per row): logits [R, ld], fp32 (logits_f32 = 1) or the element
 * type (the rows of the batched lm_head GEMM).  Row r draws with seeds[r] (device u64[R]) at counter *step + step_offset and writes
 * ids[r] (int64); no embedding row is written (srgpt_decode_batch_advance does that).  Row r's token equals what srgpt_sample_top_p_f32
 * draws from that row converted to fp32 with seed seeds[r] and the same counter.  R <= 65535, ld >= V. */
int srgpt_sample_rows(const void* logits, int logits_f32, int ld, int R, int V, const float* params, const unsigned long long* seeds,
                      const int* step, int step_offset, long long* ids, void* stream);
/* srgpt_sample_top_p_f32 / srgpt_sample_rows, and the warped row each draw picks from (HF's output_scores of a sampled step):
 * logits / temperature (an IEEE fp32 division) for every token the top-k cut and the nucleus keep, -inf for every other token.  The
 * draws are those of the calls without scores.  The one-row form writes scores + (*step + step_offset) * step_stride (step_stride >= V);
 * the R-row form writes row r to scores + (*step + step_offset) * step_stride + r * V (step_stride >= R * V). */
int srgpt_sample_top_p_scores_f32(const float* logits, int V, const float* params, const unsigned long long* seed, const int* step,
                                  int step_offset, long long* out_ids, const void* embed_table, void* next_x, int K, float* scores,
                                  long long step_stride, void* stream);
int srgpt_sample_rows_scores(const void* logits, int logits_f32, int ld, int R, int V, const float* params, const unsigned long long* seeds,
                             const int* step, int step_offset, long long* ids, float* scores, long long step_stride, void* stream);
/* The four entry points above with HF's TypicalLogitsWarper, EpsilonLogitsWarper and EtaLogitsWarper after top-p, in HF's order, each on
 * the set the earlier cuts kept (sampling.cu): params = device float[6] {temperature, top_p, top_k (0 = off), typical_p, epsilon_cutoff,
 * eta_cutoff}.  Typical acts when typical_p < 1, epsilon when 0 < epsilon_cutoff < 1, eta when 0 < eta_cutoff < 1; epsilon and eta keep
 * the tokens tied at the largest logit of what typical kept.  The draw uses the same counter stream, over the final kept set, and the
 * warped row is -inf outside it.  With all three off, ids and rows equal those of the float[3] entry points. */
int srgpt_sample_warped_f32(const float* logits, int V, const float* params, const unsigned long long* seed, const int* step, int step_offset,
                            long long* out_ids, const void* embed_table, void* next_x, int K, void* stream);
int srgpt_sample_warped_scores_f32(const float* logits, int V, const float* params, const unsigned long long* seed, const int* step,
                                   int step_offset, long long* out_ids, const void* embed_table, void* next_x, int K, float* scores,
                                   long long step_stride, void* stream);
int srgpt_sample_rows_warped(const void* logits, int logits_f32, int ld, int R, int V, const float* params, const unsigned long long* seeds,
                             const int* step, int step_offset, long long* ids, void* stream);
int srgpt_sample_rows_warped_scores(const void* logits, int logits_f32, int ld, int R, int V, const float* params,
                                    const unsigned long long* seeds, const int* step, int step_offset, long long* ids, float* scores,
                                    long long step_stride, void* stream);
/* HF's logits processors on the device (logits_process.cu): replaces RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor,
 * NoBadWordsLogitsProcessor, MinLengthLogitsProcessor and MinNewTokensLengthLogitsProcessor (transformers generation/logits_process.py),
 * which HF runs on the host behind generate(repetition_penalty=, no_repeat_ngram_size=, bad_words_ids=, min_length=, min_new_tokens=)
 * (llava/model/language_model/llava_llama.py:212 forwards them; llava/eval/model_vqa.py:76), plus the greedy arg max after them.
 * logits: rows [rows, ld], fp32 (logits_f32 = 1) or the element type.  Row r's history is hist[r * hist_row_stride + t * hist_tok_stride]
 * for t < min(*step + step_offset, hist_cap) (step NULL: step_offset alone).  fparams = device float[2] {penalty, 1 / penalty};
 * spec = device int[spec_cap] {flags (1 penalty, 2 n-gram, 4 bad words, 8 minimum length), n-gram size, minimum new tokens, n_eos,
 * n_bad, eos ids[n_eos], bad-word offsets[n_bad + 1], bad-word tokens[]} - both read at run time, so a captured graph serves every
 * setting.  Writes the processed fp32 rows to out [rows, ldo] (may be NULL) and, when ids is given, the arg max of each processed
 * row to ids[rows] (lowest index on ties, NaN never wins). */
int srgpt_logits_process(const void* logits, int logits_f32, int ld, int rows, int V, const long long* hist, int hist_row_stride,
                         int hist_tok_stride, int hist_cap, const int* step, int step_offset, const float* fparams, const int* spec,
                         int spec_cap, float* out, int ldo, long long* ids, void* stream);
/* out_ids[*step + step_offset] = ids[0] and, when given, next_x[K] = embed_table[ids[0]]: the processed greedy choice replaces the one
 * srgpt_lm_head_argmax_bf16 / srgpt_llama_decode_step_bf16 wrote (call with step_offset = -1, as srgpt_sample_top_p_f32). */
int srgpt_logits_pick_token(const long long* ids, const int* step, int step_offset, long long* out_ids, const void* embed_table,
                            void* next_x, int K, void* stream);

/* ---- host preprocessing on the GPU (preprocess.cu; llava/mm_utils.py:421-542: process_images / process_regions) ----------
 * The pinned image processor (transformers 4.37.2 SiglipImageProcessor) = Pillow BICUBIC resize of the uint8 image + rescale +
 * normalise; masks = cv2 INTER_NEAREST.  Pillow's resampler is integer arithmetic over host-built coefficient tables
 * (spatialrgpt_b200/preprocess.py, same double arithmetic as libImaging/Resample.c), so the results are bit-exact. */
int srgpt_resample_u8(const void* in, void* out, int H, int W, int C, int axis, int out_size, const int* kk, const int* bounds, int ksize,
                      void* stream);
/* mean3 / std3: HOST arrays of 3 floats (passed by value to the kernel) */
int srgpt_u8_to_normalized_chw(const void* in, float* out, int H, int W, int C, double scale, const float* mean3, const float* std3,
                               int do_normalize, void* stream);
int srgpt_resize_nearest_u8(const void* in, float* out, int H, int W, int Hout, int Wout, const int* ys, const int* xs, void* stream);

/* ---- batched decode (B sequences, one new token each; llava_arch.py:549-611 pads, modeling_llama.py:540-562 un-pads: here
 * the rows are never padded).  The projections are srgpt_gemm_bf16 over the B rows (tall stream-K configuration: every weight is
 * streamed once for the whole batch), RoPE / KV append is srgpt_rope_kv_append_varlen_bf16 with one row per sequence. */
int srgpt_attention_decode_batched_bf16(const void* q, int q_ld, void* out, int o_ld, const void* kv_pages, const int* page_tables,
                                        int pt_stride, int page_size, const int* kv_len_minus1, int batch, int n_heads, int n_kv_heads,
                                        int head_dim, float scale, void* stream);
/* ids [B] (the step's arg max per sequence) -> out_ids[*step * B + b], h[b, :] = embed_table[ids[b], :], ++pos[b], ++*step. */
int srgpt_decode_batch_advance(const long long* ids, const void* embed_table, void* h, int H, long long* out_ids, int* step, int* pos,
                               int B, void* ticket, void* stream);

/* ---- tensor-parallel decode (SURVEY.md §8e "optional TP", BASELINE config c5; no reference counterpart, parity = TP-1) ----------
 * Megatron-style sharding of the Llama decoder over `world` ranks: column-parallel fused QKV (a rank owns n_heads/world query
 * heads and their kv heads) and gate/up, row-parallel o_proj / down_proj whose fp32 partial sums are all-reduced, vocabulary-
 * parallel lm_head with an (value, index) all-gather.  The KV cache keeps the FULL layout on every rank (a rank only ever reads
 * and writes its own kv heads), so prefill stays the replicated path. */
int srgpt_gemv_tp_bf16(const void* x, const void* W, int ldw, void* y, int N, int K, const void* norm_weight, float eps, int mode,
                       int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages,
                       const int* page_table, int page_size, int kv_heads_total, int kv_head_off, float* partial_f32, void* stream);
int srgpt_attention_decode_tp_bf16(const void* q, void* out, const void* kv_pages, const int* page_table, int page_size,
                                   const int* kv_len_minus1, int n_heads_local, int group, int n_kv_total, int kv_head_off, int head_dim,
                                   float scale, void* stream);
/* h[n] = bf16(bf16(partial[n]) + h[n]) after the all-reduce of the row-parallel partial sums (modeling_llama.py:668,682). */
int srgpt_tp_residual_add_bf16(void* h, const float* partial, int n, void* stream);
/* rows [index_base, index_base + V_local) of lm_head: best = device int[2] {best bf16-rounded logit (float bits), GLOBAL index}. */
int srgpt_lm_head_local_best_bf16(const void* x, const void* W_local, int ldw, int V_local, int K, const void* norm_weight, float eps,
                                  void* workspace, int index_base, int* best, void* stream);
/* best_all = the all-gathered int[world][2]; writes out_ids[*step], next_x = embed_table[token], ++*step, ++*pos. */
int srgpt_tp_pick_token(const int* best_all, int world, const void* embed_table, void* next_x, int K, long long* out_ids, int* step,
                        int* pos, void* stream);

/* Fused collectives over NVLink peer memory (tp_comm.cu): every rank's partial sums / arg-max candidates live in a SYMMETRIC buffer
 * (srgpt_tp_comm_bytes bytes, zeroed, same layout on every GPU, peer-mapped by the caller - torch symmetric memory); one kernel
 * signals the peers, waits for all of them, pulls their 16 KB partials through NVLink, reduces in rank order and applies the residual
 * add (or picks the token).  peer_bases = HOST array [world] of peer-mapped base addresses; idx < 128 numbers the collectives of a
 * step; epoch / step are device ints (request counter, the decoder's step counter), so CUDA-graph replays need no host values. */
long long srgpt_tp_comm_bytes(int world, int n_slots, int slot_floats);
long long srgpt_tp_comm_slot_offset(int world, int slot, int slot_floats);
int srgpt_tp_allreduce_residual_bf16(const unsigned long long* peer_bases, int rank, int world, long long slot_off_bytes, int idx,
                                     const int* epoch, const int* step, void* h, int n, void* stream);
int srgpt_tp_allgather_pick_token(const unsigned long long* peer_bases, int rank, int world, long long slot_off_bytes, int idx,
                                  const int* epoch, const void* embed_table, void* next_x, int K, long long* out_ids, int* step, int* pos,
                                  void* stream);

/* ---- composite entry points (layers.cu): one call per tower pass / prompt / decode step -------------------
 * Pure sequencing of the kernels above on `stream` (no allocation, no sync); they exist because a Python-side
 * launch costs more host time than several of these kernels take on the device.  Weights are the re-laid-out
 * tensors described in DESIGN.md §3 (fused qkv, interleaved gate/up).  Workspaces (bf16): ws_h [M, D|H],
 * ws_qkv [M, 3D | (nh+2nkv)hd], ws_attn [M, D | nh*hd], ws_mlp [M, I] / ws_act [S, I]. */
typedef struct {
  const void *ln1_w, *ln1_b, *qkv_w, *qkv_b, *out_w, *out_b, *ln2_w, *ln2_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
} srgpt_siglip_layer_weights;
typedef struct {
  const void *in_norm, *qkv_w, *o_w, *post_norm, *gateup_w, *down_w;
  void* kv_pages; /* this layer's KV pages [n_pages, 2, page_size, nkv, hd] */
} srgpt_llama_layer_weights;
/* n_layers SigLIP encoder layers in place on x [n_img*T, D] (HF SiglipEncoderLayer; call site vision_encoder.py:119-130). */
int srgpt_siglip_layers_bf16(void* x, const srgpt_siglip_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                             void* ws_attn, void* ws_mlp, int n_img, int T, int D, int heads, int I, float eps, void* stream);
/* The same pre-LN encoder layer with the MLP activation as a parameter (fc1_epilogue = SRGPT_EPI_BIAS_GELU_TANH: SigLIP,
 * SRGPT_EPI_BIAS_QUICK_GELU: CLIP (HF CLIPEncoderLayer; call site clip_encoder.py:11, vision_encoder.py:119-130),
 * SRGPT_EPI_BIAS_GELU_ERF: hidden_act "gelu").  T counts ALL rows of an image (CLIP: patches + the class token). */
int srgpt_vit_layers_bf16(void* x, const srgpt_siglip_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
                          void* ws_mlp, int n_img, int T, int D, int heads, int I, float eps, int fc1_epilogue, void* stream);
/* n_layers Llama decoder layers over the prompt rows x [S, H] in place, appending K/V to the paged cache
 * (LlamaDecoderLayer.forward, modeling_llama.py:623-684).  n_seqs == 1, cu_seqlens == NULL: one prompt of S rows.
 * Otherwise S is the total row count of n_seqs prompts packed back to back (cu_seqlens int32 [n_seqs+1] on the
 * device, max_seqlen = longest prompt, start_pos [n_seqs], page_tables [n_seqs, page_table_stride]): every GEMM
 * runs once over all S rows (batch 32 x 259 rows = the c3 workload), attention and the KV append per sequence. */
int srgpt_llama_prefill_layers_bf16(void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                    void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                    float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
                                    const int* page_tables, int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen,
                                    int page_table_stride, void* stream);
/* Chunked prefill: the same layers over S new rows of n_seqs chunks packed back to back (cu_seqlens, start_pos [n_seqs] on the
 * device, max_rows = longest chunk) that continue sequences whose earlier positions are already in the cache.  The sequencing of
 * srgpt_llama_prefill_layers_bf16 with attention through srgpt_attention_prefill_paged_bf16 (n_pages = pages per layer). */
int srgpt_llama_prefill_chunk_layers_bf16(void* x, const srgpt_llama_layer_weights* layers, int n_layers, void* ws_h, void* ws_qkv,
                                          void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                          float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
                                          const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs,
                                          const int* cu_seqlens, int max_rows, void* stream);
/* One whole decode step (5 kernels per layer + lm_head + argmax), h [H] in/out = residual stream of the new token. */
int srgpt_llama_decode_step_bf16(void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf,
                                 void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                 const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
                                 const void* final_norm, const void* lm_head, int V, const void* embed_table, void* lm_workspace,
                                 float* logits_out, long long* out_ids, int* step, void* stream);
/* The same step streaming the packed matrices: packed[l].<matrix>.sm == NULL (a matrix kept plain) and lm_packed == NULL or
 * lm_packed->sm == NULL take the bf16 weight of `layers` / lm_head instead.  Bit-identical to srgpt_llama_decode_step_bf16. */
typedef struct {
  srgpt_packed12 qkv, o, gateup, down;
} srgpt_llama_layer_packed;
int srgpt_llama_decode_step_packed_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers,
                                        void* q_buf, void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                        float eps, const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
                                        const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
                                        const void* embed_table, void* lm_workspace, float* logits_out, long long* out_ids, int* step,
                                        void* stream);
/* The same step streaming NF4 layer matrices (the reference's load_4bit decode, llava/model/builder.py:51-60): nf4[l].<matrix>.q
 * == NULL (K not a multiple of 1024) takes the dequantized weight of `layers`; lm_head stays unquantized, streamed from lm_packed
 * when lm_packed->sm != NULL (bfloat16 build) and from lm_head otherwise.  Bit-identical to srgpt_llama_decode_step_bf16 over the
 * dequantized weights. */
typedef struct {
  srgpt_nf4 qkv, o, gateup, down;
} srgpt_llama_layer_nf4;
int srgpt_llama_decode_step_nf4_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf,
                                     void* attn_buf, void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                     const void* cos_tab, const void* sin_tab, int* pos, const int* page_table, int page_size,
                                     const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table,
                                     void* lm_workspace, float* logits_out, long long* out_ids, int* step, void* stream);
/* srgpt_llama_prefill_layers_bf16 / srgpt_llama_prefill_chunk_layers_bf16 with every matrix whose nf4[l].<matrix>.q != NULL taken by
 * srgpt_gemm_nf4_bf16 from its planes; the element-type pointer of `layers` is then unused and may be NULL.  Bit-identical to the
 * element-type stacks over the dequantized weights. */
int srgpt_llama_prefill_layers_nf4_bf16(void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* ws_h,
                                        void* ws_qkv, void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                        float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables,
                                        int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride, void* stream);
int srgpt_llama_prefill_chunk_layers_nf4_bf16(void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers,
                                              void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act, int S, int H, int n_heads, int n_kv_heads,
                                              int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
                                              const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs,
                                              const int* cu_seqlens, int max_rows, void* stream);

/* ---- FP8 (E4M3) W8A8 quantization of the decoder-layer linears (fp8.cu, gemm_wgmma.cu; DESIGN.md §3, §7) ---------------------------
 * Every row r of a weight W [N, K] (once, at load) and of an activation x [M, K] (before every linear) is quantized alike:
 * a = max_k |x[r, k]| (fp32), inv = 448 / a, scale[r] = a / 448 (both 1 when a == 0), q[r, k] = e4m3(fl32(x[r, k] * inv)), rounded to
 * nearest even and saturated to +-448 (cvt.rn.satfinite).  A linear is y[m, n] = acc[m, n] * (scale_x[m] * scale_w[n]) in fp32, acc the fp32
 * sum of the exact E4M3 products; the epilogue's rounding points follow.  K must be a multiple of 16. */
typedef struct {
  const void* q;       /* [N, K] E4M3 codes, row-major, K bytes per row */
  const float* scale;  /* [N] */
} srgpt_fp8;
/* *n_bad += 1 for every row holding Inf or NaN (such a matrix must not be used). */
int srgpt_fp8_quantize_weight_bf16(const void* W, int ldw, int N, int K, void* q, float* scale, int* n_bad, void* stream);
/* q [M, ldq] bytes (ldq a multiple of 16), scale [M] */
int srgpt_fp8_quantize_act_bf16(const void* x, int ldx, int M, int K, void* q, int ldq, float* scale, void* stream);
/* srgpt_gemm_bf16 over E4M3 operands: A [M, lda] and W [N, ldw] bytes with their row scales sx [M] and sw [N]; epilogue SRGPT_EPI_NONE,
 * SRGPT_EPI_BIAS_RESIDUAL (no bias) or SRGPT_EPI_SWIGLU; C in the element type.  Tiles, ring, tile order and stream-K as the 16-bit
 * kernel, with K blocks of 128 elements (wgmma m64n128k32 e4m3). */
int srgpt_gemm_fp8_bf16(const void* A, int lda, const float* sx, const void* W, int ldw, const float* sw, void* C, int ldc, int M, int N, int K,
                        const void* residual, int ldr, int epilogue, void* stream);
/* A decoder layer with FP8 linears (no element-type copy of its matrices). */
typedef struct {
  const void* in_norm;
  srgpt_fp8 qkv;     /* [(nh + 2 nkv) hd, H] */
  srgpt_fp8 o;       /* [H, nh hd] */
  const void* post_norm;
  srgpt_fp8 gateup;  /* [2 I, H], rows interleaved (gate_i, up_i) */
  srgpt_fp8 down;    /* [H, I] */
  void* kv_pages;
} srgpt_llama_layer_fp8;
/* srgpt_llama_prefill_layers_bf16 / srgpt_llama_prefill_chunk_layers_bf16 with every linear as activation quantizer + FP8 GEMM.
 * Extra workspaces: ws_q8 [S, max(H, nh hd, I)] bytes and ws_scale [S] fp32. */
int srgpt_llama_prefill_layers_fp8_bf16(void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
                                        void* ws_act, void* ws_q8, float* ws_scale, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                        float eps, const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables,
                                        int page_size, int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride, void* stream);
int srgpt_llama_prefill_chunk_layers_fp8_bf16(void* x, const srgpt_llama_layer_fp8* layers, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn,
                                              void* ws_act, void* ws_q8, float* ws_scale, int S, int H, int n_heads, int n_kv_heads, int head_dim,
                                              int I, float eps, const void* cos_tab, const void* sin_tab, const int* start_pos,
                                              const int* page_tables, int page_table_stride, int page_size, int n_pages, int n_seqs,
                                              const int* cu_seqlens, int max_rows, void* stream);
/* What srgpt_llama_prefill_layers_probe_bf16 records (forward(output_hidden_states=, output_attentions=)).  Outputs are padded per
 * sequence: sequence b's local row i is output row row_off[b] + i (device int32 [n_seqs]) of blocks of out_rows rows; strides in elements.
 * hidden != NULL: before layer l the residual rows x go to hidden + l * hidden_layer_stride + b * hidden_seq_stride + row * hidden_ld
 *   (slots 0 .. n_layers - 1: the embeddings, then the residual stream after each layer but the last).
 * attn != NULL: layer l's probabilities (srgpt_attention_probs_bf16 over the rotated q / k of ws_qkv) go to attn + l * attn_layer_stride,
 *   sequence b at + b * attn_seq_stride, head h at + h * attn_head_stride, rows attn_ld apart. */
typedef struct {
  void* hidden;
  long long hidden_layer_stride, hidden_seq_stride, hidden_ld;
  void* attn;
  long long attn_layer_stride, attn_seq_stride, attn_head_stride, attn_ld;
  int out_rows;
  const int* row_off;
} srgpt_prefill_probe;
/* srgpt_llama_prefill_layers_bf16 (or its _nf4 / _fp8 forms: fp8 != NULL takes the FP8 layers, else nf4 != NULL the NF4 planes beside the
 * element-type layers) with the probes of `probe` recorded; x, the KV cache and every bit of the arithmetic are those of the unprobed
 * call.  ws_q8 / ws_scale are needed with fp8 only. */
int srgpt_llama_prefill_layers_probe_bf16(void* x, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4,
                                          const srgpt_llama_layer_fp8* fp8, int n_layers, void* ws_h, void* ws_qkv, void* ws_attn, void* ws_act,
                                          void* ws_q8, float* ws_scale, int S, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                          const void* cos_tab, const void* sin_tab, const int* start_pos, const int* page_tables, int page_size,
                                          int n_seqs, const int* cu_seqlens, int max_seqlen, int page_table_stride,
                                          const srgpt_prefill_probe* probe, void* stream);
/* srgpt_gemv_bf16 over FP8 planes (fp8_gemv_kernel, gemv.cu), every mode: x (RMS-normalised first when norm_weight is given) is quantized
 * in the kernel by the activation definition above, the weight codes are turned into their element-type values exactly, and a row's sum
 * acc of exact products (fp32) becomes acc * fl32(s_x * scale[row]) before the mode's stores and rounding points.  `w` is a host pointer;
 * K a multiple of 16. */
int srgpt_gemv_fp8_bf16(const void* x, const srgpt_fp8* w, void* y, int N, int K, const void* norm_weight, float eps, const void* residual,
                        int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos,
                        void* kv_pages, const int* page_table, int page_size, void* stream);
/* One decode step over FP8 layers: srgpt_llama_decode_step_nf4_bf16's 5 kernels per layer with every layer matrix streamed by
 * srgpt_gemv_fp8_bf16, then lm_head + argmax (lm_packed may be NULL).  Buffers as srgpt_llama_decode_step_bf16's. */
int srgpt_llama_decode_step_fp8_bf16(void* h, const srgpt_llama_layer_fp8* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf,
                                     int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
                                     int* pos, const int* page_table, int page_size, const void* final_norm, const void* lm_head,
                                     const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace, float* logits_out,
                                     long long* out_ids, int* step, void* stream);
/* What srgpt_llama_decode_step_probe_bf16 records (generate(output_hidden_states=, output_attentions=) over the decode steps; strides in
 * elements; the step's slot is *step + step_offset, read before the lm_head advances step).
 * hidden != NULL: before layer l the residual row h goes to hidden + slot * hidden_step_stride + l * hidden_layer_stride (slot l), and
 *   srgpt_rmsnorm_bf16 of the last layer's row to slot n_layers; hidden_row_stride is the row stride of a batched caller (unused here).
 * attn != NULL: layer l's probabilities (srgpt_attention_probs_decode_bf16 with rows = 1, off / n_prompt / T / n_cols / ws) go to
 *   attn + l * attn_layer_stride with step / row / head strides attn_step_stride / attn_row_stride / attn_head_stride. */
typedef struct {
  void* hidden;
  long long hidden_step_stride, hidden_layer_stride, hidden_row_stride;
  void* attn;
  long long attn_step_stride, attn_layer_stride, attn_row_stride, attn_head_stride;
  int step_offset, T, n_cols;
  const int* off;
  const int* n_prompt;
  float* ws;
} srgpt_decode_probe;
/* srgpt_llama_decode_step_bf16 (or its _packed / _nf4 / _fp8 forms: the one of packed / nf4 / fp8 given, lm_packed may be NULL) with the
 * probes of `probe` recorded; h, pos, step, the KV cache, the ids and the logits are those of the unprobed call.  The final norm row
 * passes through act_buf, so I >= H when hidden is recorded. */
int srgpt_llama_decode_step_probe_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed,
                                       const srgpt_llama_layer_nf4* nf4, const srgpt_llama_layer_fp8* fp8, int n_layers, void* q_buf, void* attn_buf,
                                       void* act_buf, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab,
                                       const void* sin_tab, int* pos, const int* page_table, int page_size, const void* final_norm,
                                       const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                                       float* logits_out, long long* out_ids, int* step, const srgpt_decode_probe* probe, void* stream);

/* ---- prompt-lookup speculative decoding, batch 1, greedy (HF GenerationMixin._assisted_decoding with
 * PromptLookupCandidateGenerator, i.e. generate(prompt_lookup_num_tokens=k); call site llava_llama.py:212).
 * A verify pass runs T = k + 1 tokens at positions pos .. pos+T-1: row 0 is the last emitted token, rows 1..T-1 the drafts.
 * For every token t the kernels below do the fp32 operations of the one-token kernels at position pos+t in the same order, so
 * the accepted tokens and their logits are bit-identical to plain greedy decoding.  T is 1 .. SRGPT_SPEC_T_MAX. */
#define SRGPT_SPEC_T_MAX 8
/* srgpt_gemv_bf16 over T activation rows x [T, ldx] -> y [T, ldy] (residual, when given, has y's layout), each weight streamed
 * once for all rows.  QKV_ROPE: row t is rotated at and appends K/V at position *pos + t.  T = 1 is srgpt_gemv_bf16. */
int srgpt_gemv_multi_bf16(const void* x, int ldx, const void* W, int ldw, void* y, int ldy, int T, int N, int K, const void* norm_weight,
                          float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab,
                          const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream);
int srgpt_gemv_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, void* y, int ldy, int T, int N, int K,
                                 const void* norm_weight, float eps, const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim,
                                 const void* cos_tab, const void* sin_tab, const int* pos, void* kv_pages, const int* page_table, int page_size,
                                 void* stream);
/* srgpt_gemv_multi_bf16 streaming NF4 planes (a host pointer; K a multiple of 1024): bit-identical to it over the dequantized matrix. */
int srgpt_gemv_multi_nf4_bf16(const void* x, int ldx, const srgpt_nf4* nf4, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                              const void* residual, int mode, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab,
                              const int* pos, void* kv_pages, const int* page_table, int page_size, void* stream);
/* final norm + lm_head over T rows: fp32 logits [T, V] (optional) and per-(token, CTA) arg max partials in `workspace`
 * (T * srgpt_lm_head_workspace(V) bytes, token t's block at t * srgpt_lm_head_workspace(V)); srgpt_spec_accept reduces them. */
int srgpt_lm_head_multi_bf16(const void* x, int ldx, const void* W, int ldw, int T, int V, int K, const void* norm_weight, float eps,
                             float* logits_out, void* workspace, void* stream);
int srgpt_lm_head_multi_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, int T, int V, int K, const void* norm_weight, float eps,
                                    float* logits_out, void* workspace, void* stream);
/* Decode attention of T consecutive tokens of one sequence: token t (q row t, out row t) attends over kv rows 0 .. pos_rows[t]
 * (device int32 [T]).  The arithmetic of srgpt_attention_decode_bf16 per token. */
int srgpt_attention_decode_multi_bf16(const void* q, int q_ld, void* out, int o_ld, const void* kv_pages, const int* page_table, int page_size,
                                      const int* pos_rows, int T, int n_heads, int n_kv_heads, int head_dim, float scale, void* stream);
/* Start of a verify pass (one CTA): the drafts by n-gram lookup (PromptLookupCandidateGenerator.get_candidates: n-gram sizes from
 * ngram down to 1, the earliest match with a non-empty continuation, at most T-1 tokens) over the history prompt_ids[0..*prompt_len)
 * (a negative id is a sentinel that never matches) followed by out_ids[0..*step).  Writes draft_ids [T] (row 0 = the last emitted
 * token, missing drafts = -1), the embedding rows x [T, H], pos_rows[t] = *pos + t and state[3] = number of drafts. */
int srgpt_spec_draft(const int* prompt_ids, const int* prompt_len, const long long* out_ids, const int* step, const int* pos, int* pos_rows, int T, int ngram,
                     const void* embed_table, void* x, int H, int* draft_ids, int* state, void* stream);
/* End of a verify pass (one CTA): the T arg maxes (lowest index on ties), a = the number of leading drafts equal to the model's
 * choices, out_ids[*step .. *step + a] = the a + 1 new tokens, *step and *pos advance by a + 1.  state (int32 [8]): [0] passes,
 * [1] drafted, [2] accepted, [4] step before the pass, [5] tokens emitted, [6] step after.  logits_all != NULL: the accepted
 * rows of logits_rows [T, V] are copied to logits_all rows *step ...  Writes past out_cap are dropped. */
int srgpt_spec_accept(const void* workspace, int V, int T, const int* draft_ids, long long* out_ids, int out_cap, int* step, int* pos, int* state,
                      const float* logits_rows, float* logits_all, void* stream);
/* One whole verify pass: draft, 5 kernels per layer, lm_head, accept.  Buffers: h [T, H], q_buf / attn_buf [T, nh*hd], act_buf
 * [T, I], lm_workspace T * srgpt_lm_head_workspace(V) bytes, logits_rows [T, V] (needed when logits_all != NULL). */
int srgpt_llama_verify_step_bf16(void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int T,
                                 int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos,
                                 int* pos_rows, const int* page_table, int page_size, const void* final_norm, const void* lm_head, int V,
                                 const void* embed_table, void* lm_workspace, float* logits_rows, float* logits_all, const int* prompt_ids,
                                 const int* prompt_len, int ngram, int* draft_ids, long long* out_ids, int out_cap, int* step, int* state, void* stream);
int srgpt_llama_verify_step_packed_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers,
                                        void* q_buf, void* attn_buf, void* act_buf, int T, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                        float eps, const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows, const int* page_table,
                                        int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
                                        const void* embed_table, void* lm_workspace, float* logits_rows, float* logits_all, const int* prompt_ids,
                                        const int* prompt_len, int ngram, int* draft_ids, long long* out_ids, int out_cap, int* step, int* state, void* stream);
/* The verify pass streaming NF4 layer matrices: nf4[l].<matrix>.q != NULL takes srgpt_gemv_multi_nf4_bf16 (the element-type pointer of
 * `layers` may then be NULL), q == NULL the element-type matrix; lm_head as in srgpt_llama_decode_step_nf4_bf16. */
int srgpt_llama_verify_step_nf4_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf,
                                     void* attn_buf, void* act_buf, int T, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                     const void* cos_tab, const void* sin_tab, int* pos, int* pos_rows, const int* page_table, int page_size,
                                     const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table,
                                     void* lm_workspace, float* logits_rows, float* logits_all, const int* prompt_ids, const int* prompt_len, int ngram,
                                     int* draft_ids, long long* out_ids, int out_cap, int* step, int* state, void* stream);

/* ---- batch-invariant decoding: B <= SRGPT_SPEC_T_MAX sequences in one weight pass, each row with the arithmetic of its one-token step.
 * Row b is the newest token of the sequence at position pos_rows[b] (device int32 [B]) whose page table is page_tables + b * pt_stride,
 * so every sequence's ids and logits are bit-identical to decoding it alone with srgpt_llama_decode_step_*. */
/* srgpt_gemv_multi_bf16 in QKV_ROPE mode over rows of different sequences: row t is rotated at and appends K/V at position pos_rows[t]
 * through page_tables + t * pt_stride (pt_stride = 0: one page table, the verify pass).  Row t equals srgpt_gemv_bf16 at that position. */
int srgpt_gemv_rows_bf16(const void* x, int ldx, const void* W, int ldw, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                         int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows, void* kv_pages,
                         const int* page_tables, int pt_stride, int page_size, void* stream);
int srgpt_gemv_rows_packed_bf16(const void* x, int ldx, const srgpt_packed12* packed, void* y, int ldy, int T, int N, int K, const void* norm_weight,
                                float eps, int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows,
                                void* kv_pages, const int* page_tables, int pt_stride, int page_size, void* stream);
int srgpt_gemv_rows_nf4_bf16(const void* x, int ldx, const srgpt_nf4* nf4, void* y, int ldy, int T, int N, int K, const void* norm_weight, float eps,
                             int n_heads, int n_kv_heads, int head_dim, const void* cos_tab, const void* sin_tab, const int* pos_rows, void* kv_pages,
                             const int* page_tables, int pt_stride, int page_size, void* stream);
/* Decode attention of T rows: row t (q row t, out row t) attends over kv rows 0 .. pos_rows[t] of the page table page_tables + t * pt_stride.
 * The arithmetic of srgpt_attention_decode_bf16 per row.  srgpt_attention_decode_multi_bf16 is the pt_stride = 0 case. */
int srgpt_attention_decode_rows_bf16(const void* q, int q_ld, void* out, int o_ld, const void* kv_pages, const int* page_tables, int pt_stride,
                                     int page_size, const int* pos_rows, int T, int n_heads, int n_kv_heads, int head_dim, float scale, void* stream);
/* The end of a step of B rows (one CTA): row b's token is its arg max from the srgpt_lm_head_multi_* partials in `workspace` (lowest index
 * on ties, as srgpt_lm_head_argmax_bf16), or ids[b] when ids != NULL.  out_ids[*step * B + b] = the token, x row b (x [B, H]) = its
 * embedding row, ++pos_rows[b], then ++*step. */
int srgpt_rows_advance(const void* workspace, int V, const long long* ids, int B, const void* embed_table, void* x, int H, long long* out_ids, int* step,
                       int* pos_rows, void* stream);
/* One decode step of B sequences: 5 kernels per layer (srgpt_gemv_rows_*, srgpt_attention_decode_rows_bf16, srgpt_gemv_multi_* for o /
 * gate-up / down), lm_head over the B rows, then srgpt_rows_advance.  Sampled when seeds != NULL: row b draws from logits_rows row b with
 * seeds[b] at counter *step (srgpt_sample_rows into ids [B], one more kernel).  Buffers: h [B, H], q_buf / attn_buf [B, nh*hd], act_buf
 * [B, I], lm_workspace B * srgpt_lm_head_workspace(V) bytes, logits_rows fp32 [B, V] (optional when greedy).  pt_stride > 0.  The FP8
 * layer format has no form of this step. */
int srgpt_llama_decode_rows_bf16(void* h, const srgpt_llama_layer_weights* layers, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int B, int H,
                                 int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab, int* pos_rows,
                                 const int* page_tables, int pt_stride, int page_size, const void* final_norm, const void* lm_head, int V,
                                 const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params,
                                 const unsigned long long* seeds, long long* ids, long long* out_ids, int* step, void* stream);
int srgpt_llama_decode_rows_packed_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed, int n_layers,
                                        void* q_buf, void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads, int head_dim, int I,
                                        float eps, const void* cos_tab, const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride,
                                        int page_size, const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V,
                                        const void* embed_table, void* lm_workspace, float* logits_rows, const float* sample_params,
                                        const unsigned long long* seeds, long long* ids, long long* out_ids, int* step, void* stream);
int srgpt_llama_decode_rows_nf4_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf,
                                     void* attn_buf, void* act_buf, int B, int H, int n_heads, int n_kv_heads, int head_dim, int I, float eps,
                                     const void* cos_tab, const void* sin_tab, int* pos_rows, const int* page_tables, int pt_stride, int page_size,
                                     const void* final_norm, const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table,
                                     void* lm_workspace, float* logits_rows, const float* sample_params, const unsigned long long* seeds, long long* ids,
                                     long long* out_ids, int* step, void* stream);

/* ---- classifier-free guidance (guidance.cu): replaces HF UnbatchedClassifierFreeGuidanceLogitsProcessor (transformers
 * generation/logits_process.py), which GenerationMixin puts first among the logits processors behind generate(guidance_scale=,
 * negative_prompt_ids=) (call site llava_llama.py:212).  Prompt b decodes in row b of a rows step of 2P rows and its unconditional
 * branch (its negative prompt, then the tokens chosen for prompt b) in row P + b.
 * srgpt_guidance_rows: logits fp32 [2P, V] (the rows step's logits_rows), P <= SRGPT_SPEC_T_MAX / 2, scale = device float g.  Per pair:
 * s = log_softmax(row b), u = log_softmax(row P + b), each (x - m) - log(sum exp(x - m)) in fp32; guided row b [V] (fp32 [P, V], not
 * overlapping logits) = fl(fl(g * fl(s - u)) + u); logits and guided 16-byte aligned.  lse (optional, fp32 [2P][2]) = {m, log sum
 * exp(x - m)} of every row.  ids (optional, int64 [2P]): ids[b] = ids[P + b] = the arg max of guided row b (lowest index on ties, NaN never wins, 0 for an all-NaN row).  One
 * 512-thread CTA per pair, fixed reduction order. */
int srgpt_guidance_rows(const float* logits, int V, int P, const float* scale, float* guided, float* lse, long long* ids, void* stream);
/* ids[P + b] = ids[b] for b < P (a prompt's drawn token is its unconditional branch's next token). */
int srgpt_guidance_pair_ids(long long* ids, int P, void* stream);
typedef struct {
  const float* scale;  /* device float: g */
  float* guided_rows;  /* fp32 [B / 2, V]: the guided rows the choice is made from */
} srgpt_guidance;
/* srgpt_llama_decode_rows_* with guidance: B = 2P rows, row P + b the unconditional branch of row b.  After lm_head, srgpt_guidance_rows
 * over logits_rows (needed); greedy: its arg max goes to ids (needed) for both rows of a pair; sampled (seeds != NULL, seeds [P]):
 * srgpt_sample_rows draws row b from guided row b, then srgpt_guidance_pair_ids.  srgpt_rows_advance then takes ids for all B rows.
 * guidance == NULL is the step of the format's own entry point.  packed and nf4 select the weight format (at most one non-NULL;
 * lm_packed may be NULL); one more kernel than the unguided step when greedy, three more than the unguided sampled step's one.
 * One entry point for every format, running the same layer body (decode_rows in layers.cu) as the three above, rather than a new
 * argument on each of them: their argument lists stay as they are, so existing callers and bindings of the C ABI keep working. */
int srgpt_llama_decode_rows_guided_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed,
                                        const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int B, int H,
                                        int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
                                        int* pos_rows, const int* page_tables, int pt_stride, int page_size, const void* final_norm,
                                        const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                                        float* logits_rows, const float* sample_params, const unsigned long long* seeds, long long* ids,
                                        long long* out_ids, int* step, const srgpt_guidance* guidance, void* stream);
/* The sampled rows step, plain (guidance == NULL) or guided, drawing with srgpt_sample_rows_warped: warp_params = device float[6] as
 * there, seeds needed.  Arguments otherwise as srgpt_llama_decode_rows_guided_bf16; the same kernels, the warped sampler in place of
 * srgpt_sample_rows. */
int srgpt_llama_decode_rows_warped_bf16(void* h, const srgpt_llama_layer_weights* layers, const srgpt_llama_layer_packed* packed,
                                        const srgpt_llama_layer_nf4* nf4, int n_layers, void* q_buf, void* attn_buf, void* act_buf, int B, int H,
                                        int n_heads, int n_kv_heads, int head_dim, int I, float eps, const void* cos_tab, const void* sin_tab,
                                        int* pos_rows, const int* page_tables, int pt_stride, int page_size, const void* final_norm,
                                        const void* lm_head, const srgpt_packed12* lm_packed, int V, const void* embed_table, void* lm_workspace,
                                        float* logits_rows, const float* warp_params, const unsigned long long* seeds, long long* ids,
                                        long long* out_ids, int* step, const srgpt_guidance* guidance, void* stream);

/* ---- contrastive search (contrastive.cu, beam.cu): replaces _ranking_fast and the candidate bookkeeping of HF
 * GenerationMixin.contrastive_search (transformers 4.37.2 generation/utils.py), which generate() runs behind llava_llama.py:212 when
 * num_beams == 1, do_sample is false, penalty_alpha > 0 and top_k > 1.  B prompts x k candidates decode as rows g * k + i of the
 * batched step; every prompt keeps its context, the final-norm hidden rows of its positions so far (HF's last_hidden_states), in
 * ctx [B, L_cap, H] (element type); prompt g's context length is pos[g * k], the position its candidates are processed at.
 * srgpt_contrastive_partial_floats: the fp32 entries of the penalty's per-chunk maxima for (B, k, L_cap) (-1 on invalid arguments). */
long long srgpt_contrastive_partial_floats(int B, int k, int L_cap);
/* The degeneration penalty, first pass: cand [B * k, ldc] (the step's final-norm rows) against ctx[g, 0 .. pos[g * k]).  One CTA per
 * (32 context rows, prompt); each context row's norm and its dot products with the candidates (staged in shared memory, 8 at a time)
 * in one pass, fp32 accumulation.  partial [B, ceil(L_cap / 32), k] = each chunk's largest cosine per candidate (chunks past the
 * context are not written).  1 <= k <= 64, H % 8 == 0, H <= 12800. */
int srgpt_contrastive_penalty_bf16(const void* cand, int ldc, const void* ctx, int L_cap, int H, const int* pos, int B, int k, float* partial,
                                   void* stream);
/* The choice, one CTA per prompt g: pen[g * k + i] = the largest partial of candidate i over the chunks of the context (fixed order);
 * score = fl(fl(alpha[0] * exp(cand_scores)) - fl(alpha[1] * pen)) with alpha = device fp32 {1 - penalty_alpha, penalty_alpha};
 * cand_scores / cand_tokens [B * k] = srgpt_beam_candidates_bf16 over the next-logits rows with zero beam scores.  sel[g] = the
 * largest score's index (the lowest on ties; a token < 0 never wins).  Then out_ids[*step * B + g] = its token, ctx[g, L] = xn row
 * g * k + sel (when L < L_cap), next_logits[g] = logits row g * k + sel, pos[g * k + i] = L + 1 for every i, and the last CTA
 * advances *step.  ticket: one zeroed device uint, returned to zero. */
int srgpt_contrastive_select_bf16(const float* cand_scores, const int* cand_tokens, const float* partial, const float* alpha, const void* xn, int ldx,
                                  int H, const void* logits, int ldl, int V, void* ctx, int L_cap, void* next_logits, int ldn, int* pos, int B, int k,
                                  long long* out_ids, int* step, void* ticket, int* sel, float* pen, float* score, void* stream);
/* The KV broadcast of a contrastive step (beam.cu): for each prompt g, the K and V of every layer at position pos[g * k + sel[g]] +
 * pos_offset are copied from row g * k + sel[g] into the other k - 1 rows of the prompt, pages looked up in page_tables [rows, pt_stride]
 * (the cache's tables, row r = sequence r).  pages as srgpt_kv_copy_pages.  HF keeps the chosen candidate's cache; here the k rows'
 * histories stay identical, so one position per step is all that moves. */
int srgpt_kv_broadcast_rows(void* pages, int n_layers, int n_pages, int page_rows, int row_bytes, const int* page_tables, int pt_stride,
                            const int* pos, int pos_offset, const int* sel, int n_groups, int k, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SRGPT_B200_H_ */
