"""ctypes binding of libsrgpt_b200.so (the C-ABI declared in include/srgpt_b200.h).

There is deliberately NO fallback: if the shared library cannot be built/loaded, or a kernel
returns an error, a ``SrgptError`` is raised.  Nothing in this package computes on the CPU or
through torch operators on the product path.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

from . import _build

_lock = threading.Lock()
_libs = {}       # element type ("bf16" / "f16") -> typed CDLL
_elem = "bf16"   # element type whose library load() returns; switched by ops.elem_dtype() around a model's calls


class SrgptError(RuntimeError):
    pass


vp, ci, cf, cll = C.c_void_p, C.c_int, C.c_float, C.c_longlong

# name -> (restype, argtypes); mirrors include/srgpt_b200.h one to one
SIGNATURES = {
    "srgpt_abi_version": (ci, []),
    "srgpt_elem_type": (ci, []),
    "srgpt_last_error": (C.c_char_p, []),
    "srgpt_device_info": (ci, [C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)]),
    "srgpt_trace_begin": (ci, [vp, ci]),
    "srgpt_trace_end": (ci, []),
    "srgpt_gemm_workspace_bytes": (cll, []),
    "srgpt_gemm_set_workspace": (ci, [vp, cll]),
    "srgpt_gemm_bf16": (ci, [vp, ci, vp, ci, vp, ci, ci, ci, ci, vp, vp, ci, ci, ci, ci, vp]),
    "srgpt_layernorm_bf16": (ci, [vp, ci, vp, vp, vp, ci, ci, ci, cf, ci, vp]),
    "srgpt_downsample_layernorm_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, cf, vp]),
    "srgpt_rmsnorm_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, cf, vp]),
    "srgpt_patchify_bf16": (ci, [vp, ci, vp, ci, ci, ci, ci, vp]),
    "srgpt_clip_embed_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, vp]),
    "srgpt_splice_rows_bf16": (ci, [vp, vp, vp, vp, vp, vp, vp, ci, ci, vp]),
    "srgpt_mask_weights_workspace": (cll, [ci, ci, ci]),
    "srgpt_mask_weights": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, ci, cf, ci, vp]),
    "srgpt_mask_pool_workspace": (cll, [ci, ci, ci, ci]),
    "srgpt_mask_pool_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, vp]),
    "srgpt_adaptive_avgpool_bf16": (ci, [vp, vp, ci, ci, ci, ci, ci, vp]),
    "srgpt_reorder_rows_bf16": (ci, [vp, vp, ci, ci, ci, ci, ci, vp]),
    "srgpt_depth_to_u8x3": (ci, [vp, ci, ci, vp, ci, ci, vp, vp]),
    "srgpt_attention_prefill_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, cf, ci, vp]),
    "srgpt_attention_prefill_varlen_bf16": (ci, [vp, vp, vp, vp, ci, ci, ci, ci, vp, ci, ci, ci, ci, ci, cf, ci, vp]),
    "srgpt_rope_kv_append_bf16": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_rope_kv_append_varlen_bf16": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, ci, ci, vp, vp]),
    "srgpt_attention_prefill_paged_bf16": (ci, [vp, ci, vp, ci, vp, ci, vp, ci, ci, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp]),
    "srgpt_rows_equal": (ci, [vp, vp, ci, cll, vp, vp]),
    "srgpt_attention_decode_bf16": (ci, [vp, vp, vp, vp, ci, vp, ci, ci, ci, cf, vp]),
    "srgpt_gemv_bf16": (ci, [vp, vp, ci, vp, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_lm_head_workspace": (cll, [ci]),
    "srgpt_lm_head_argmax_bf16": (ci, [vp, vp, ci, ci, ci, vp, cf, vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_argmax_f32": (ci, [vp, ci, ci, vp, vp]),
    "srgpt_argmax_bf16": (ci, [vp, ci, ci, ci, vp, vp]),
    "srgpt_beam_candidates_bf16": (ci, [vp, ci, ci, ci, vp, ci, vp, vp, vp]),
    "srgpt_beam_candidates_scores_bf16": (ci, [vp, ci, ci, ci, vp, ci, vp, vp, vp, cll, vp]),
    "srgpt_beam_candidates_scored_bf16": (ci, [vp, ci, ci, ci, vp, ci, vp, vp, vp, vp]),
    "srgpt_step_scores": (ci, [vp, ci, cll, ci, ci, vp, ci, vp, cll, cll, vp]),
    "srgpt_beam_select": (ci, [vp, vp, ci, ci, ci, vp, vp, vp, vp]),
    "srgpt_beam_group_select": (ci, [vp, ci, ci, vp, vp, vp, ci, ci, ci, ci, ci, vp, ci, ci, cf, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_kv_copy_workspace_bytes": (cll, [ci, ci, ci, ci]),
    "srgpt_kv_copy_pages": (ci, [vp, ci, ci, ci, ci, vp, ci, ci, vp, cll, vp]),
    "srgpt_token_logprobs": (ci, [vp, cll, ci, ci, vp, vp, ci, vp, cll, vp, vp, vp, vp]),
    "srgpt_sample_top_p_f32": (ci, [vp, ci, vp, vp, vp, ci, vp, vp, vp, ci, vp]),
    "srgpt_sample_rows": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, ci, vp, vp]),
    "srgpt_sample_top_p_scores_f32": (ci, [vp, ci, vp, vp, vp, ci, vp, vp, vp, ci, vp, cll, vp]),
    "srgpt_sample_rows_scores": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, ci, vp, vp, cll, vp]),
    "srgpt_sample_warped_f32": (ci, [vp, ci, vp, vp, vp, ci, vp, vp, vp, ci, vp]),
    "srgpt_sample_rows_warped": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, ci, vp, vp]),
    "srgpt_sample_warped_scores_f32": (ci, [vp, ci, vp, vp, vp, ci, vp, vp, vp, ci, vp, cll, vp]),
    "srgpt_sample_rows_warped_scores": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, ci, vp, vp, cll, vp]),
    "srgpt_logits_process": (ci, [vp, ci, ci, ci, ci, vp, ci, ci, ci, vp, ci, vp, vp, ci, vp, ci, vp, vp]),
    "srgpt_logits_pick_token": (ci, [vp, vp, ci, vp, vp, vp, ci, vp]),
    "srgpt_resample_u8": (ci, [vp, vp, ci, ci, ci, ci, ci, vp, vp, ci, vp]),
    "srgpt_u8_to_normalized_chw": (ci, [vp, vp, ci, ci, ci, C.c_double, vp, vp, ci, vp]),
    "srgpt_resize_nearest_u8": (ci, [vp, vp, ci, ci, ci, ci, vp, vp, vp]),
    "srgpt_attention_decode_batched_bf16": (ci, [vp, ci, vp, ci, vp, vp, ci, ci, vp, ci, ci, ci, ci, cf, vp]),
    "srgpt_decode_batch_advance": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, vp, vp]),
    "srgpt_gemv_tp_bf16": (ci, [vp, vp, ci, vp, ci, ci, vp, cf, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, ci, ci, vp, vp]),
    "srgpt_attention_decode_tp_bf16": (ci, [vp, vp, vp, vp, ci, vp, ci, ci, ci, ci, ci, cf, vp]),
    "srgpt_tp_residual_add_bf16": (ci, [vp, vp, ci, vp]),
    "srgpt_lm_head_local_best_bf16": (ci, [vp, vp, ci, ci, ci, vp, cf, vp, ci, vp, vp]),
    "srgpt_tp_pick_token": (ci, [vp, ci, vp, vp, ci, vp, vp, vp, vp]),
    "srgpt_tp_comm_bytes": (cll, [ci, ci, ci]),
    "srgpt_tp_comm_slot_offset": (cll, [ci, ci, ci]),
    "srgpt_tp_allreduce_residual_bf16": (ci, [vp, ci, ci, cll, ci, vp, vp, vp, ci, vp]),
    "srgpt_tp_allgather_pick_token": (ci, [vp, ci, ci, cll, ci, vp, vp, vp, ci, vp, vp, vp, vp]),
    "srgpt_siglip_layers_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp]),
    "srgpt_vit_layers_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, cf, ci, vp]),
    "srgpt_llama_prefill_layers_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp]),
    "srgpt_llama_prefill_chunk_layers_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, ci, ci, vp, ci,
                                                   vp]),
    "srgpt_llama_decode_step_bf16":(ci, [vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, vp, vp, ci, vp, vp, vp, vp,
                                          vp, vp]),
    "srgpt_pack12_scan_bf16": (ci, [vp, ci, ci, ci, vp, vp, vp, vp]),
    "srgpt_pack12_bf16": (ci, [vp, ci, ci, ci, vp, vp, vp, vp, vp, vp]),
    "srgpt_unpack12_bf16": (ci, [vp, ci, ci, vp, ci, vp]),
    "srgpt_gemv_packed_bf16": (ci, [vp, vp, vp, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_lm_head_argmax_packed_bf16": (ci, [vp, vp, ci, ci, vp, cf, vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_llama_decode_step_packed_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp, vp,
                                                 vp, vp, vp, vp]),
    "srgpt_nf4_quantize_bf16": (ci, [vp, ci, ci, ci, vp, vp, vp, vp]),
    "srgpt_nf4_double_quant": (ci, [vp, cll, vp, vp, vp, vp]),
    "srgpt_nf4_dequantize_bf16": (ci, [vp, vp, ci, ci, vp, ci, vp]),
    "srgpt_nf4_lane_order": (ci, [vp, ci, ci, vp, vp]),
    "srgpt_nf4_unpack_bf16": (ci, [vp, ci, ci, vp, ci, vp]),
    "srgpt_gemv_nf4_bf16": (ci, [vp, vp, vp, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_llama_decode_step_nf4_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp, vp,
                                              vp, vp, vp, vp]),
    "srgpt_fp8_quantize_weight_bf16": (ci, [vp, ci, ci, ci, vp, vp, vp, vp]),
    "srgpt_fp8_quantize_act_bf16": (ci, [vp, ci, ci, ci, vp, ci, vp, vp]),
    "srgpt_gemm_fp8_bf16": (ci, [vp, ci, vp, vp, ci, vp, vp, ci, ci, ci, ci, vp, ci, ci, vp]),
    "srgpt_llama_prefill_layers_fp8_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, ci, ci,
                                                 vp]),
    "srgpt_llama_prefill_chunk_layers_fp8_bf16": (ci, [vp, vp, ci, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, ci,
                                                       ci, vp, ci, vp]),
    "srgpt_gemv_fp8_bf16": (ci, [vp, vp, vp, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_llama_decode_step_fp8_bf16": (ci, [vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp, vp, vp, vp,
                                              vp, vp]),
    "srgpt_gemv_multi_bf16": (ci, [vp, ci, vp, ci, vp, ci, ci, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_gemv_multi_packed_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_lm_head_multi_bf16": (ci, [vp, ci, vp, ci, ci, ci, ci, vp, cf, vp, vp, vp]),
    "srgpt_lm_head_multi_packed_bf16": (ci, [vp, ci, vp, ci, ci, ci, vp, cf, vp, vp, vp]),
    "srgpt_attention_decode_multi_bf16": (ci, [vp, ci, vp, ci, vp, vp, ci, vp, ci, ci, ci, ci, cf, vp]),
    "srgpt_spec_draft": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, vp, vp, ci, vp, vp, vp]),
    "srgpt_spec_accept": (ci, [vp, ci, ci, vp, vp, ci, vp, vp, vp, vp, vp, vp]),
    "srgpt_llama_verify_step_bf16": (ci, [vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, vp, ci, vp, vp, ci, vp, vp, vp, vp,
                                          vp, vp, ci, vp, vp, ci, vp, vp, vp]),
    "srgpt_llama_verify_step_packed_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp,
                                                 vp, vp, vp, vp, vp, ci, vp, vp, ci, vp, vp, vp]),
    "srgpt_gemm_nf4_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, vp, ci, ci, vp]),
    "srgpt_gemv_multi_nf4_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, vp, cf, vp, ci, ci, ci, ci, vp, vp, vp, vp, vp, ci, vp]),
    "srgpt_llama_prefill_layers_nf4_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp]),
    "srgpt_llama_prefill_chunk_layers_nf4_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, ci, ci,
                                                       vp, ci, vp]),
    "srgpt_llama_verify_step_nf4_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp,
                                              vp, vp, vp, vp, vp, ci, vp, vp, ci, vp, vp, vp]),
    "srgpt_gemv_rows_bf16": (ci, [vp, ci, vp, ci, vp, ci, ci, ci, ci, vp, cf, ci, ci, ci, vp, vp, vp, vp, vp, ci, ci, vp]),
    "srgpt_gemv_rows_packed_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, vp, cf, ci, ci, ci, vp, vp, vp, vp, vp, ci, ci, vp]),
    "srgpt_gemv_rows_nf4_bf16": (ci, [vp, ci, vp, vp, ci, ci, ci, ci, vp, cf, ci, ci, ci, vp, vp, vp, vp, vp, ci, ci, vp]),
    "srgpt_attention_decode_rows_bf16": (ci, [vp, ci, vp, ci, vp, vp, ci, ci, vp, ci, ci, ci, ci, cf, vp]),
    "srgpt_rows_advance": (ci, [vp, ci, vp, ci, vp, vp, ci, vp, vp, vp, vp]),
    "srgpt_llama_decode_rows_bf16": (ci, [vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, vp, ci, vp, vp, vp, vp,
                                          vp, vp, vp, vp, vp]),
    "srgpt_llama_decode_rows_packed_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, vp, vp, ci, vp,
                                                 vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_llama_decode_rows_nf4_bf16": (ci, [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, vp, vp, ci, vp,
                                              vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_guidance_rows": (ci, [vp, ci, ci, vp, vp, vp, vp, vp]),
    "srgpt_guidance_pair_ids": (ci, [vp, ci, vp]),
    "srgpt_llama_decode_rows_guided_bf16": (ci, [vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, vp, vp,
                                                 ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_llama_decode_rows_warped_bf16": (ci, [vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci, vp, vp, vp,
                                                 ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_contrastive_partial_floats": (cll, [ci, ci, ci]),
    "srgpt_contrastive_penalty_bf16": (ci, [vp, ci, vp, ci, ci, vp, ci, ci, vp, vp]),
    "srgpt_contrastive_select_bf16": (ci, [vp, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, ci, vp, ci, vp, ci, ci, vp, vp, vp, vp, vp, vp, vp]),
    "srgpt_kv_broadcast_rows": (ci, [vp, ci, ci, ci, ci, vp, ci, vp, ci, vp, ci, ci, vp]),
    "srgpt_attention_probs_bf16": (ci, [vp, ci, vp, ci, ci, vp, ci, ci, ci, ci, cf, vp, cll, cll, cll, ci, vp, vp]),
    "srgpt_llama_prefill_layers_probe_bf16": (ci, [vp, vp, vp, vp, ci, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, ci,
                                                   vp, ci, ci, vp, vp]),
    "srgpt_attention_probs_decode_bf16": (ci, [vp, ci, vp, vp, ci, ci, vp, ci, ci, ci, ci, cf, vp, vp, ci, ci, vp, ci, vp, cll, cll, cll, vp, vp]),
    "srgpt_store_step_rows_bf16": (ci, [vp, ci, ci, vp, ci, vp, cll, cll, vp]),
    "srgpt_llama_decode_step_probe_bf16": (ci, [vp, vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, cf, vp, vp, vp, vp, ci, vp, vp, vp, ci, vp,
                                                vp, vp, vp, vp, vp, vp]),
}

SPEC_T_MAX = 8  # SRGPT_SPEC_T_MAX: tokens per verify pass (the last emitted token + up to 7 drafts)


class SiglipLayerWeights(C.Structure):
    _fields_ = [(n, vp) for n in ("ln1_w", "ln1_b", "qkv_w", "qkv_b", "out_w", "out_b", "ln2_w", "ln2_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b")]


class LlamaLayerWeights(C.Structure):
    _fields_ = [(n, vp) for n in ("in_norm", "qkv_w", "o_w", "post_norm", "gateup_w", "down_w", "kv_pages")]


class Packed12(C.Structure):
    """srgpt_packed12: one matrix in the 12-bit decode packing (all NULL = the matrix stays plain bf16)."""
    _fields_ = [(n, vp) for n in ("sm", "ex", "base", "row_ptr", "exc")]


class LlamaLayerPacked(C.Structure):
    _fields_ = [(n, Packed12) for n in ("qkv", "o", "gateup", "down")]


class Nf4(C.Structure):
    """srgpt_nf4: one matrix's NF4 planes for the decode GEMV (q NULL = the step reads the dequantized matrix)."""
    _fields_ = [("q", vp), ("scale", vp)]


class LlamaLayerNf4(C.Structure):
    _fields_ = [(n, Nf4) for n in ("qkv", "o", "gateup", "down")]


class Guidance(C.Structure):
    """srgpt_guidance: the device scale g and the guided rows [B / 2, V] of a guided rows step."""
    _fields_ = [("scale", vp), ("guided_rows", vp)]


class PrefillProbe(C.Structure):
    """srgpt_prefill_probe: where a probed prefill stack stores its hidden states and attention probabilities (strides in elements)."""
    _fields_ = [("hidden", vp), ("hidden_layer_stride", cll), ("hidden_seq_stride", cll), ("hidden_ld", cll), ("attn", vp),
                ("attn_layer_stride", cll), ("attn_seq_stride", cll), ("attn_head_stride", cll), ("attn_ld", cll), ("out_rows", ci),
                ("row_off", vp)]


class DecodeProbe(C.Structure):
    """srgpt_decode_probe: where a probed decode step stores its hidden rows and attention probabilities (strides in elements)."""
    _fields_ = [("hidden", vp), ("hidden_step_stride", cll), ("hidden_layer_stride", cll), ("hidden_row_stride", cll), ("attn", vp),
                ("attn_step_stride", cll), ("attn_layer_stride", cll), ("attn_row_stride", cll), ("attn_head_stride", cll), ("step_offset", ci),
                ("T", ci), ("n_cols", ci), ("off", vp), ("n_prompt", vp), ("ws", vp)]


class Fp8(C.Structure):
    """srgpt_fp8: one matrix's E4M3 codes [N, K] and row scales [N]."""
    _fields_ = [("q", vp), ("scale", vp)]


class LlamaLayerFp8(C.Structure):
    _fields_ = [("in_norm", vp), ("qkv", Fp8), ("o", Fp8), ("post_norm", vp), ("gateup", Fp8), ("down", Fp8), ("kv_pages", vp)]


def lib_path(elem: str = "bf16") -> str:
    return _build.VARIANTS[elem][0]


def current_elem() -> str:
    return _elem


def set_elem(elem: str) -> str:
    """Selects which build of the library (bf16 or f16 elements) ``load()`` hands out; returns the previous setting."""
    global _elem
    if elem not in _build.VARIANTS:
        raise SrgptError(f"unsupported element type {elem!r} (have {sorted(_build.VARIANTS)})")
    prev, _elem = _elem, elem
    return prev


def load(build_if_missing: bool = True, elem: str = None):
    """Load (building first if the .so is missing/stale and nvcc is present) and type the library of the given (default: the
    current) element type."""
    elem = elem or _elem
    with _lock:
        if elem in _libs:
            return _libs[elem]
        path = lib_path(elem)
        if build_if_missing and _build.is_stale():
            try:
                _build.build(verbose=False)
            except Exception as e:  # stale-but-present is still loadable; missing is fatal
                if not os.path.exists(path):
                    raise SrgptError(f"{os.path.basename(path)} is missing and could not be built: {e}") from e
        if not os.path.exists(path):
            raise SrgptError(f"{path} not found; run `python -c 'import __graft_entry__ as g; g.build()'`")
        try:
            import torch  # noqa: F401  (loads libcudart.so.12 that the library links against)
        except Exception:
            pass
        lib = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as e:
                raise SrgptError(f"{path} does not export {name}") from e
            fn.restype = res
            fn.argtypes = args
        if lib.srgpt_abi_version() != 1:
            raise SrgptError(f"ABI version mismatch between _lib.py and {os.path.basename(path)}")
        if lib.srgpt_elem_type() != {"bf16": 0, "f16": 1}[elem]:
            raise SrgptError(f"{path} was not built for {elem} elements")
        _libs[elem] = lib
        return lib


def last_error() -> str:
    return (load().srgpt_last_error() or b"").decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise SrgptError(f"{what} failed with code {rc}: {last_error()}")


def device_info():
    sm, maj, mnr = ci(0), ci(0), ci(0)
    check(load().srgpt_device_info(C.byref(sm), C.byref(maj), C.byref(mnr)), "srgpt_device_info")
    return sm.value, maj.value, mnr.value
