"""``load_pretrained_model`` for the reference's four-directory checkpoint layout.

Reference: llava/model/builder.py:36-213 (loader), llava/model/llava_arch.py:63-109 (init_vlm),
:181-250 (save_pretrained = the on-disk layout), llava/model/utils.py:25-55 (sub-directory
resolution):

    <ckpt>/config.json                 LlavaConfig: architectures, enable_region, enable_depth, mm_* fields,
                                       llm_cfg / vision_tower_cfg / mm_projector_cfg / region_extractor_cfg
    <ckpt>/llm/                        HF LlamaForCausalLM weights + config + tokenizer files
    <ckpt>/vision_tower/               HF SiglipVisionModel weights + config + preprocessor_config.json
    <ckpt>/mm_projector/               {"mm_projector_type": "mlp_downsample"} + weights
    <ckpt>/region_extractor/           {"region_extractor_type": "regiongpt"} + weights

``read_checkpoint`` is pure host code (testable without a GPU); ``load_pretrained_model`` then puts the
weights on the device in the kernel layouts and returns the reference's 4-tuple.
"""
from __future__ import annotations

import glob
import json
import os
from typing import Any, Dict, Optional, Tuple

import torch

from .config import LlamaDims, LlavaConfig, VisionConfig
from .constants import (DEFAULT_DEPTH_TOKEN, DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IMAGE_PATCH_TOKEN,
                        DEFAULT_MASK_TOKEN)

SUBDIRS = ("llm", "vision_tower", "mm_projector", "region_extractor")


def _read_json(path: str) -> Dict[str, Any]:
    with open(path) as f:
        return json.load(f)


def load_state_dict(directory: str) -> Dict[str, torch.Tensor]:
    """All tensors of an HF-style weight directory: (sharded) safetensors first, then pytorch_model*.bin."""
    files = sorted(glob.glob(os.path.join(directory, "*.safetensors")))
    out: Dict[str, torch.Tensor] = {}
    if files:
        from safetensors.torch import load_file

        for f in files:
            out.update(load_file(f, device="cpu"))
        return out
    files = sorted(glob.glob(os.path.join(directory, "pytorch_model*.bin")))
    if not files:
        raise FileNotFoundError(f"no *.safetensors or pytorch_model*.bin under {directory}")
    for f in files:
        out.update(torch.load(f, map_location="cpu", weights_only=True))
    return out


def _sub_path(root: str, top: Dict[str, Any], key: str) -> str:
    """llava/model/utils.py:41-53: dict / config object -> <root>/<name>; string -> that path."""
    cfg = top.get(key + "_cfg")
    if isinstance(cfg, str) and cfg:
        return cfg
    return os.path.join(root, key)


def _vision_config(d: Dict[str, Any]) -> VisionConfig:
    arch = " ".join(d.get("architectures") or []).lower()
    d = d.get("vision_config", d)  # a full SiglipConfig / CLIPConfig nests the vision part
    mt = d.get("model_type") or ""
    is_clip = ("clip" in arch or "clip" in mt) and "siglip" not in (arch + mt)  # multimodal_encoder/builder.py:38-47 keys on the architecture name
    for other in ("intern", "radio"):  # multimodal_encoder/builder.py:27-35: towers of other model families (SURVEY.md: out of scope)
        if other in arch or other in mt:
            raise NotImplementedError(f"vision tower family {other!r} is outside the SpatialRGPT generate() path (SigLIP and CLIP towers are built)")
    if is_clip:
        return VisionConfig(image_size=d.get("image_size", 224), patch_size=d.get("patch_size", 32), hidden_size=d.get("hidden_size", 768),
                            num_hidden_layers=d.get("num_hidden_layers", 12), num_attention_heads=d.get("num_attention_heads", 12),
                            intermediate_size=d.get("intermediate_size", 3072), layer_norm_eps=d.get("layer_norm_eps", 1e-5),
                            hidden_act=d.get("hidden_act", "quick_gelu"), model_type="clip_vision_model")
    return VisionConfig(image_size=d.get("image_size", 384), patch_size=d.get("patch_size", 14), hidden_size=d.get("hidden_size", 1152),
                        num_hidden_layers=d.get("num_hidden_layers", 27), num_attention_heads=d.get("num_attention_heads", 16),
                        intermediate_size=d.get("intermediate_size", 4304), layer_norm_eps=d.get("layer_norm_eps", 1e-6),
                        hidden_act=d.get("hidden_act", "gelu_pytorch_tanh"))


def _llama_dims(d: Dict[str, Any]) -> LlamaDims:
    nh = d["num_attention_heads"]
    rope = d.get("rope_theta")
    if rope is None and isinstance(d.get("rope_parameters"), dict):
        rope = d["rope_parameters"].get("rope_theta")
    # rope_scaling as the reference's modeling file reads it (modeling_llama.py:267-292): {"type": "linear" | "dynamic", "factor": f};
    # plus the context extension the loader applies itself (language_model/builder.py:31-38: model_max_length > max_position_embeddings)
    factor = 1.0
    rs = d.get("rope_scaling")
    orig_ctx, model_max = d.get("max_position_embeddings"), d.get("model_max_length")
    if orig_ctx and model_max and model_max > orig_ctx:
        import math
        rs = {"type": "linear", "factor": float(math.ceil(model_max / orig_ctx))}
    if rs not in (None, {}):
        kind = rs.get("type", rs.get("rope_type"))
        if kind == "linear":
            factor = float(rs["factor"])
        elif kind == "dynamic":
            # NTK scaling only changes the base once a sequence exceeds max_position_embeddings (modeling_llama.py:148-156); this
            # decoder never runs past it (max_seq_len <= max_position_embeddings is enforced by load_pretrained_model)
            factor = 1.0
        elif kind in (None, "default"):
            factor = 1.0
        else:
            raise ValueError(f"Unknown RoPE scaling type {kind}")  # modeling_llama.py:291
    return LlamaDims(hidden_size=d["hidden_size"], num_hidden_layers=d["num_hidden_layers"], num_attention_heads=nh,
                     num_key_value_heads=d.get("num_key_value_heads", nh), head_dim=d.get("head_dim") or d["hidden_size"] // nh,
                     intermediate_size=d["intermediate_size"], vocab_size=d["vocab_size"], rope_theta=float(rope or 10000.0), rope_scaling_factor=factor,
                     rms_norm_eps=d.get("rms_norm_eps", 1e-6), max_position_embeddings=d.get("max_position_embeddings", 4096),
                     bos_token_id=d.get("bos_token_id"), eos_token_id=d.get("eos_token_id"), pad_token_id=d.get("pad_token_id"),
                     tokenizer_model_max_length=d.get("tokenizer_model_max_length"),
                     tokenizer_padding_side=d.get("tokenizer_padding_side", "right"))


def is_mm_model(model_path: str) -> bool:
    """llava/model/utils.py:58-73: a VLM checkpoint names a llava architecture in its top-level config."""
    cfg = os.path.join(model_path, "config.json")
    if not os.path.exists(cfg):
        return False
    return any("llava" in a.lower() for a in _read_json(cfg).get("architectures", []))


def read_checkpoint(model_path: str, load_tokenizer: bool = True):
    """Parse a reference checkpoint directory -> (LlavaConfig, state dicts keyed like the reference, tokenizer,
    image_processor).  Registers <mask>/<depth> (and optional <im_patch>/<im_start>/<im_end>) exactly as
    builder.py:186-199 and records the ids on the config."""
    top = _read_json(os.path.join(model_path, "config.json"))
    paths = {k: _sub_path(model_path, top, k) for k in SUBDIRS}
    llm_cfg = _read_json(os.path.join(paths["llm"], "config.json"))
    vt_cfg = _read_json(os.path.join(paths["vision_tower"], "config.json"))
    mp_cfg = _read_json(os.path.join(paths["mm_projector"], "config.json"))
    enable_region = bool(top.get("enable_region", False))
    re_cfg = _read_json(os.path.join(paths["region_extractor"], "config.json")) if enable_region else {}

    if top.get("s2"):
        raise NotImplementedError("S2 multi-scale tower wrappers (CLIPVisionTowerS2 / SiglipVisionTowerS2, multimodal_encoder/builder.py:36-47)")
    cfg = LlavaConfig(
        model_type=top.get("model_type", "llava_llama"), architectures=tuple(top.get("architectures", ("LlavaLlamaModel",))),
        resume_path=model_path, image_aspect_ratio=top.get("image_aspect_ratio", "resize"),
        mm_vision_select_layer=top.get("mm_vision_select_layer", -2),
        mm_vision_select_feature=top.get("mm_vision_select_feature", "cls_patch"),
        mm_use_im_start_end=bool(top.get("mm_use_im_start_end", False)),
        mm_use_im_patch_token=bool(top.get("mm_use_im_patch_token", True)),  # loader default True (builder.py:194)
        enable_region=enable_region, enable_depth=bool(top.get("enable_depth", False)),
        model_dtype=top.get("model_dtype", "torch.float16"),  # llava_arch.py:74 default
        vision=_vision_config(vt_cfg), llama=_llama_dims(llm_cfg),
        mm_projector_type=mp_cfg.get("mm_projector_type", "mlp_downsample"),
        region_extractor_type=re_cfg.get("region_extractor_type", "regiongpt"))

    # HF generate() stops on generation_config.eos_token_id (llava_llama.py:212 -> GenerationMixin), which for Llama-3 chat
    # checkpoints is a LIST that includes <|eot_id|>; config.json alone only names <|end_of_text|>
    gen_cfg_path = os.path.join(paths["llm"], "generation_config.json")
    if os.path.exists(gen_cfg_path):
        gen_cfg = _read_json(gen_cfg_path)
        if gen_cfg.get("eos_token_id") is not None:
            cfg.llama.eos_token_id = gen_cfg["eos_token_id"]
        if gen_cfg.get("pad_token_id") is not None and cfg.llama.pad_token_id is None:
            cfg.llama.pad_token_id = gen_cfg["pad_token_id"]

    sd = {"llm": load_state_dict(paths["llm"]), "vision_tower": load_state_dict(paths["vision_tower"]),
          "mm_projector": load_state_dict(paths["mm_projector"])}
    if enable_region:
        sd["region_extractor"] = load_state_dict(paths["region_extractor"])
    # keys may carry the wrapper prefixes the reference strips at save time (llava_arch.py:194-225)
    sd["vision_tower"] = {k.split("vision_tower.vision_tower.")[-1]: v for k, v in sd["vision_tower"].items()}

    tokenizer = image_processor = None
    if load_tokenizer:
        from transformers import AutoImageProcessor, AutoTokenizer

        try:
            tokenizer = AutoTokenizer.from_pretrained(paths["llm"], use_fast=False, legacy=False)  # builder.py / language_model/builder.py:77-90
        except Exception:
            tokenizer = AutoTokenizer.from_pretrained(paths["llm"])
        try:
            image_processor = AutoImageProcessor.from_pretrained(paths["vision_tower"])
        except Exception:
            image_processor = None
        if enable_region:
            tokenizer.add_tokens([DEFAULT_MASK_TOKEN, DEFAULT_DEPTH_TOKEN], special_tokens=True)
            cfg.llm_mask_token_id = tokenizer.convert_tokens_to_ids(DEFAULT_MASK_TOKEN)
            cfg.llm_depth_token_id = tokenizer.convert_tokens_to_ids(DEFAULT_DEPTH_TOKEN)
        if cfg.mm_use_im_patch_token:
            tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
        if cfg.mm_use_im_start_end:
            tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
        _resize_token_embeddings(cfg, sd["llm"], len(tokenizer))
    return cfg, sd, tokenizer, image_processor


def _resize_token_embeddings(cfg: LlavaConfig, llm_sd: Dict[str, torch.Tensor], new_size: int) -> None:
    """builder.py:199 ``model.resize_token_embeddings(len(tokenizer))``: grow (or shrink) embed_tokens and lm_head;
    new rows are initialised like HF does (normal, std = initializer_range 0.02)."""
    emb = llm_sd["model.embed_tokens.weight"]
    old = emb.shape[0]
    if new_size == old:
        return
    g = torch.Generator().manual_seed(0)
    for key in ("model.embed_tokens.weight", "lm_head.weight"):
        if key not in llm_sd:
            continue
        w = llm_sd[key]
        if new_size < old:
            llm_sd[key] = w[:new_size].contiguous()
        else:
            extra = (torch.randn(new_size - old, w.shape[1], generator=g) * 0.02).to(w.dtype)
            llm_sd[key] = torch.cat([w, extra], dim=0)
    cfg.llama.vocab_size = new_size


def load_pretrained_model(model_path: str, model_name: str, model_base: Optional[str] = None, load_8bit: bool = False,
                          load_4bit: bool = False, device_map: str = "auto", device: str = "cuda", **kwargs):
    """Reference signature (builder.py:36-45) -> (tokenizer, model, image_processor, context_len).

    The model comes back in fp16 like the reference's (builder.py:62 sets torch_dtype = float16 unconditionally); callers that want
    bf16 cast afterwards exactly as the reference's do (``model.to(dtype=torch.bfloat16)``, eval_spatial.py:221).  ``torch_dtype=``
    (torch.float16 / torch.bfloat16) is an extension that loads straight into that dtype.  ``quantization="nf4"`` is an extension too:
    the decoder-layer linears are NF4-quantized at load (weights.from_state_dicts) and dequantized into that dtype; the batch-1 decode
    step streams the 4-bit planes.  ``quantization="fp8"`` quantizes the same linears to per-row E4M3 weights (W8A8: every activation row
    is quantized alike before each linear), keeps no element-type copy of them, and runs them on the FP8 tensor cores (prefill, batched
    decode, beams) and through the FP8 decode GEMV (the one-token step); ``prompt_lookup_num_tokens`` then raises.
    ``nf4_dequantized_copy=False`` (with ``quantization="nf4"`` only) keeps no dequantized copy of the layer matrices that have NF4 planes:
    prefill, batched decode, beams and the verify pass read the planes too (bit-identical).  ``load_4bit`` / ``load_8bit`` (bitsandbytes)
    still raise."""
    if load_8bit or load_4bit:
        raise NotImplementedError("bitsandbytes quantised loading is outside the hot path (builder.py:51-60)")
    if model_base is not None:
        raise NotImplementedError("LoRA / delta checkpoints (builder.py:66-140) are outside the hot path")
    if not kwargs.get("nf4_dequantized_copy", True) and kwargs.get("quantization") != "nf4":
        raise ValueError(f"nf4_dequantized_copy=False needs quantization='nf4', not {kwargs.get('quantization')!r}")
    if not is_mm_model(model_path):
        raise ValueError(f"{model_path} is not a llava-style VLM checkpoint (config.json 'architectures')")
    from .llava_llama import LlavaLlamaModel
    from .weights import from_state_dicts

    cfg, sd, tokenizer, image_processor = read_checkpoint(model_path)
    dev = torch.device(device if device != "cuda" else f"cuda:{torch.cuda.current_device()}")
    max_seq = int(kwargs.pop("max_seq_len", min(cfg.llama.max_position_embeddings, 4096)))
    dtype = kwargs.pop("torch_dtype", None) or torch.float16
    if dtype not in (torch.float16, torch.bfloat16):
        raise NotImplementedError(f"torch_dtype {dtype}: the sm_90a kernels compute in torch.float16 or torch.bfloat16")
    quantization = kwargs.pop("quantization", None)
    nf4_dequantized_copy = kwargs.pop("nf4_dequantized_copy", True)
    model = LlavaLlamaModel(cfg, from_state_dicts(cfg, sd, dev, dtype=dtype, quantization=quantization, nf4_dequantized_copy=nf4_dequantized_copy),
                            tokenizer=tokenizer,
                            image_processor=image_processor, max_seq_len=max_seq)
    context_len = getattr(cfg.llama, "max_sequence_length", 2048) if hasattr(cfg.llama, "max_sequence_length") else 2048
    return tokenizer, model, image_processor, context_len


def prepare_config_for_eval(config: LlavaConfig, kwargs: dict) -> None:
    """builder.py:228-240: resolve the model dtype; SigLIP forces device_map 'cuda'."""
    kwargs.pop("torch_dtype", None)
    kwargs["device_map"] = "cuda"
