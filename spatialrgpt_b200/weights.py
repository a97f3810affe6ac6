"""Device-resident parameters in the layouts the sm_90a kernels consume.

Source layout = the reference's four-directory checkpoint (llava_arch.py:181-250): state dicts
``vision_tower`` (HF SiglipVisionModel keys), ``region_extractor`` (base_extractor.py),
``mm_projector`` (base_projector.py), ``llm`` (HF LlamaForCausalLM keys).  Transformations done
ONCE at load time (pure re-layout, no arithmetic):
  * SigLIP q/k/v weights and biases concatenated -> one [3D, D] GEMM;
  * Conv2d(3,D,14,14) flattened to [D, 588] and zero-padded to ld 592 (16-byte TMA rows);
  * ConvTranspose2d(k=2,s=2) [Cin, Cout, 2, 2] -> [(di,dj,Cout), Cin] so deconv == one GEMM whose
    output rows are already the up-sampled pixels (nested 2x2 order), bias tiled x4;
  * Llama q/k/v concatenated -> [(nh + 2 nkv) hd, H]; gate/up rows INTERLEAVED (gate_i, up_i) so the
    SwiGLU product is local to one accumulator pair / one warp.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from .config import LlavaConfig

BF16 = torch.bfloat16


def _pad_cols(w: torch.Tensor, ld: int) -> torch.Tensor:
    if w.shape[1] == ld:
        return w.contiguous()
    out = torch.zeros((w.shape[0], ld), dtype=w.dtype, device=w.device)
    out[:, : w.shape[1]] = w
    return out


def patch_ldk(patch: int) -> int:
    return (3 * patch * patch + 7) // 8 * 8


@dataclass
class VisionLayerW:
    ln1_w: torch.Tensor
    ln1_b: torch.Tensor
    qkv_w: torch.Tensor
    qkv_b: torch.Tensor
    out_w: torch.Tensor
    out_b: torch.Tensor
    ln2_w: torch.Tensor
    ln2_b: torch.Tensor
    fc1_w: torch.Tensor
    fc1_b: torch.Tensor
    fc2_w: torch.Tensor
    fc2_b: torch.Tensor


@dataclass
class VisionW:
    patch_w: torch.Tensor  # [D, ldk]
    patch_b: Optional[torch.Tensor]  # None for CLIP (bias-free convolution)
    pos_emb: torch.Tensor  # [T, D]  (CLIP: [T + 1, D], row 0 = the class token's position)
    layers: List[VisionLayerW] = field(default_factory=list)
    cls_emb: Optional[torch.Tensor] = None   # CLIP: class_embedding [D]
    pre_ln_w: Optional[torch.Tensor] = None  # CLIP: pre_layrnorm
    pre_ln_b: Optional[torch.Tensor] = None


@dataclass
class RegionW:
    deconv1_w: torch.Tensor  # [4C, C]
    deconv1_b: torch.Tensor  # [4C]
    ln_w: torch.Tensor
    ln_b: torch.Tensor
    deconv2_w: torch.Tensor
    deconv2_b: torch.Tensor
    rgb_w: torch.Tensor  # [H, C]
    rgb_b: torch.Tensor
    depth_w: torch.Tensor
    depth_b: torch.Tensor


@dataclass
class ProjectorW:
    """``mlp_downsample``: LayerNorm(4C) + two linears.  The other reference types (base_projector.py:69-72,81-91) keep their
    linears in ``linears`` [(weight [out, in], bias)] - one for ``linear``, N for ``mlpNx_gelu``, none for ``identity``."""
    ln_w: Optional[torch.Tensor] = None  # [4C]
    ln_b: Optional[torch.Tensor] = None
    fc1_w: Optional[torch.Tensor] = None  # [H, 4C]
    fc1_b: Optional[torch.Tensor] = None
    fc2_w: Optional[torch.Tensor] = None  # [H, H]
    fc2_b: Optional[torch.Tensor] = None
    linears: List = field(default_factory=list)


@dataclass
class LlamaLayerW:
    in_norm: torch.Tensor
    qkv_w: torch.Tensor  # [(nh + 2 nkv) hd, H]
    o_w: torch.Tensor  # [H, nh hd]
    post_norm: torch.Tensor
    gateup_w: torch.Tensor  # [2 I, H], rows interleaved (gate_i, up_i)
    down_w: torch.Tensor  # [H, I]
    # quantization="nf4": {"qkv", "o", "gateup", "down"} -> the fused matrix's Nf4W planes, or None where K is not a multiple of 1024
    # (the *_w tensors above are then the dequantized matrices).  With nf4_dequantized_copy=False a matrix that has planes keeps no
    # dequantized copy: its *_w field holds the same Nf4W.  quantization="fp8": the *_w fields hold Fp8W and there is no element-type
    # copy of the matrices.
    nf4: Optional[Dict[str, Optional["Nf4W"]]] = None


@dataclass
class LlamaW:
    embed: torch.Tensor  # [V, H]
    norm: torch.Tensor
    lm_head: torch.Tensor  # [V, H]
    layers: List[LlamaLayerW] = field(default_factory=list)
    quantization: Optional[str] = None  # None, "nf4" or "fp8" (the decoder-layer linears only)
    nf4_dequantized_copy: bool = True  # quantization="nf4": False = the matrices with planes keep no element-type copy


@dataclass
class Packed12W:
    """A bf16 weight [N, K] in the lossless 12-bit packing the batch-1 decode GEMV streams (DESIGN.md §3, include/srgpt_b200.h
    srgpt_packed12): sm [N, K] u8 sign/mantissa, ex [N, K/2] u8 exponent codes, base [N] u8, and the exceptions
    exc[row_ptr[r]:row_ptr[r+1]] = column << 8 | exponent (int32).  Built by ops.pack12."""
    sm: torch.Tensor
    ex: torch.Tensor
    base: torch.Tensor
    row_ptr: torch.Tensor
    exc: torch.Tensor

    @property
    def shape(self):
        return self.sm.shape

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (self.sm, self.ex, self.base, self.row_ptr, self.exc))


@dataclass
class Nf4W:
    """An NF4-quantized weight [N, K] as the batch-1 decode GEMV streams it (DESIGN.md §3, include/srgpt_b200.h srgpt_nf4): q [N, K/2]
    uint8 codes in the GEMV's lane order, scale [N, K/64] fp32 resolved scales.  Built by ops.nf4_planes."""
    q: torch.Tensor
    scale: torch.Tensor

    @property
    def shape(self):
        return (self.q.shape[0], self.q.shape[1] * 2)

    def nbytes(self) -> int:
        return self.q.numel() + self.scale.numel() * 4


@dataclass
class Fp8W:
    """An FP8 (E4M3) weight [N, K] of the W8A8 decoder-layer linears (DESIGN.md §3, include/srgpt_b200.h srgpt_fp8): q [N, K] uint8 codes,
    scale [N] fp32 row scales; the weight stands for q * scale.  Built by ops.fp8_quantize_weight."""
    q: torch.Tensor
    scale: torch.Tensor

    @property
    def shape(self):
        return self.q.shape

    def nbytes(self) -> int:
        return self.q.numel() + self.scale.numel() * 4


@dataclass
class ModelWeights:
    vision: VisionW
    region: Optional[RegionW]
    projector: ProjectorW
    llama: LlamaW

    def nbytes(self) -> int:
        total = 0

        def walk(o):
            nonlocal total
            if isinstance(o, torch.Tensor):
                total += o.numel() * o.element_size()
            elif isinstance(o, (list, tuple)):
                for x in o:
                    walk(x)
            elif hasattr(o, "__dataclass_fields__"):
                for k in o.__dataclass_fields__:
                    walk(getattr(o, k))

        walk(self)
        return total

    @property
    def dtype(self) -> torch.dtype:
        return self.llama.embed.dtype

    def to(self, dtype: torch.dtype) -> "ModelWeights":
        """In-place cast of every floating-point weight (what ``model.to(dtype=...)`` does to the reference's modules,
        llava/eval/eval_spatial.py:221); the kernel layouts (padding, interleaving, fused qkv) are dtype independent."""
        if self.llama.quantization is not None and dtype != self.dtype:
            raise NotImplementedError(f"the {self.llama.quantization} layer matrices are dequantized into the element type they were loaded in "
                                      f"({self.dtype}); load the model with torch_dtype={dtype} instead of casting it")

        def walk(o):
            if isinstance(o, torch.Tensor):
                return o.to(dtype) if o.is_floating_point() else o
            if isinstance(o, list):
                return [walk(x) for x in o]
            if isinstance(o, tuple):
                return tuple(walk(x) for x in o)
            if hasattr(o, "__dataclass_fields__"):
                for k in o.__dataclass_fields__:
                    setattr(o, k, walk(getattr(o, k)))
            return o

        walk(self)
        return self


def _deconv_as_gemm(w: torch.Tensor) -> torch.Tensor:
    """ConvTranspose2d weight [Cin, Cout, 2, 2] -> [(di*2+dj)*Cout + co, Cin]."""
    cin, cout = w.shape[0], w.shape[1]
    return w.permute(2, 3, 1, 0).reshape(4 * cout, cin).contiguous()


def interleave_rows(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    return torch.stack((gate, up), dim=1).reshape(2 * gate.shape[0], gate.shape[1]).contiguous()


def from_state_dicts(cfg: LlavaConfig, sd: Dict[str, Dict[str, torch.Tensor]], device, n_tower_layers: Optional[int] = None,
                     dtype: torch.dtype = BF16, quantization: Optional[str] = None, nf4_dequantized_copy: bool = True) -> ModelWeights:
    """sd = {"vision_tower": ..., "region_extractor": ..., "mm_projector": ..., "llm": ...} with the
    reference's key names; tensors may live on the CPU in any float dtype.  ``dtype``: torch.bfloat16 or torch.float16.
    ``quantization="nf4"``: every decoder-layer linear (q/k/v/o/gate/up/down_proj) is NF4-quantized on the device as its own [out, in]
    matrix, before qkv is fused and gate/up interleaved (the reference's load_4bit, llava/model/builder.py:51-60); the layer keeps the
    dequantized matrices for every path and the NF4 planes for the batch-1 decode step.  Embeddings, lm_head, norms, towers, projector
    and region extractor stay unquantized.
    ``nf4_dequantized_copy=False`` (only with ``quantization="nf4"``): a fused matrix with planes (K a multiple of 1024) drops its
    dequantized copy once the planes are checked against it, and every path reads the planes (the NF4 GEMM, the one-token and multi-token
    NF4 GEMVs), bit-identical to the copy.  Layer matrices take 4.5 bits per weight instead of 16 + 4.5.
    ``quantization="fp8"``: W8A8 with E4M3 codes (DESIGN.md §3): every decoder-layer linear is quantized on the device per output row, one
    matrix at a time, and the layer holds only the codes and row scales; every path (prefill, batched decode, beams, the one-token step)
    quantizes each activation row the same way before the FP8 GEMM.  Embeddings, lm_head, norms, towers, projector and region extractor
    stay unquantized."""
    if quantization not in (None, "nf4", "fp8"):
        raise ValueError(f"quantization={quantization!r}: supported are None, 'nf4' and 'fp8'")
    if not nf4_dequantized_copy and quantization != "nf4":
        raise ValueError(f"nf4_dequantized_copy=False needs quantization='nf4', not {quantization!r}")
    dev = torch.device(device)

    def g(d, k):
        return d[k].to(device=dev, dtype=dtype)

    v, vc = sd["vision_tower"], cfg.vision
    D = vc.hidden_size
    pw = g(v, "vision_model.embeddings.patch_embedding.weight").reshape(D, -1)
    if vc.is_clip:  # HF CLIPVisionModel: no conv bias, class token, pre_layrnorm (sic)
        vision = VisionW(patch_w=_pad_cols(pw, patch_ldk(vc.patch_size)), patch_b=None,
                         pos_emb=g(v, "vision_model.embeddings.position_embedding.weight").contiguous(),
                         cls_emb=g(v, "vision_model.embeddings.class_embedding").reshape(-1).contiguous(),
                         pre_ln_w=g(v, "vision_model.pre_layrnorm.weight"), pre_ln_b=g(v, "vision_model.pre_layrnorm.bias"))
    else:
        vision = VisionW(patch_w=_pad_cols(pw, patch_ldk(vc.patch_size)),
                         patch_b=g(v, "vision_model.embeddings.patch_embedding.bias").contiguous(),
                         pos_emb=g(v, "vision_model.embeddings.position_embedding.weight").contiguous())
    if vision.pos_emb.shape[0] != vc.tokens:
        raise ValueError(f"position embedding has {vision.pos_emb.shape[0]} rows, expected {vc.tokens} "
                         f"(the reference resizes it at training time, vision_encoder.py:36-113)")
    nl = vc.num_hidden_layers if n_tower_layers is None else n_tower_layers
    for i in range(nl):
        p = f"vision_model.encoder.layers.{i}."
        vision.layers.append(VisionLayerW(
            ln1_w=g(v, p + "layer_norm1.weight"), ln1_b=g(v, p + "layer_norm1.bias"),
            qkv_w=torch.cat([g(v, p + f"self_attn.{n}.weight") for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous(),
            qkv_b=torch.cat([g(v, p + f"self_attn.{n}.bias") for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous(),
            out_w=g(v, p + "self_attn.out_proj.weight").contiguous(), out_b=g(v, p + "self_attn.out_proj.bias"),
            ln2_w=g(v, p + "layer_norm2.weight"), ln2_b=g(v, p + "layer_norm2.bias"),
            fc1_w=g(v, p + "mlp.fc1.weight").contiguous(), fc1_b=g(v, p + "mlp.fc1.bias"),
            fc2_w=g(v, p + "mlp.fc2.weight").contiguous(), fc2_b=g(v, p + "mlp.fc2.bias")))

    region = None
    if cfg.enable_region:
        r = sd["region_extractor"]
        region = RegionW(
            deconv1_w=_deconv_as_gemm(g(r, "feature_refinement_module.0.weight")),
            deconv1_b=g(r, "feature_refinement_module.0.bias").repeat(4).contiguous(),
            ln_w=g(r, "feature_refinement_module.1.weight"), ln_b=g(r, "feature_refinement_module.1.bias"),
            deconv2_w=_deconv_as_gemm(g(r, "feature_refinement_module.3.weight")),
            deconv2_b=g(r, "feature_refinement_module.3.bias").repeat(4).contiguous(),
            rgb_w=g(r, "rgb_projector.weight").contiguous(), rgb_b=g(r, "rgb_projector.bias"),
            depth_w=g(r, "depth_projector.weight").contiguous(), depth_b=g(r, "depth_projector.bias"))

    m = sd["mm_projector"]
    ptype = cfg.mm_projector_type
    if ptype == "mlp_downsample":
        projector = ProjectorW(ln_w=g(m, "layers.1.weight"), ln_b=g(m, "layers.1.bias"),
                               fc1_w=g(m, "layers.2.weight").contiguous(), fc1_b=g(m, "layers.2.bias"),
                               fc2_w=g(m, "layers.4.weight").contiguous(), fc2_b=g(m, "layers.4.bias"))
    elif ptype == "identity":
        projector = ProjectorW()
    elif ptype == "linear":  # nn.Linear stored as `layers` itself (base_projector.py:71-72)
        projector = ProjectorW(linears=[(g(m, "layers.weight").contiguous(), g(m, "layers.bias"))])
    else:
        import re as _re
        mt = _re.match(r"^mlp(\d+)x_gelu$", ptype or "")
        if not mt:
            raise ValueError(f"Unknown projector type: {ptype}")  # base_projector.py:91
        # nn.Sequential(Linear, GELU, Linear, ...): linears sit at the even indices (base_projector.py:83-88)
        projector = ProjectorW(linears=[(g(m, f"layers.{2 * i}.weight").contiguous(), g(m, f"layers.{2 * i}.bias")) for i in range(int(mt.group(1)))])

    l, lc = sd["llm"], cfg.llama
    llama = LlamaW(embed=g(l, "model.embed_tokens.weight").contiguous(), norm=g(l, "model.norm.weight"),
                   lm_head=g(l, "lm_head.weight" if "lm_head.weight" in l else "model.embed_tokens.weight").contiguous(), quantization=quantization,
                   nf4_dequantized_copy=nf4_dequantized_copy)
    for i in range(lc.num_hidden_layers):
        p = f"model.layers.{i}."
        if quantization == "nf4":
            llama.layers.append(_nf4_layer(l, p, g, dtype, dequantized_copy=nf4_dequantized_copy))
            continue
        if quantization == "fp8":
            llama.layers.append(_fp8_layer(l, p, g, dtype))
            continue
        llama.layers.append(LlamaLayerW(
            in_norm=g(l, p + "input_layernorm.weight"),
            qkv_w=torch.cat([g(l, p + f"self_attn.{n}.weight") for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous(),
            o_w=g(l, p + "self_attn.o_proj.weight").contiguous(),
            post_norm=g(l, p + "post_attention_layernorm.weight"),
            gateup_w=interleave_rows(g(l, p + "mlp.gate_proj.weight"), g(l, p + "mlp.up_proj.weight")),
            down_w=g(l, p + "mlp.down_proj.weight").contiguous()))
    return ModelWeights(vision, region, projector, llama)


def _nf4_layer(l: Dict[str, torch.Tensor], p: str, g, dtype: torch.dtype, dequantized_copy: bool = True) -> LlamaLayerW:
    """One decoder layer with NF4 linears: each original matrix quantized and dequantized on its own, then the codes, scales and
    dequantized matrices fused exactly as the plain layer's weights (q/k/v rows concatenated, gate/up rows interleaved).
    dequantized_copy=False: a matrix with planes keeps only them (its *_w field holds the Nf4W); the layer's dequantized copies are
    freed before it returns, so a load holds at most one layer's transient copies."""
    from . import ops
    with ops.elem_dtype(dtype):
        quant = {}
        for n in ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"):
            key = p + ("self_attn." if n.endswith(("q_proj", "k_proj", "v_proj", "o_proj")) else "mlp.") + n + ".weight"
            codes, scale = ops.nf4_quantize(g(l, key).contiguous())
            quant[n] = (codes, scale, ops.nf4_dequantize(codes, scale))
        # each original matrix is released as soon as its fused form exists (the load's transient stays about one layer)
        fused = {"qkv": [torch.cat([quant[n][k] for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous() for k in range(3)]}
        for n in ("q_proj", "k_proj", "v_proj"):
            del quant[n]
        fused["o"] = list(quant.pop("o_proj"))
        fused["gateup"] = [interleave_rows(quant["gate_proj"][k], quant["up_proj"][k]) for k in range(3)]
        del quant["gate_proj"], quant["up_proj"]
        fused["down"] = list(quant.pop("down_proj"))
        planes, mats = {}, {}
        for name in ("qkv", "o", "gateup", "down"):
            codes, scale, deq = fused.pop(name)
            planes[name] = ops.nf4_planes(codes, scale, deq)[0]
            mats[name] = deq if dequantized_copy or planes[name] is None else planes[name]
            del codes, scale, deq
    return LlamaLayerW(in_norm=g(l, p + "input_layernorm.weight"), qkv_w=mats["qkv"], o_w=mats["o"],
                       post_norm=g(l, p + "post_attention_layernorm.weight"), gateup_w=mats["gateup"], down_w=mats["down"], nf4=planes)


def _fp8_layer(l: Dict[str, torch.Tensor], p: str, g, dtype: torch.dtype) -> LlamaLayerW:
    """One decoder layer with FP8 linears.  The scales are per output row, so each original matrix is quantized on its own (only one
    element-type matrix is on the device at a time) and the codes and scales are fused as the plain layer's weights are (q/k/v rows
    concatenated, gate/up rows interleaved)."""
    from . import ops
    with ops.elem_dtype(dtype):
        quant = {}
        for n in ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"):
            key = p + ("self_attn." if n.endswith(("q_proj", "k_proj", "v_proj", "o_proj")) else "mlp.") + n + ".weight"
            quant[n] = ops.fp8_quantize_weight(g(l, key).contiguous(), name=key)
        fused = {
            "qkv": [torch.cat([quant[n][k] for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous() for k in range(2)],
            "o": list(quant["o_proj"]),
            "gateup": [interleave_rows(quant["gate_proj"][0], quant["up_proj"][0]),
                       torch.stack((quant["gate_proj"][1], quant["up_proj"][1]), 1).reshape(-1).contiguous()],
            "down": list(quant["down_proj"]),
        }
        del quant
    w = {name: Fp8W(q=f[0], scale=f[1]) for name, f in fused.items()}
    return LlamaLayerW(in_norm=g(l, p + "input_layernorm.weight"), qkv_w=w["qkv"], o_w=w["o"], post_norm=g(l, p + "post_attention_layernorm.weight"),
                       gateup_w=w["gateup"], down_w=w["down"])


def random_init(cfg: LlavaConfig, device, seed: int = 0, std: float = 0.02, n_tower_layers: Optional[int] = None,
                dtype: torch.dtype = BF16) -> ModelWeights:
    """Seeded synthetic weights generated directly on the device in the kernel layouts (no 16 GB
    host staging for the 8B benchmarks; there are no checkpoints offline).  Same distributions as
    the test fixtures' weight generator but NOT the same values — parity tests go through
    ``from_state_dicts`` instead."""
    dev = torch.device(device)
    gen = torch.Generator(device=dev).manual_seed(seed)

    def rn(*shape, s=std):
        return (torch.randn(*shape, generator=gen, device=dev, dtype=torch.float32) * s).to(dtype)

    def nw(n):
        return (1.0 + 0.1 * torch.randn(n, generator=gen, device=dev)).to(dtype)

    def nb(n):
        return (0.05 * torch.randn(n, generator=gen, device=dev)).to(dtype)

    vc, lc = cfg.vision, cfg.llama
    D, I, T = vc.hidden_size, vc.intermediate_size, vc.grid * vc.grid
    if vc.is_clip:
        vision = VisionW(patch_w=_pad_cols(rn(D, 3 * vc.patch_size ** 2), patch_ldk(vc.patch_size)), patch_b=None, pos_emb=rn(T + 1, D),
                         cls_emb=rn(D), pre_ln_w=nw(D), pre_ln_b=nb(D))
    else:
        vision = VisionW(patch_w=_pad_cols(rn(D, 3 * vc.patch_size ** 2), patch_ldk(vc.patch_size)), patch_b=rn(D), pos_emb=rn(T, D))
    nl = vc.num_hidden_layers if n_tower_layers is None else n_tower_layers
    for _ in range(nl):
        vision.layers.append(VisionLayerW(nw(D), nb(D), rn(3 * D, D, s=2 * std), rn(3 * D), rn(D, D, s=2 * std), rn(D),
                                          nw(D), nb(D), rn(I, D, s=2 * std), rn(I), rn(D, I, s=2 * std), rn(D)))
    H = lc.hidden_size
    region = None
    if cfg.enable_region:
        region = RegionW(rn(4 * D, D, s=2 * std), rn(D).repeat(4).contiguous(), nw(D), nb(D), rn(4 * D, D, s=2 * std),
                         rn(D).repeat(4).contiguous(), rn(H, D, s=2 * std), rn(H), rn(H, D, s=2 * std), rn(H))
    projector = ProjectorW(nw(4 * D), nb(4 * D), rn(H, 4 * D), rn(H), rn(H, H), rn(H))
    qkv_rows = (lc.num_attention_heads + 2 * lc.num_key_value_heads) * lc.head_dim
    llama = LlamaW(embed=rn(lc.vocab_size, H, s=0.3), norm=nw(H), lm_head=rn(lc.vocab_size, H, s=4 * std))
    for _ in range(lc.num_hidden_layers):
        llama.layers.append(LlamaLayerW(nw(H), rn(qkv_rows, H), rn(H, lc.num_attention_heads * lc.head_dim), nw(H),
                                        rn(2 * lc.intermediate_size, H), rn(H, lc.intermediate_size)))
    return ModelWeights(vision, region, projector, llama)
