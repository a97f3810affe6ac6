"""forward(output_hidden_states=True, output_attentions=True) restated over the oracle's decoder (oracle.srgpt_oracle.llama_forward, whose
default result this leaves alone): the same layer arithmetic, with HF LlamaModel's records.  hidden_states: L + 1 tensors [S, H], the
embeddings, the residual stream after each layer but the last, and the final norm.  attentions: L tensors [nh, S, S], each layer's
softmax(Q K^T * hd^-0.5 + causal mask) in fp32, cast to ``dtype``."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import srgpt_oracle as O


def llama_forward_outputs(cfg: O.OracleConfig, w, inputs_embeds: torch.Tensor, dtype: torch.dtype = torch.float32):
    """One unpadded sequence inputs_embeds [S, H] -> (fp32 logits [S, V], hidden_states tuple, attentions tuple)."""
    W = lambda k: w[k].to(dtype)  # noqa: E731
    x = inputs_embeds.to(dtype)
    S = x.shape[0]
    cos, sin = O.rope_cos_sin(cfg, torch.arange(S), dtype)
    nh, nkv, hd = cfg.heads, cfg.kv_heads, cfg.head_dim
    hidden, attentions = [x], []
    causal = torch.arange(S)[None, :] <= torch.arange(S)[:, None]
    for i in range(cfg.layers):
        p = f"model.layers.{i}."
        h = O.rms_norm(x, W(p + "input_layernorm.weight"), cfg.rms_eps)
        q = F.linear(h, W(p + "self_attn.q_proj.weight")).view(S, nh, hd).transpose(0, 1)
        k = F.linear(h, W(p + "self_attn.k_proj.weight")).view(S, nkv, hd).transpose(0, 1)
        v = F.linear(h, W(p + "self_attn.v_proj.weight")).view(S, nkv, hd).transpose(0, 1)
        q = (q * cos[None]) + (O.rotate_half(q) * sin[None])
        k = (k * cos[None]) + (O.rotate_half(k) * sin[None])
        kk, vv = k.repeat_interleave(nh // nkv, dim=0), v.repeat_interleave(nh // nkv, dim=0)
        att = torch.matmul(q, kk.transpose(-1, -2)).float() * (hd ** -0.5)
        att = F.softmax(att.masked_fill(~causal[None], float("-inf")), dim=-1).to(dtype)
        attentions.append(att)
        o = F.linear(torch.matmul(att, vv).transpose(0, 1).reshape(S, nh * hd), W(p + "self_attn.o_proj.weight"))
        x = x + o
        h = O.rms_norm(x, W(p + "post_attention_layernorm.weight"), cfg.rms_eps)
        h = F.linear(F.silu(F.linear(h, W(p + "mlp.gate_proj.weight"))) * F.linear(h, W(p + "mlp.up_proj.weight")), W(p + "mlp.down_proj.weight"))
        x = x + h
        if i < cfg.layers - 1:
            hidden.append(x)
    x = O.rms_norm(x, W("model.norm.weight"), cfg.rms_eps)
    hidden.append(x)
    return F.linear(x, W("lm_head.weight")).float(), tuple(hidden), tuple(attentions)
