"""Generate tests/golden/forward_outputs_kats.npz: HF ``LlamaForCausalLM(inputs_embeds=..., output_hidden_states=True,
output_attentions=True)`` with eager attention, on a stock LlamaForCausalLM holding the oracle's seeded weights (the model of
``make_golden.py beam``), for one prompt and for a left-padded batch of unequal prompts.  fp32 on CPU, transformers of this image:

    python tests/golden/make_forward_outputs_golden.py

tests/test_forward_outputs_cpu.py pins tests/forward_outputs_oracle.py against it.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import srgpt_oracle as O  # noqa: E402
from tests.golden.make_golden import BEAM_WEIGHT_SEED, CASES  # noqa: E402

SINGLE_LEN = 11
BATCH_LENS = [11, 4, 8]  # left-padded to 11


@torch.no_grad()
def run_forward_outputs_kats():
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    sd = O.make_weights(cfg, seed=BEAM_WEIGHT_SEED)
    lcfg = LlamaConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                       num_key_value_heads=cfg.kv_heads, vocab_size=cfg.vocab, rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta,
                       max_position_embeddings=4096, tie_word_embeddings=False, head_dim=cfg.head_dim, attention_bias=False, mlp_bias=False,
                       bos_token_id=1, eos_token_id=None, pad_token_id=None)
    lcfg._attn_implementation = "eager"
    llm = LlamaForCausalLM(lcfg).float().eval()
    llm.load_state_dict({k: v.float() for k, v in sd["llm"].items()}, strict=True)
    g = torch.Generator().manual_seed(0)
    arrays = {"weight_seed": np.int64(BEAM_WEIGHT_SEED), "batch_lens": np.array(BATCH_LENS, dtype=np.int64)}
    single = (torch.randn(SINGLE_LEN, cfg.hidden, generator=g) * 0.3).to(torch.bfloat16).float()
    out = llm(inputs_embeds=single[None], output_hidden_states=True, output_attentions=True)
    arrays["single_embeds"] = single.numpy()
    arrays["single_hidden"] = torch.stack(out.hidden_states)[:, 0].numpy()
    arrays["single_attn"] = torch.stack(out.attentions)[:, 0].numpy()
    arrays["single_logits"] = out.logits[0].numpy()
    prompts = [(torch.randn(n, cfg.hidden, generator=g) * 0.3).to(torch.bfloat16).float() for n in BATCH_LENS]
    T = max(BATCH_LENS)
    emb = torch.zeros(len(prompts), T, cfg.hidden)
    mask = torch.zeros(len(prompts), T, dtype=torch.long)
    for b, p in enumerate(prompts):
        emb[b, T - p.shape[0]:] = p
        mask[b, T - p.shape[0]:] = 1
    out = llm(inputs_embeds=emb, attention_mask=mask, output_hidden_states=True, output_attentions=True)
    arrays["batch_embeds"] = emb.numpy()
    arrays["batch_mask"] = mask.numpy()
    arrays["batch_hidden"] = torch.stack(out.hidden_states).numpy()
    arrays["batch_attn"] = torch.stack(out.attentions).numpy()
    path = os.path.join(HERE, "forward_outputs_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"forward_outputs_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_forward_outputs_kats()
