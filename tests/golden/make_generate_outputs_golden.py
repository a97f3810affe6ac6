"""Generate tests/golden/generate_outputs_kats.npz: HF ``LlamaForCausalLM.generate(inputs_embeds=..., output_attentions=True,
output_hidden_states=True, return_dict_in_generate=True)``, greedy, eager attention, on a stock LlamaForCausalLM holding the oracle's
seeded weights (the model of ``make_golden.py beam``), for one prompt and for a left-padded batch of unequal prompts.  fp32 on CPU,
transformers of this image:

    python tests/golden/make_generate_outputs_golden.py

tests/test_generate_outputs_cpu.py pins tests/generate_outputs_oracle.py against it.
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

SINGLE_LEN = 9
BATCH_LENS = [9, 4, 6]  # left-padded to 9
N_NEW = 6


def _save(arrays, prefix, out):
    """HF's per-token tuples as stacked arrays: entry 0 ([L+1, B, T, H] / [L, B, nh, T, T]) and the decode entries, each attention
    entry t zero-extended to T + N_NEW - 1 columns."""
    arrays[prefix + "ids"] = out.sequences.numpy()
    arrays[prefix + "hidden0"] = torch.stack(out.hidden_states[0]).numpy()
    arrays[prefix + "attn0"] = torch.stack(out.attentions[0]).numpy()
    steps = len(out.hidden_states)
    arrays[prefix + "hidden_steps"] = torch.stack([torch.stack(out.hidden_states[t]) for t in range(1, steps)]).numpy()
    width = out.attentions[0][0].shape[-1] + N_NEW - 1
    att = [torch.nn.functional.pad(torch.stack(out.attentions[t]), (0, width - out.attentions[t][0].shape[-1])) for t in range(1, steps)]
    arrays[prefix + "attn_steps"] = torch.stack(att).numpy()


@torch.no_grad()
def run_generate_outputs_kats():
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    sd = O.make_weights(cfg, seed=BEAM_WEIGHT_SEED)
    lcfg = LlamaConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                       num_key_value_heads=cfg.kv_heads, vocab_size=cfg.vocab, rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta,
                       max_position_embeddings=4096, tie_word_embeddings=False, head_dim=cfg.head_dim, attention_bias=False, mlp_bias=False,
                       bos_token_id=1, eos_token_id=None, pad_token_id=0)
    lcfg._attn_implementation = "eager"
    llm = LlamaForCausalLM(lcfg).float().eval()
    llm.load_state_dict({k: v.float() for k, v in sd["llm"].items()}, strict=True)
    g = torch.Generator().manual_seed(1)
    kw = dict(max_new_tokens=N_NEW, min_new_tokens=N_NEW, do_sample=False, output_attentions=True, output_hidden_states=True,
              return_dict_in_generate=True, pad_token_id=0)
    arrays = {"weight_seed": np.int64(BEAM_WEIGHT_SEED), "batch_lens": np.array(BATCH_LENS, dtype=np.int64), "n_new": np.int64(N_NEW)}
    single = (torch.randn(SINGLE_LEN, cfg.hidden, generator=g) * 0.3).to(torch.bfloat16).float()
    arrays["single_embeds"] = single.numpy()
    _save(arrays, "single_", llm.generate(inputs_embeds=single[None], attention_mask=torch.ones(1, SINGLE_LEN, dtype=torch.long), **kw))
    prompts = [(torch.randn(n, cfg.hidden, generator=g) * 0.3).to(torch.bfloat16).float() for n in BATCH_LENS]
    T = max(BATCH_LENS)
    emb = torch.zeros(len(prompts), T, cfg.hidden)
    mask = torch.zeros(len(prompts), T, dtype=torch.long)
    for b, p in enumerate(prompts):
        emb[b, T - p.shape[0]:] = p
        mask[b, T - p.shape[0]:] = 1
    arrays["batch_embeds"] = emb.numpy()
    arrays["batch_mask"] = mask.numpy()
    _save(arrays, "batch_", llm.generate(inputs_embeds=emb, attention_mask=mask, **kw))
    path = os.path.join(HERE, "generate_outputs_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"generate_outputs_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_generate_outputs_kats()
