"""Generate tests/golden/cfg_kats.npz: HF ``LlamaForCausalLM.generate(inputs_embeds=..., guidance_scale=g, negative_prompt_ids=...,
do_sample=False, return_dict_in_generate=True, output_scores=True, output_logits=True)`` on a stock LlamaForCausalLM holding the oracle's
seeded weights (the model of ``make_output_scores_golden.py``).  fp32 on CPU, transformers of this image:

    python tests/golden/make_cfg_golden.py

Cases: g in {0.5, 1.5, 3.0}; one prompt and two prompts, unpadded negative prompts, one negative prompt longer than its prompt.  Per
case: the prompt ids, the negative prompt ids, the new ids, every step's guided rows (HF's scores) and raw logits, and the top-1 / top-2
margin of each guided row.
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

PROMPT_LEN = 20
MAX_NEW = 10
CFG_CASES = [  # (name, guidance scale, number of prompts, negative prompt length)
    ("g0.5_b1", 0.5, 1, 8),
    ("g1.5_b1_long", 1.5, 1, 28),  # the negative prompt is longer than its prompt
    ("g3.0_b1", 3.0, 1, 6),
    ("g1.5_b2", 1.5, 2, 8),
    ("g3.0_b2", 3.0, 2, 12),
]


def model():
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
    return cfg, sd, llm


@torch.no_grad()
def run_cfg_kats():
    cfg, _, llm = model()
    g = torch.Generator().manual_seed(23)
    arrays = {"weight_seed": np.int64(BEAM_WEIGHT_SEED), "max_new": np.int64(MAX_NEW)}
    for name, scale, n, t_neg in CFG_CASES:
        ids = torch.randint(3, cfg.vocab - 3, (n, PROMPT_LEN), generator=g)
        neg = torch.randint(3, cfg.vocab - 3, (n, t_neg), generator=g)
        out = llm.generate(inputs_embeds=llm.model.embed_tokens(ids), guidance_scale=scale, negative_prompt_ids=neg, do_sample=False,
                           max_new_tokens=MAX_NEW, min_new_tokens=0, pad_token_id=0, eos_token_id=None, return_dict_in_generate=True,
                           output_scores=True, output_logits=True)
        sc = torch.stack(out.scores)  # [steps, rows, V]
        top2 = sc.topk(2, -1).values
        arrays[f"{name}__scale"] = np.float32(scale)
        arrays[f"{name}__input_ids"] = ids.numpy()
        arrays[f"{name}__negative_ids"] = neg.numpy()
        arrays[f"{name}__ids"] = out.sequences.numpy()
        arrays[f"{name}__scores"] = sc.float().numpy()
        arrays[f"{name}__logits"] = torch.stack(out.logits).float().numpy()
        arrays[f"{name}__margin"] = (top2[..., 0] - top2[..., 1]).float().numpy()
        print(name, out.sequences.tolist(), float(arrays[f"{name}__margin"].min()))
    path = os.path.join(HERE, "cfg_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"cfg_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_cfg_kats()
