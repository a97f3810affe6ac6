"""Generate tests/golden/output_scores_kats.npz: HF ``LlamaForCausalLM.generate(inputs_embeds=..., return_dict_in_generate=True,
output_scores=True)`` and ``compute_transition_scores`` on a stock LlamaForCausalLM holding the oracle's seeded weights (the model of
``make_golden.py beam``).  fp32 on CPU, transformers of this image:

    python tests/golden/make_output_scores_golden.py

Cases: greedy with logits processors (one prompt), beam search over one prompt, and beam search over two prompts of the same length (no
padding).  Per case: the ids, every step's scores, the transition scores and, for beams, sequences_scores and beam_indices.  Per step
the top-1 / top-2 margin of the scores is recorded: tests/test_gpu_output_scores.py compares ids and beam indices on the steps whose
margin clears the bf16 / fp16 tolerance.
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
SCORE_CASES = [  # (name, number of prompts, generate() kwargs)
    ("greedy_proc", 1, dict(repetition_penalty=1.3, no_repeat_ngram_size=3, max_new_tokens=12)),
    ("beam1", 1, dict(num_beams=3, max_new_tokens=8, length_penalty=1.0)),
    ("beam2", 2, dict(num_beams=3, max_new_tokens=8, length_penalty=0.7)),
]


def prompts(n: int, vocab: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(11)
    return torch.randint(3, vocab - 3, (n, PROMPT_LEN), generator=g)


@torch.no_grad()
def run_output_scores_kats():
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
    arrays = {"weight_seed": np.int64(BEAM_WEIGHT_SEED), "input_ids": prompts(2, cfg.vocab).numpy()}
    for name, n, kw in SCORE_CASES:
        ids = torch.from_numpy(arrays["input_ids"][:n])
        out = llm.generate(inputs_embeds=llm.model.embed_tokens(ids), do_sample=False, pad_token_id=0, eos_token_id=None,
                           return_dict_in_generate=True, output_scores=True, **kw)
        sc = torch.stack(out.scores)  # [steps, rows, V]
        top2 = sc.topk(2, -1).values
        beams = getattr(out, "beam_indices", None)
        trans = llm.compute_transition_scores(out.sequences, out.scores, beams, normalize_logits=False)
        arrays[f"{name}__ids"] = out.sequences.numpy()
        arrays[f"{name}__scores"] = sc.float().numpy()
        arrays[f"{name}__margin"] = torch.nan_to_num(top2[..., 0] - top2[..., 1], posinf=1e30).float().numpy()
        arrays[f"{name}__transition"] = trans.float().numpy()
        if beams is not None:
            arrays[f"{name}__beam_indices"] = beams.numpy()
            arrays[f"{name}__sequences_scores"] = out.sequences_scores.float().numpy()
        print(name, out.sequences.tolist(), None if beams is None else beams.tolist())
    path = os.path.join(HERE, "output_scores_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"output_scores_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_output_scores_kats()
