"""Generate tests/golden/processor_kats.npz: HF ``LlamaForCausalLM.generate(inputs_embeds=..., **processors)`` (greedy) with the
logits processors generate() accepts (repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_new_tokens, min_length), on a stock
LlamaForCausalLM holding the oracle's seeded weights (the model of ``make_golden.py beam``).  fp32 on CPU, transformers of this image:

    python tests/golden/make_processor_golden.py

The prompt is given as token ids embedded by the model's own table, so generate(input_ids) of the text path sees the same rows.  Every
case must differ from plain greedy decoding (the processors visibly act).  Per step the processed top-1 / top-2 margin (HF's
output_scores) is recorded: tests/test_gpu_logits_processors.py compares the steps whose margin clears the bf16 / fp16 tolerance.
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

PROCESSOR_CASES = [  # (name, generate() kwargs); eos "plain3" = the plain greedy continuation's token at step 3
    ("penalty", dict(repetition_penalty=1.6)),
    ("ngram3", dict(no_repeat_ngram_size=3)),
    ("ngram2", dict(no_repeat_ngram_size=2)),
    ("ngram1", dict(no_repeat_ngram_size=1)),
    ("bad_words", dict(bad_words_ids="plain")),
    ("min_new_tokens_eos", dict(min_new_tokens=9, eos="plain3")),
    ("min_length_eos", dict(min_length=27, eos="plain3")),
    ("all", dict(repetition_penalty=1.3, no_repeat_ngram_size=3, bad_words_ids="plain", min_new_tokens=6, eos="plain3")),
]
PROCESSOR_NEW_TOKENS = 16


@torch.no_grad()
def run_processor_kats():
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
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, cfg.vocab - 3, (1, 20), generator=g)
    emb = llm.model.embed_tokens(ids)
    n_new = PROCESSOR_NEW_TOKENS

    def run(**kw):
        out = llm.generate(inputs_embeds=emb, do_sample=False, max_new_tokens=n_new, pad_token_id=0, output_scores=True,
                           return_dict_in_generate=True, **kw)
        sc = torch.stack([s[0] for s in out.scores])
        top2 = sc.topk(2, -1).values
        margin = torch.nan_to_num(top2[:, 0] - top2[:, 1], posinf=1e30)
        return out.sequences[0], margin

    plain, _ = run(eos_token_id=None)
    arrays = {"input_ids": ids[0].numpy(), "plain": plain.numpy(), "weight_seed": np.int64(BEAM_WEIGHT_SEED)}
    print("plain", plain.tolist())
    for name, kw in PROCESSOR_CASES:
        kw = dict(kw)
        eos = int(plain[3]) if kw.pop("eos", None) == "plain3" else None
        if kw.get("bad_words_ids") == "plain":  # a single token of the plain answer, a pair of it, and a pair that never matches
            kw["bad_words_ids"] = [[int(plain[2])], [int(plain[0]), int(plain[1])], [int(plain[1]), int(plain[0]) + 1]]
        out, margin = run(eos_token_id=eos, **kw)
        n = out.numel()
        assert out.tolist() != plain[:n].tolist() or n != plain.numel(), (name, "the processors did not act")
        if eos is not None:
            assert eos in plain[:4].tolist() and (eos not in out.tolist() or out.tolist().index(eos) >= kw.get("min_new_tokens", 7)), name
        arrays[f"{name}__ids"] = out.numpy()
        arrays[f"{name}__margin"] = margin.float().numpy()
        arrays[f"{name}__eos"] = np.int64(-1 if eos is None else eos)
        if "bad_words_ids" in kw:
            arrays[f"{name}__bad"] = np.array([len(b) for b in kw["bad_words_ids"]] + [t for b in kw["bad_words_ids"] for t in b], dtype=np.int64)
        print(name, kw, "eos", eos, out.tolist(), "min margin %.4f" % float(margin.min()))
    path = os.path.join(HERE, "processor_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"processor_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_processor_kats()
