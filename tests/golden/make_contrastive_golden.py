"""Generate tests/golden/contrastive_kats.npz: contrastive search (transformers 4.37.2 ``GenerationMixin.contrastive_search`` +
``_ranking_fast``, reached through ``generate(penalty_alpha=a, top_k=k)``) over the stock ``LlamaForCausalLM`` of this image holding the
oracle's seeded weights (the model of ``make_cfg_golden.py``), fp32 on CPU:

    python tests/golden/make_contrastive_golden.py

The transformers of this image no longer ships contrastive search, so the loop is restated below from 4.37.2: the prompt's forward with
output_hidden_states=True gives the context (hidden_states[-1], after the final norm) and the first logits row; every step forwards
each of the k most probable tokens as its own batch-1 step over a deep copy of the cache.  A batch of unpadded, equal-length prompts
is the same computation per prompt, so each prompt of a case runs on its own.

Cases: (k, alpha) in {(2, 0.3), (4, 0.6), (6, 0.9)}, each with one prompt, two equal-length prompts, one prompt of more than 64 rows,
and one prompt whose third token is then used as its EOS id.  Per case: the prompt ids, the new ids and, per prompt and step, the
top-k ids and probabilities, the penalties, the scores and the margin between the best and the second-best score.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from tests.golden.make_cfg_golden import model  # noqa: E402

MAX_NEW = 12
SETTINGS = [(2, 0.3), (4, 0.6), (6, 0.9)]
SHAPES = [("b1", 1, 20), ("b2", 2, 20), ("long", 1, 80), ("eos", 1, 24)]  # (name, prompts, prompt length)


@torch.no_grad()
def contrastive_search(llm, ids: torch.Tensor, k: int, alpha: float, max_new: int, eos=None):
    """One prompt (ids [S]) -> (new ids, per-step top-k ids, probabilities, penalties, scores)."""
    out = llm(input_ids=ids[None], use_cache=True, output_hidden_states=True)
    assert torch.allclose(llm.lm_head(out.hidden_states[-1]), out.logits, atol=1e-5)  # hidden_states[-1] is after the final norm
    past, context, logit_next = out.past_key_values, out.hidden_states[-1][0], out.logits[0, -1].float()
    new, rec = [], {"topk_ids": [], "topk_probs": [], "pen": [], "score": []}
    for _ in range(max_new):
        top_p, top_i = logit_next.softmax(-1).topk(k)
        steps = [llm(input_ids=t.view(1, 1), past_key_values=copy.deepcopy(past), use_cache=True, output_hidden_states=True) for t in top_i]
        nxt = torch.stack([o.hidden_states[-1][0, -1] for o in steps])  # [k, H]
        cos = (nxt / nxt.norm(dim=-1, keepdim=True)) @ (context / context.norm(dim=-1, keepdim=True)).T  # [k, L]
        pen = cos.max(-1).values
        score = (1.0 - alpha) * top_p - alpha * pen
        sel = int(torch.nonzero(score == score.max()).flatten()[0])  # torch.max: the first index on ties
        for key, v in zip(rec, (top_i, top_p, pen, score)):
            rec[key].append(v)
        new.append(int(top_i[sel]))
        if eos is not None and new[-1] == eos:
            break
        past, logit_next = steps[sel].past_key_values, steps[sel].logits[0, -1].float()
        context = torch.cat([context, nxt[sel][None]])
    return new, {key: torch.stack(v) for key, v in rec.items()}


@torch.no_grad()
def run_contrastive_kats():
    cfg, _, llm = model()
    g = torch.Generator().manual_seed(31)
    arrays = {"max_new": np.int64(MAX_NEW)}
    for k, alpha in SETTINGS:
        for shape, n, S in SHAPES:
            name = f"k{k}_a{alpha}_{shape}"
            ids = torch.randint(3, cfg.vocab - 3, (n, S), generator=g)
            eos = None
            if shape == "eos":  # the prompt's own third token becomes its EOS id, so the run stops there
                eos = contrastive_search(llm, ids[0], k, alpha, 3)[0][2]
            arrays[f"{name}__k"] = np.int64(k)
            arrays[f"{name}__alpha"] = np.float64(alpha)
            arrays[f"{name}__eos"] = np.int64(-1 if eos is None else eos)
            arrays[f"{name}__input_ids"] = ids.numpy()
            for b in range(n):
                new, rec = contrastive_search(llm, ids[b], k, alpha, MAX_NEW, eos)
                top2 = rec["score"].topk(2, -1).values
                arrays[f"{name}__ids{b}"] = np.array(new, dtype=np.int64)
                for key, v in rec.items():
                    arrays[f"{name}__{key}{b}"] = v.numpy()
                arrays[f"{name}__margin{b}"] = (top2[:, 0] - top2[:, 1]).numpy()
                print(name, b, new, float(arrays[f"{name}__margin{b}"].min()))
    path = os.path.join(HERE, "contrastive_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"contrastive_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_contrastive_kats()
