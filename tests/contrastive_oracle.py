"""Contrastive search on the CPU: HF GenerationMixin.contrastive_search + _ranking_fast (transformers 4.37.2 generation/utils.py) behind
generate(penalty_alpha=, top_k=) restated over the oracle's Llama forward (oracle/srgpt_oracle.py), as the checker of the device path
(LlamaDecoder.generate_contrastive, csrc/contrastive.cu).

  * the context is the final-norm hidden state of every position so far, prompt rows included (the oracle's last residual rows through
    the final norm, what hidden_states[-1] holds);
  * per step: p = softmax of the fp32 logits row, its k largest; each candidate forwarded over the cache; pen = the largest cosine of the
    candidate's final-norm row against the context; score = (1 - alpha) * p - alpha * pen; the first index of the largest score wins;
  * the chosen candidate's cache, logits row and hidden row carry on.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import srgpt_oracle as O


def penalty(next_hidden: torch.Tensor, context: torch.Tensor) -> torch.Tensor:
    """_ranking_fast's degeneration penalty: next_hidden [k, H], context [L, H] -> [k], each normalized first, as HF does."""
    cos = (next_hidden / next_hidden.norm(dim=-1, keepdim=True)) @ (context / context.norm(dim=-1, keepdim=True)).T
    return cos.max(-1).values


def first_max(score: torch.Tensor) -> int:
    """torch.max's index: the first among the largest."""
    return int(torch.nonzero(score == score.max()).flatten()[0])


def contrastive_generate(cfg, w_llm: Dict[str, torch.Tensor], inputs_embeds: torch.Tensor, top_k: int, penalty_alpha: float,
                         max_new_tokens: int, eos_token_id=None, dtype: torch.dtype = torch.float32):
    """Contrastive search of one prompt (embeddings [S, H]).  Returns (new ids, {"topk_ids", "topk_probs", "pen", "score"} per step)."""
    emb = w_llm["model.embed_tokens.weight"]
    norm_w = w_llm["model.norm.weight"].to(dtype)

    def forward(x, cache):
        logits, cache, hs = O.llama_forward(cfg, w_llm, x, cache, dtype, return_hidden=True)
        return logits[-1].float(), cache, O.rms_norm(hs[-1], norm_w, cfg.rms_eps).float()

    logit, cache, context = forward(inputs_embeds, None)
    ids, rec = [], {"topk_ids": [], "topk_probs": [], "pen": [], "score": []}
    for _ in range(max_new_tokens):
        top_p, top_i = F.softmax(logit, dim=-1).topk(top_k)
        steps = [forward(emb[t][None].to(dtype), cache) for t in top_i.tolist()]
        nxt = torch.stack([s[2][-1] for s in steps])
        pen = penalty(nxt, context)
        score = (1.0 - penalty_alpha) * top_p - penalty_alpha * pen
        sel = first_max(score)
        for key, v in zip(rec, (top_i, top_p, pen, score)):
            rec[key].append(v)
        ids.append(int(top_i[sel]))
        if eos_token_id is not None and ids[-1] == eos_token_id:
            break
        logit, cache = steps[sel][0], steps[sel][1]
        context = torch.cat([context, nxt[sel][None]])
    return torch.tensor(ids, dtype=torch.long), {key: torch.stack(v) for key, v in rec.items()}
