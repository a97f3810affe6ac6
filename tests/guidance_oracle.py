"""Classifier-free guidance on the CPU: HF's UnbatchedClassifierFreeGuidanceLogitsProcessor (transformers generation/logits_process.py)
behind generate(guidance_scale=, negative_prompt_ids=) restated over the oracle's Llama forward (oracle/srgpt_oracle.py), as the checker
of the device path (LlamaDecoder.generate_rows with negative prompts, csrc/guidance.cu).

  * the guided row: scores = log_softmax(c), u = log_softmax(uncond[-1]), both fp32; guided = g * (scores - u) + u, three separately
    rounded fp32 operations (torch's eager ops);
  * the unconditional branch: the text model over the negative prompt ids, at positions from 0, then the tokens chosen for the prompt;
  * greedy takes the arg max of the guided row: the largest value, the lowest index on ties, NaN never wins (0 for an all-NaN row).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import srgpt_oracle as O


def guided_row(cond: torch.Tensor, uncond: torch.Tensor, g: float) -> torch.Tensor:
    """The processed row of one step from the conditional and unconditional fp32 logits rows [..., V]."""
    s = F.log_softmax(cond.float(), dim=-1)
    u = F.log_softmax(uncond.float(), dim=-1)
    gt = torch.tensor(g, dtype=torch.float32)
    return (gt * (s - u)) + u


def combine(s: torch.Tensor, u: torch.Tensor, g: float) -> torch.Tensor:
    """The three-op combine over given fp32 log-probs (sub, mul, add, each rounded)."""
    return (torch.tensor(g, dtype=torch.float32) * (s - u)) + u


def argmax_rule(row: torch.Tensor) -> int:
    """The arg max of a fp32 row: lowest index among the maxima, NaN never wins, 0 when every value is NaN."""
    r = row.float()
    ok = ~torch.isnan(r)
    if not bool(ok.any()):
        return 0
    m = r[ok].max()
    return int(torch.nonzero(ok & (r == m)).flatten()[0])


def guided_generate(cfg, w_llm: Dict[str, torch.Tensor], inputs_embeds: torch.Tensor, negative_ids: torch.Tensor, guidance_scale: float,
                    max_new_tokens: int, dtype: torch.dtype = torch.float32):
    """Guided greedy decoding of one prompt (embeddings [S, H]) with its negative prompt ids [T].  Returns (new ids, the raw conditional
    fp32 logits [n, V], the guided rows [n, V])."""
    emb = w_llm["model.embed_tokens.weight"]
    logits, cache = O.llama_forward(cfg, w_llm, inputs_embeds, None, dtype)
    ulogits, ucache = O.llama_forward(cfg, w_llm, emb[negative_ids.long()].to(dtype), None, dtype)
    ids, raw, rows = [], [], []
    for t in range(max_new_tokens):
        c, u = logits[-1].float(), ulogits[-1].float()
        row = guided_row(c, u, guidance_scale)
        nxt = argmax_rule(row)
        ids.append(nxt)
        raw.append(c)
        rows.append(row)
        if t == max_new_tokens - 1:
            break
        x = emb[nxt][None].to(dtype)
        logits, cache = O.llama_forward(cfg, w_llm, x, cache, dtype)
        ulogits, ucache = O.llama_forward(cfg, w_llm, x, ucache, dtype)
    return torch.tensor(ids, dtype=torch.long), torch.stack(raw), torch.stack(rows)
