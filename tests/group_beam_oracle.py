"""Diverse (group) beam search on the CPU: HF GenerationMixin.group_beam_search + HammingDiversityLogitsProcessor + BeamSearchScorer
(transformers 4.37.2 generation/utils.py, logits_process.py, beam_search.py; 5.5 removed them) behind generate(num_beams=k,
num_beam_groups=G, diversity_penalty=lambda), restated over the oracle's Llama forward (oracle/srgpt_oracle.py) as the checker of the
device path (LlamaDecoder.generate_beam_batch with num_beam_groups, csrc/beam.cu group_select_kernel).

  * groups: gs = k // G; beam i belongs to group i // gs; the beam scores start at 0 on the first beam of every group
    (beam_scores[:, ::gs] = 0) and -1e9 elsewhere;
  * one step: the model runs once over all k beams; then for g = 0 .. G-1 in order: the group's rows of log_softmax(logits.float()),
    minus diversity_penalty * (how often groups 0 .. g-1 chose the token in this step) in fp32 (fl(logp - fl(lambda * c))), plus the
    beam score; the top max(2, 1 + n_eos) * gs of the group's flattened [gs x V] table, ties (score desc, beam asc, token asc);
    BeamSearchScorer.process for the group with its own hypothesis list of size gs: an EOS of rank < gs closes a hypothesis, the first
    gs non-EOS candidates become the next beams; a group that is done emits pad_token_id (default: the first EOS id) from its first
    beam, and that token counts for the later groups' penalty too;
  * done, finalize and stop: each group is done when its list is full and (early_stopping or its worst kept score >= the best
    candidate score of this step / cur_len ** length_penalty); the run ends when every group is done, at max_new_tokens, or when the
    stopping criterion holds for every running beam; at finalize the open beams of every group that is not done become hypotheses,
    and the answer is the last of all groups' hypotheses (in group order) after a stable sort by score, so a tie goes to the later
    group; the first EOS is appended when it is shorter than max_new_tokens.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import srgpt_oracle as O


class Hyps:
    """BeamHypotheses of beam_search.py for one group: at most n kept, the worst dropped first (the first of equal scores)."""

    def __init__(self, n: int, length_penalty: float, early_stopping: bool):
        self.n, self.lp, self.es = n, length_penalty, early_stopping
        self.beams: List = []  # (score, tokens) in insertion order
        self.worst = 1e9

    def add(self, sum_logprobs: float, toks: List[int], gen_len: int) -> None:
        score = sum_logprobs / (gen_len ** self.lp)
        if len(self.beams) < self.n or score > self.worst:
            self.beams.append((score, toks))
            if len(self.beams) > self.n:
                del self.beams[min(range(len(self.beams)), key=lambda j: (self.beams[j][0], j))]
            self.worst = min(s for s, _ in self.beams)

    def is_done(self, best_sum_logprobs: float, cur_len: int) -> bool:
        if len(self.beams) < self.n:
            return False
        return self.es or self.worst >= best_sum_logprobs / (cur_len ** self.lp)


def group_beam_search(first_logits: torch.Tensor, advance: Callable[[List[int], List[int]], torch.Tensor], num_beams: int,
                      num_beam_groups: int, diversity_penalty: float, max_new_tokens: int, eos_token_id=None, length_penalty: float = 1.0,
                      early_stopping: bool = False, pad_token_id: Optional[int] = None, stopping_fn=None) -> Dict:
    """The loop over given logits: first_logits [V] (the prompt's last row), advance(parents, tokens) -> the [k, V] logits of the next
    step once beam i continues beam parents[i] with tokens[i].  Returns {"ids": the answer, "steps": per step and group the ranked
    candidates [(score, beam in group, token)] (None for a done group) and the chosen (parent, token) of every beam}."""
    eos = [] if eos_token_id is None else (list(eos_token_id) if isinstance(eos_token_id, (list, tuple, set)) else [int(eos_token_id)])
    pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)
    k, G = num_beams, num_beam_groups
    gs = k // G
    n_keep = max(2, 1 + len(eos)) * gs
    logits = first_logits.float()[None].expand(k, -1)
    V = logits.shape[1]
    beam_scores = torch.full((k,), -1e9, dtype=torch.float32)
    beam_scores[::gs] = 0.0
    seqs: List[List[int]] = [[] for _ in range(k)]
    hyps = [Hyps(gs, length_penalty, early_stopping) for _ in range(G)]
    done = [False] * G
    steps = []
    for step in range(max_new_tokens):
        cur_len = step + 1
        logp = F.log_softmax(logits.float(), dim=-1)
        current = torch.zeros(k, dtype=torch.long)
        parents = list(range(k))
        new_scores = beam_scores.clone()
        rec = {"ranked": [], "chosen": []}
        for g in range(G):
            lo = g * gs
            if done[g]:  # process: pad_token_id for every beam, from index 0 of the group
                current[lo:lo + gs] = pad
                parents[lo:lo + gs] = [lo] * gs
                new_scores[lo:lo + gs] = 0.0
                rec["ranked"].append(None)
                continue
            scores = logp[lo:lo + gs].clone()
            if g > 0:  # HammingDiversityLogitsProcessor
                scores -= diversity_penalty * torch.bincount(current[:lo], minlength=V)
            table = (scores + beam_scores[lo:lo + gs, None]).view(-1)
            order = torch.sort(-table, stable=True).indices[:n_keep].tolist()  # (score desc, flat index asc) = (beam asc, token asc)
            ranked = [(float(table[fi]), fi // V, fi % V) for fi in order]
            rec["ranked"].append(ranked)
            nxt = []
            for rank, (sc, b, t) in enumerate(ranked):
                if t in eos:
                    if rank >= gs:
                        continue
                    hyps[g].add(sc, list(seqs[lo + b]), cur_len)
                else:
                    nxt.append((sc, b, t))
                if len(nxt) == gs:
                    break
            assert len(nxt) == gs, "beam search ran out of non-EOS candidates"
            done[g] = done[g] or hyps[g].is_done(ranked[0][0], cur_len)
            for i, (sc, b, t) in enumerate(nxt):
                current[lo + i] = t
                parents[lo + i] = lo + b
                new_scores[lo + i] = sc
        rec["chosen"] = list(zip(parents, current.tolist()))
        steps.append(rec)
        seqs = [seqs[parents[i]] + [int(current[i])] for i in range(k)]
        beam_scores = new_scores
        if all(done) or step == max_new_tokens - 1:
            break
        if stopping_fn is not None and all(stopping_fn(torch.tensor(seqs[g * gs + i], dtype=torch.long))
                                           for g in range(G) if not done[g] for i in range(gs)):
            break
        logits = advance(parents, current.tolist())
    for g in range(G):
        if not done[g]:
            for i in range(gs):
                hyps[g].add(float(beam_scores[g * gs + i]), list(seqs[g * gs + i]), len(seqs[g * gs + i]))
    best = list(sorted((h for hy in hyps for h in hy.beams), key=lambda h: h[0])[-1][1])
    if len(best) < max_new_tokens and eos:
        best.append(eos[0])
    return {"ids": best, "steps": steps}


def group_beam_generate(cfg, w_llm: Dict[str, torch.Tensor], inputs_embeds: torch.Tensor, num_beams: int, num_beam_groups: int,
                        diversity_penalty: float, max_new_tokens: int, eos_token_id=None, length_penalty: float = 1.0,
                        early_stopping: bool = False, pad_token_id: Optional[int] = None, stopping_fn=None,
                        dtype: torch.dtype = torch.float32) -> Dict:
    """Diverse beam search of one prompt given as embeddings [S, H] over the oracle's model (new ids only)."""
    emb = w_llm["model.embed_tokens.weight"]
    logits, cache = O.llama_forward(cfg, w_llm, inputs_embeds, None, dtype)
    caches = [cache] * num_beams  # llama_forward never mutates a cache it is given

    def advance(parents: List[int], tokens: List[int]) -> torch.Tensor:
        rows, new = [], []
        for p, t in zip(parents, tokens):
            lg, c = O.llama_forward(cfg, w_llm, emb[t][None].to(dtype), caches[p], dtype)
            rows.append(lg[-1].float())
            new.append(c)
        caches[:] = new
        return torch.stack(rows)

    return group_beam_search(logits[-1], advance, num_beams, num_beam_groups, diversity_penalty, max_new_tokens, eos_token_id,
                             length_penalty, early_stopping, pad_token_id, stopping_fn)
