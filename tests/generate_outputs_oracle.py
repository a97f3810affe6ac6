"""generate(output_hidden_states=True, output_attentions=True, return_dict_in_generate=True) of greedy decoding restated over the oracle's
decoder (tests/forward_outputs_oracle.py): entry 0 is forward's records of the prompt, and decode step t is forward over the prompt plus
the first t generated tokens, its last row, with the attention columns placed as HF places them in a padded batch: prompt key p at
off + p, generated key j at T + j, 0 elsewhere."""
from __future__ import annotations

import torch

from oracle import srgpt_oracle as O
from tests.forward_outputs_oracle import llama_forward_outputs


def decode_columns(n: int, off: int, T: int, t: int) -> torch.Tensor:
    """The column of each of the n + t keys of decode step t (1-based) of a prompt of n rows at padded offset off in a batch of width T."""
    return torch.cat([off + torch.arange(n), T + torch.arange(t)])


def generate_outputs(cfg: O.OracleConfig, w, prompt: torch.Tensor, n_new: int, off: int = 0, T: int = None, dtype: torch.dtype = torch.float32):
    """One prompt [n, H] decoded greedily for n_new tokens -> (ids [n_new], hidden_states, attentions) with HF's structure for this row:
    hidden_states[0] L + 1 tensors [n, H] and attentions[0] L tensors [nh, n, n] (the prompt's own block), then per decode step t
    hidden_states[t] L + 1 tensors [1, H] and attentions[t] L tensors [nh, 1, T + t] in the padded columns."""
    T = prompt.shape[0] if T is None else T
    n = prompt.shape[0]
    embed = w["model.embed_tokens.weight"].float()
    x = prompt.float()
    logits, hs, att = llama_forward_outputs(cfg, w, x, dtype)
    ids = [int(logits[-1].argmax())]
    hidden, attentions = [hs], [att]
    for t in range(1, n_new):
        x = torch.cat([x, embed[ids[-1]][None]], 0)
        logits, hs, att = llama_forward_outputs(cfg, w, x, dtype)
        hidden.append(tuple(h[-1:] for h in hs))
        cols = decode_columns(n, off, T, t)
        rows = []
        for a in att:
            full = torch.zeros(a.shape[0], 1, T + t, dtype=a.dtype)
            full[:, 0, cols] = a[:, -1]
            rows.append(full)
        attentions.append(tuple(rows))
        ids.append(int(logits[-1].argmax()))
    return torch.tensor(ids), tuple(hidden), tuple(attentions)
