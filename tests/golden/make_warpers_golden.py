"""Writes tests/golden/warpers_kats.npz: transformers 5.5's warper chain (generation/logits_process.py: TemperatureLogitsWarper,
TopKLogitsWarper, TopPLogitsWarper, TypicalLogitsWarper, EpsilonLogitsWarper, EtaLogitsWarper, in _get_logits_processor's order and
with its on-conditions, min_tokens_to_keep = 1) over seeded fp32 rows of V = 1000 and V = 128256: random, peaked, flat and tied rows.
Every row is bf16-representable (the batched lm_head's rows).  Stored: the rows, the settings, HF's kept masks (packed bits) and, for
V = 1000, HF's warped rows.  Run: python -m tests.golden.make_warpers_golden"""
import os

import numpy as np
import torch
from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper,
                                                    TopPLogitsWarper, TypicalLogitsWarper)

# (temperature, top_k (0 = off), top_p, typical_p, epsilon_cutoff, eta_cutoff)
SETTINGS = [
    (1.0, 0, 1.0, 0.9, 0.0, 0.0), (0.7, 0, 1.0, 0.2, 0.0, 0.0),        # typical alone
    (1.0, 0, 1.0, 1.0, 3e-4, 0.0), (1.0, 0, 1.0, 1.0, 0.02, 0.0),      # epsilon alone
    (1.0, 0, 1.0, 1.0, 0.0, 3e-4), (1.0, 0, 1.0, 1.0, 0.0, 0.05),      # eta alone
    (0.8, 50, 0.95, 0.9, 3e-4, 2e-3), (1.2, 0, 0.9, 0.5, 1e-3, 1e-3),  # all three after temperature / top-k / top-p
]


def hf_chain(x: torch.Tensor, T, k, p, typ, eps, eta) -> torch.Tensor:
    ws = []
    if T != 1.0:
        ws.append(TemperatureLogitsWarper(T))
    if k != 0:
        ws.append(TopKLogitsWarper(k))
    if p < 1.0:
        ws.append(TopPLogitsWarper(p))
    if typ < 1.0:
        ws.append(TypicalLogitsWarper(typ))
    if 0.0 < eps < 1.0:
        ws.append(EpsilonLogitsWarper(eps))
    if 0.0 < eta < 1.0:
        ws.append(EtaLogitsWarper(eta))
    s = x[None].clone()
    for w in ws:
        s = w(None, s)
    return s[0]


def rows(V: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    out = [torch.randn(V, generator=g) * 2.0,                                             # random
           torch.randn(V, generator=g) * 0.5]                                             # peaked: a few tokens far above the rest
    out[1][torch.randperm(V, generator=g)[:8]] += torch.linspace(4.0, 9.0, 8)
    out.append(torch.zeros(V))                                                            # flat
    tied = torch.randint(0, 6, (V,), generator=g).float() * 0.75                          # six levels: every cut falls on a tie
    tied[torch.randperm(V, generator=g)[:3]] = 6.0
    out.append(tied)
    return torch.stack(out).to(torch.bfloat16).float()


def main():
    data = {"settings": np.array(SETTINGS, dtype=np.float64)}
    for V, seed in ((1000, 1), (128256, 2)):
        x = rows(V, seed)
        warped = torch.stack([torch.stack([hf_chain(r, *st) for st in SETTINGS]) for r in x])  # [rows, settings, V]
        data[f"x_{V}"] = x.to(torch.bfloat16).view(torch.int16).numpy()
        data[f"keep_{V}"] = np.packbits(torch.isfinite(warped).numpy(), axis=-1)
        if V == 1000:
            data[f"warped_{V}"] = warped.numpy()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "warpers_kats.npz")
    np.savez_compressed(path, **data)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
