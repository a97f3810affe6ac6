"""Measure likelihood scoring (LlamaDecoder.score_candidates, behind LlavaLlamaModel.score) at Llama-3-8B shapes: the full-depth decoder
with seeded random weights, one 259-row prompt and 1203 candidates (the size of the LVIS category list) whose lengths of 1-4 tokens
are drawn from a seeded histogram, against generate(max_new_tokens=8) on the same prompt.

Per call (medians over the repetitions after a warm-up call):
  * score ms - a host clock around the call, ending in a device synchronise;
  * its split, from CUDA events around each part's call: the prompt prefill, the candidates' chunked prefill, final norm + lm_head,
    and token_logprobs (the row log-sum-exp and the gather kernels, with the host's pair checks and upload);
  * the kernel's own time and GB/s over the largest pass's logits rows, from CUDA events around 20 launches back to back,
    bytes = rows x V x element size (the logits it reads once);
  * generate(max_new_tokens=8) ms on the same prompt.
The card name, power limit and SM clocks are read in the same run.

    python tools/score_run.py [--reps 3] [--candidates 1203]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.beam_batch_run import EventTimer  # noqa: E402
from tools.nf4_run import card, timed  # noqa: E402

S = 259
LENGTH_HISTOGRAM = [0.3, 0.4, 0.2, 0.1]  # P(length = 1, 2, 3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--candidates", type=int, default=1203)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(d, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    prompt = dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g))
    lens = (torch.multinomial(torch.tensor(LENGTH_HISTOGRAM), args.candidates, replacement=True, generator=g) + 1).tolist()
    cands = [torch.randint(1000, 30000, (n,), generator=g).tolist() for n in lens]
    free_b, _ = torch.cuda.mem_get_info()
    per_row = 2 * ((d.vocab_size + 7) // 8 * 8 + 3 * d.hidden_size + (2 * d.num_attention_heads + 2 * d.num_key_value_heads) * d.head_dim
                   + d.intermediate_size)
    row_budget = int(max(3, min(8192, free_b // 4 // per_row)))  # the rule of LlavaLlamaModel._score_row_budget

    parts = {"prompt_prefill": EventTimer(dec.prefill_packed), "candidate_prefill": EventTimer(ops.llama_prefill_chunk_layers),
             "lm_head": EventTimer(dec.lm_head_rows), "token_logprobs": EventTimer(ops.token_logprobs)}
    dec.prefill_packed, dec.lm_head_rows = parts["prompt_prefill"], parts["lm_head"]
    ops.llama_prefill_chunk_layers, ops.token_logprobs = parts["candidate_prefill"], parts["token_logprobs"]
    kernel_rows = []

    def score():
        return dec.score_candidates(prompt, [S], cands, row_budget)

    real_tl = parts["token_logprobs"].fn

    def counting(lg, *a, **k):
        kernel_rows.append(lg.shape[0])
        return real_tl(lg, *a, **k)

    parts["token_logprobs"].fn = counting
    res = {k: [] for k in ("score_ms", "generate8_ms", *parts)}
    ref = None
    for rep in range(1 + args.reps):
        for p in parts.values():
            p.take_ms()
        kernel_rows.clear()
        t, out = timed(score)
        ms = {k: p.take_ms() for k, p in parts.items()}
        if ref is None:
            ref = out
        assert torch.equal(out, ref), "score_candidates is not reproducible"
        t8, _ = timed(lambda: dec.generate_from_embeds(prompt, 8))
        if rep == 0:
            continue
        res["score_ms"].append(t * 1e3)
        res["generate8_ms"].append(t8 * 1e3)
        for k, v in ms.items():
            res[k].append(sum(v))
    med = {k: round(statistics.median(v), 2) for k, v in res.items()}
    n_rows = sum(n - 1 for n in lens)
    R, V, esz = max(kernel_rows), d.vocab_size, torch.finfo(dec.dtype).bits // 8
    lg = torch.empty((R, (V + 7) // 8 * 8), dtype=dec.dtype, device="cuda")[:, :V]
    lg.copy_(torch.randn((R, V), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda") * 3)
    rows, tg = list(range(R)), torch.randint(0, V, (R,), generator=g)
    with ops.elem_dtype(dec.dtype):
        for _ in range(3):
            real_tl(lg, rows, tg)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            real_tl(lg, rows, tg)
        b.record()
    torch.cuda.synchronize()
    kernel_us = a.elapsed_time(b) * 1e3 / 20
    result = {"card": card(), "prompt_rows": S, "candidates": args.candidates, "candidate_rows": n_rows, "row_budget": row_budget,
              "length_histogram": {i + 1: lens.count(i + 1) for i in range(len(LENGTH_HISTOGRAM))}, "reps": args.reps, "ms": med,
              "token_logprobs_launches_per_score": len(kernel_rows), "token_logprobs_rows_per_score": sum(kernel_rows),
              "kernel_rows": R, "kernel_us": round(kernel_us, 1), "kernel_GBps": round(R * V * esz / (kernel_us * 1e-6) / 1e9, 1),
              "score_vs_generate8": round(med["score_ms"] / med["generate8_ms"], 2)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
