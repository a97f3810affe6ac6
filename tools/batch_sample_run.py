"""Measure sampled generation over a batch of prompts in the batched decode step (LlamaDecoder.generate_batch(sampling=...)) against the
same prompts one after the other (generate_from_embeds with the same per-row seeds) and against the greedy batched step, at Llama-3-8B
shapes: the full-depth decoder with seeded random weights, 259-row prompts, 128 new tokens (no EOS, so every run takes all steps),
temperature 0.7, top_p 0.9 and the default top_k 50, B in {1, 4, 8, 16, 32, 64}.  The arms alternate within each repetition.  Then
num_return_sequences n in {4, 16} on one prompt against the same prompt repeated n times in a batch.

Per workload and arm (medians over the repetitions after a warm-up run):
  * ms per step (the run minus its prefills, over the steps: 128 for a batch, B x 128 for the sequential arm);
  * new tokens per second summed over the rows;
  * prefill ms - CUDA events around the prefill calls;
  * device us per step of sample_rows over the B rows of the batched lm_head, from CUDA events around 200 launches.
The card name, power limit and SM clocks are read in the same run.

    python tools/batch_sample_run.py [--reps 2] [--batches 1,4,8,16,32,64] [--nrs 4,16]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder, sequence_seeds  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.beam_batch_run import EventTimer  # noqa: E402
from tools.nf4_run import card, timed  # noqa: E402

S, N, SEED = 259, 128, 1234
SAMPLING = dict(temperature=0.7, top_p=0.9, seed=SEED)


def sample_rows_us(dec, B: int, n: int = 200) -> float:
    """Device us per launch of sample_rows over B bf16 rows of the vocabulary (the batched step's lm_head rows)."""
    V = dec.dims.vocab_size
    g = torch.Generator(device="cuda").manual_seed(B)
    lg = torch.empty((B, (V + 7) // 8 * 8), dtype=dec.dtype, device="cuda")[:, :V]
    lg.copy_(torch.randn((B, V), generator=g, device="cuda") * 3)
    seeds = torch.tensor(sequence_seeds(SEED, B), dtype=torch.int64, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    dec._set_sampling(SAMPLING)
    with ops.elem_dtype(dec.dtype):
        for _ in range(10):
            ops.sample_rows(lg, dec.sample_params, seeds, step, 0, ids)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            ops.sample_rows(lg, dec.sample_params, seeds, step, 0, ids)
        b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def summarize(v, rows: int, steps: int) -> dict:
    total, pre = statistics.median(v["total_ms"]), statistics.median(v["prefill_ms"])
    return {"total_ms": round(total, 1), "prefill_ms": round(pre, 2), "ms_per_step": round((total - pre) / steps, 3),
            "new_tokens_per_s": round(rows * N / (total / 1e3), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batches", default="1,4,8,16,32,64")
    ap.add_argument("--nrs", default="4,16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batch_sample_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(d, w, max_seq_len=1024)
    batches = [int(b) for b in args.batches.split(",")]
    nrs = [int(n) for n in args.nrs.split(",") if n]
    g = torch.Generator().manual_seed(7)
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g)) for _ in range(max(batches + nrs))]
    prefill = EventTimer(dec.prefill_packed)
    prefill_one = EventTimer(dec.prefill_hidden)
    dec.prefill_packed, dec.prefill_hidden = prefill, prefill_one
    out = {"card": card(), "prompt_rows": S, "new_tokens": N, "sampling": {**SAMPLING, "top_k": 50}, "reps": args.reps, "by_batch": {},
           "num_return_sequences": {}}

    def sequential(B):
        seeds = sequence_seeds(SEED, B)
        return [dec.generate_from_embeds(prompts[b], N, sampling=dict(SAMPLING, seed=seeds[b])) for b in range(B)]

    for i, B in enumerate(batches):
        x = torch.cat(prompts[:B])
        arms = {"batched": lambda: dec.generate_batch(x, [S] * B, N, sampling=SAMPLING),
                "sequential": lambda: sequential(B),
                "greedy_batched": lambda: dec.generate_batch(x, [S] * B, N)}
        res = {a: {"total_ms": [], "prefill_ms": []} for a in arms}
        ids = {}
        for rep in range(1 + args.reps):  # round 0 warms the graphs up (the sequential arm's graph once)
            for arm, fn in arms.items():
                if rep == 0 and arm == "sequential" and i > 0:
                    continue
                prefill.take_ms(); prefill_one.take_ms()
                t, r = timed(fn)
                ids[arm] = [v.tolist() for v in r]
                if rep == 0:
                    continue
                res[arm]["total_ms"].append(t * 1e3)
                res[arm]["prefill_ms"].append(sum(prefill.take_ms()) + sum(prefill_one.take_ms()))
        row = {arm: summarize(v, B, N if arm != "sequential" else B * N) for arm, v in res.items()}
        row["batched"]["sample_rows_us_per_step"] = round(sample_rows_us(dec, B), 1)
        row["speedup_vs_sequential"] = round(row["sequential"]["total_ms"] / row["batched"]["total_ms"], 2)
        row["step_vs_greedy"] = round(row["batched"]["ms_per_step"] / row["greedy_batched"]["ms_per_step"], 3)
        row["rows_with_equal_ids"] = sum(a == b for a, b in zip(ids["batched"], ids["sequential"]))
        out["by_batch"][B] = row
        print(f"B={B}: {row}", file=sys.stderr, flush=True)
    for n in nrs:
        p = prompts[0]
        arms = {"num_return_sequences": lambda: dec.generate_batch(p, [S], N, sampling=SAMPLING, num_return_sequences=n),
                "repeated_prompt": lambda: dec.generate_batch(p.repeat(n, 1), [S] * n, N, sampling=SAMPLING)}
        res = {a: {"total_ms": [], "prefill_ms": []} for a in arms}
        ids = {}
        for rep in range(1 + args.reps):
            for arm, fn in arms.items():
                prefill.take_ms()
                t, r = timed(fn)
                ids[arm] = [v.tolist() for v in r]
                if rep == 0:
                    continue
                res[arm]["total_ms"].append(t * 1e3)
                res[arm]["prefill_ms"].append(sum(prefill.take_ms()))
        row = {arm: summarize(v, n, N) for arm, v in res.items()}
        row["sample_rows_us_per_step"] = round(sample_rows_us(dec, n), 1)
        row["prefill_saving_ms"] = round(row["repeated_prompt"]["prefill_ms"] - row["num_return_sequences"]["prefill_ms"], 2)
        row["rows_with_equal_ids"] = sum(a == b for a, b in zip(ids["num_return_sequences"], ids["repeated_prompt"]))
        out["num_return_sequences"][n] = row
        print(f"n={n}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
