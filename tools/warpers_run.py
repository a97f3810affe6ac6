"""Measure typical / epsilon / eta sampling at Llama-3-8B shapes (V = 128256): the full-depth decoder with seeded random weights, a
259-row prompt, 64 new tokens, temperature 0.7, top_p 0.9 and the default top_k 50, at B = 1 (generate_from_embeds) and B = 32
(generate_batch).  Arms: every warper off (today's sampler), typical_p = 0.9, epsilon_cutoff = 3e-4, eta_cutoff = 2e-3, and all three.

Per B and arm (medians over the repetitions after a warm-up run; the arms alternate within each repetition):
  * sampler us per step: CUDA events around 200 launches of the step's sampler over B bf16 rows of the vocabulary (the batch-1 step's
    one-row fp32 sampler at B = 1, sample_rows over the batched lm_head's rows at B = 32);
  * decode ms per step: CUDA events around the run minus its prefill, over the steps.
The card name, power limit and SM clocks are read in the same run.

    python tools/warpers_run.py [--reps 3] [--batches 1,32]   (one JSON line on stdout)
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
from tools.nf4_run import card  # noqa: E402

S, N, SEED = 259, 64, 1234
BASE = dict(temperature=0.7, top_p=0.9, seed=SEED)
ARMS = {"off": {}, "typical": dict(typical_p=0.9), "epsilon": dict(epsilon_cutoff=3e-4), "eta": dict(eta_cutoff=2e-3),
        "all": dict(typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=2e-3)}


def sampler_us(dec, B: int, arm: dict, n: int = 200) -> float:
    """Device us per launch of the sampler the step runs, over B rows of the vocabulary with this arm's params."""
    V = dec.dims.vocab_size
    g = torch.Generator(device="cuda").manual_seed(B)
    lg = torch.empty((B, (V + 7) // 8 * 8), dtype=dec.dtype, device="cuda")[:, :V]
    lg.copy_(torch.randn((B, V), generator=g, device="cuda") * 3)
    seeds = torch.tensor(sequence_seeds(SEED, B), dtype=torch.int64, device="cuda")
    step = torch.ones(1, dtype=torch.int32, device="cuda")
    ids = torch.zeros(max(B, 2), dtype=torch.int64, device="cuda")
    dec._set_sampling(dict(BASE, **arm))
    params = dec._draw_params
    row = lg[0].float().contiguous()
    launch = (lambda: ops.sample_top_p(row, params, seeds[:1], step, -1, ids)) if B == 1 else (
        lambda: ops.sample_rows(lg, params, seeds, step, 0, ids[:B]))
    with ops.elem_dtype(dec.dtype):
        for _ in range(10):
            launch()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            launch()
        b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("warpers_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    batches = [int(b) for b in args.batches.split(",")]
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g)) for _ in range(max(batches))]
    prefill = EventTimer(dec.prefill_packed)
    prefill_one = EventTimer(dec.prefill_hidden)
    dec.prefill_packed, dec.prefill_hidden = prefill, prefill_one
    out = {"card": card(), "vocab": cfg.llama.vocab_size, "prompt_rows": S, "new_tokens": N, "sampling": {**BASE, "top_k": 50},
           "arms": ARMS, "reps": args.reps, "by_batch": {}}
    for B in batches:
        x = torch.cat(prompts[:B])

        def run(arm):
            smp = dict(BASE, **arm)
            return dec.generate_from_embeds(prompts[0], N, sampling=smp) if B == 1 else dec.generate_batch(x, [S] * B, N, sampling=smp)

        step_ms = {a: [] for a in ARMS}
        for rep in range(1 + args.reps):
            for name, arm in ARMS.items():
                prefill.take_ms(); prefill_one.take_ms()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                run(arm)
                e1.record()
                torch.cuda.synchronize()
                pre = sum(prefill.take_ms()) + sum(prefill_one.take_ms())
                if rep:
                    step_ms[name].append((e0.elapsed_time(e1) - pre) / (N - 1))
        row = {}
        for name, arm in ARMS.items():
            us = [sampler_us(dec, B, arm) for _ in range(3)]
            row[name] = {"sampler_us_per_step": round(statistics.median(us), 1), "sampler_us_spread": [round(min(us), 1), round(max(us), 1)],
                         "decode_ms_per_step": round(statistics.median(step_ms[name]), 3)}
        out["by_batch"][B] = row
        print(f"B={B}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
