"""Measure contrastive search (LlamaDecoder.generate_contrastive) at Llama-3-8B shapes: the full-depth decoder with seeded random weights,
259-row prompts, 128 new tokens (no EOS, so every run takes all its steps), penalty_alpha = 0.6, k in {4, 8} and B in {1, 8}.  For
comparison, at the same B: greedy decoding (generate_from_embeds at B = 1, generate_batch above) and beam search with num_beams = k
(generate_beam_batch, whose step has the same B * k rows).

Per (k, B) and arm (medians over the repetitions after a warm-up round):
  * ms per emitted token: the run's wall time over its 128 tokens, and the step alone ((run of 128 tokens - run of 1 token) / 127);
  * CUDA-event us per step of the penalty, select and KV broadcast kernels, from an eager run (use_graph=False) of the same request.
The card name, power limit and SM clocks are read in the same run.

    python tools/contrastive_run.py [--reps 3]   (one JSON line on stdout)
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

S, N, ALPHA = 259, 128, 0.6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ks", default="4,8")
    ap.add_argument("--batches", default="1,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contrastive_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    batches, ks = [int(b) for b in args.batches.split(",")], [int(k) for k in args.ks.split(",")]
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g)) for _ in range(max(batches))]
    out = {"card": card(), "prompt_rows": S, "new_tokens": N, "penalty_alpha": ALPHA, "reps": args.reps, "runs": {}}
    for k in ks:
        for B in batches:
            x, lens = torch.cat(prompts[:B]), [S] * B
            arms = {
                "contrastive": lambda n: dec.generate_contrastive(x, lens, k, ALPHA, n),
                "greedy": (lambda n: [dec.generate_from_embeds(x, n)]) if B == 1 else (lambda n: dec.generate_batch(x, lens, n)),
                "beams": lambda n: dec.generate_beam_batch(x, lens, k, n),
            }
            res = {a: {"run_ms": [], "one_ms": []} for a in arms}
            for rep in range(1 + args.reps):  # round 0 captures the graphs
                for arm, fn in arms.items():
                    t, _ = timed(lambda: fn(N))
                    t1, _ = timed(lambda: fn(1))
                    if rep:
                        res[arm]["run_ms"].append(t * 1e3)
                        res[arm]["one_ms"].append(t1 * 1e3)
            row = {}
            for arm, v in res.items():
                run, one = statistics.median(v["run_ms"]), statistics.median(v["one_ms"])
                row[arm] = {"ms_per_token": round(run / N, 3), "step_ms": round((run - one) / (N - 1), 3)}
            # kernel times of the contrastive step, from an eager run with CUDA events around each launch
            timers = {name: EventTimer(getattr(ops, name)) for name in ("contrastive_penalty", "contrastive_select", "kv_broadcast_rows")}
            saved = {name: getattr(ops, name) for name in timers}
            try:
                for name, t in timers.items():
                    setattr(ops, name, t)
                for rep in range(2):
                    for t in timers.values():
                        t.take_ms()
                    dec.generate_contrastive(x, lens, k, ALPHA, N, use_graph=False)
                row["kernel_us_per_step"] = {name.replace("contrastive_", "").replace("_rows", ""): round(statistics.median(t.take_ms()) * 1e3, 1)
                                             for name, t in timers.items()}
            finally:
                for name, fn in saved.items():
                    setattr(ops, name, fn)
            out["runs"][f"k{k}_B{B}"] = row
            print(f"k={k} B={B}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
