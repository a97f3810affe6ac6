"""Measure beam search over a batch of prompts (LlamaDecoder.generate_beam_batch) against the same prompts one after the other
(generate_beam), at Llama-3-8B shapes: the full-depth decoder with seeded random weights, k = 3 beams, 259-row prompts, 64 new tokens
(no EOS, so every run takes all 64 steps), B in {1, 4, 8, 16, 32, 42}.  The two arms alternate within each repetition.

Per B and arm (medians over the repetitions after a warm-up round):
  * ms per beam step (the run minus its prefills, over the steps: 64 for the batch, B x 64 for the sequential arm);
  * new tokens per second summed over the prompts;
  * prefill ms (the batch prefills each prompt once, generate_beam k times) - CUDA events around prefill_packed;
  * device us per step in the merge (beam_select) and the KV copies (kv_copy_pages, including the upload of its pair list) of the batch,
    and the one-off copy of each prompt's pages into its other beams;
  * whether both arms produced the same ids for every prompt.
The card name, power limit and SM clocks are read in the same run.

    python tools/beam_batch_run.py [--reps 3] [--batches 1,4,8,16,32,42]   (one JSON line on stdout)
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
from tools.nf4_run import card, timed  # noqa: E402

K, S, N = 3, 259, 64


class EventTimer:
    """Wraps a function so every call is bracketed by CUDA events on the current stream; take_ms() returns each call's device ms."""

    def __init__(self, fn):
        self.fn, self.marks = fn, []

    def __call__(self, *a, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = self.fn(*a, **kw)
        e.record()
        self.marks.append((s, e))
        return r

    def take_ms(self) -> list:
        torch.cuda.synchronize()
        t = [s.elapsed_time(e) for s, e in self.marks]
        self.marks = []
        return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,4,8,16,32,42")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_batch_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(d, w, max_seq_len=1024)
    batches = [int(b) for b in args.batches.split(",")]
    g = torch.Generator().manual_seed(7)
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g)) for _ in range(max(batches))]
    prefill = dec.prefill_packed = EventTimer(dec.prefill_packed)
    select = ops.beam_select = EventTimer(ops.beam_select)
    copy = ops.kv_copy_pages = EventTimer(ops.kv_copy_pages)
    out = {"card": card(), "num_beams": K, "prompt_rows": S, "new_tokens": N, "reps": args.reps, "by_batch": {}}
    for B in batches:
        x = torch.cat(prompts[:B])
        res = {a: {"total_ms": [], "prefill_ms": [], "select_us": [], "replicate_us": [], "copy_us": []} for a in ("batch", "sequential")}
        ids = {}
        for rep in range(1 + args.reps):  # round 0 warms the graphs up
            for arm in ("batch", "sequential"):
                for timer in (prefill, select, copy):
                    timer.take_ms()
                if arm == "batch":
                    t, r = timed(lambda: dec.generate_beam_batch(x, [S] * B, K, N))
                else:
                    t, r = timed(lambda: [dec.generate_beam(p, K, N) for p in prompts[:B]])
                ids[arm] = [v.tolist() for v in r]
                if rep == 0:
                    continue
                res[arm]["total_ms"].append(t * 1e3)
                res[arm]["prefill_ms"].append(sum(prefill.take_ms()))
                res[arm]["select_us"].append(sum(select.take_ms()) * 1e3)
                c = copy.take_ms() + [0.0]  # the batch's first copy replicates the prompts into the other beams, the rest are per step
                res[arm]["replicate_us"].append(c[0] * 1e3)
                res[arm]["copy_us"].append(sum(c[1:]) * 1e3)
        row = {}
        for arm, v in res.items():
            steps = N if arm == "batch" else B * N
            total, pre = statistics.median(v["total_ms"]), statistics.median(v["prefill_ms"])
            row[arm] = {"total_ms": round(total, 1), "prefill_ms": round(pre, 2), "ms_per_step": round((total - pre) / steps, 3),
                        "new_tokens_per_s": round(B * N / (total / 1e3), 1)}
            if arm == "batch":
                row[arm]["merge_us_per_step"] = round(statistics.median(v["select_us"]) / N, 1)
                row[arm]["kv_copy_us_per_step"] = round(statistics.median(v["copy_us"]) / N, 1)
                row[arm]["prompt_replication_us"] = round(statistics.median(v["replicate_us"]), 1)
        row["speedup"] = round(row["sequential"]["total_ms"] / row["batch"]["total_ms"], 2)
        row["ids_equal"] = ids["batch"] == ids["sequential"]
        out["by_batch"][B] = row
        print(f"B={B}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
