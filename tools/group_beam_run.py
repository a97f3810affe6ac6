"""Measure diverse beam search (LlamaDecoder.generate_beam_batch with num_beam_groups) against plain beam search over the same rows, at
Llama-3-8B shapes: the full-depth decoder with seeded random weights, 259-row prompts, 64 new tokens (no EOS, so every run takes all 64
steps), k in {4, 8} beams, G in {2, k} groups (diversity_penalty 0.5), B in {1, 8} prompts.  The arms alternate within each repetition.

Per (k, B) and arm (medians over the repetitions after a warm-up round):
  * ms per beam step (the run minus its prefill, over the 64 steps);
  * device us per step in the candidates kernel (beam_candidates / beam_candidates_scored) and in the per-prompt choice (beam_select /
    beam_group_select), from CUDA events around each launch.
The card name, power limit and SM clocks are read in the same run.

    python tools/group_beam_run.py [--reps 3]   (one JSON line on stdout)
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

S, N, LAMBDA = 259, 64, 0.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_beam_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(d, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (S,), generator=g)) for _ in range(8)]
    prefill = dec.prefill_packed = EventTimer(dec.prefill_packed)
    timers = {"cand": EventTimer(ops.beam_candidates), "cand_scored": EventTimer(ops.beam_candidates_scored),
              "select": EventTimer(ops.beam_select), "group_select": EventTimer(ops.beam_group_select)}
    ops.beam_candidates, ops.beam_candidates_scored = timers["cand"], timers["cand_scored"]
    ops.beam_select, ops.beam_group_select = timers["select"], timers["group_select"]
    out = {"card": card(), "prompt_rows": S, "new_tokens": N, "diversity_penalty": LAMBDA, "reps": args.reps, "runs": {}}
    for k in (4, 8):
        for B in (1, 8):
            x = torch.cat(prompts[:B])
            arms = {"plain": 1, "groups_2": 2, f"groups_{k}": k}
            res = {a: {"total_ms": [], "prefill_ms": [], "cand_us": [], "select_us": []} for a in arms}
            for rep in range(1 + args.reps):  # round 0 warms the graphs up
                for arm, G in arms.items():
                    for t in list(timers.values()) + [prefill]:
                        t.take_ms()
                    kw = {} if G == 1 else dict(num_beam_groups=G, diversity_penalty=LAMBDA)
                    t, r = timed(lambda: dec.generate_beam_batch(x, [S] * B, k, N, **kw))
                    assert all(v.numel() == N for v in r)
                    if rep == 0:
                        continue
                    res[arm]["total_ms"].append(t * 1e3)
                    res[arm]["prefill_ms"].append(sum(prefill.take_ms()))
                    res[arm]["cand_us"].append(sum(timers["cand" if G == 1 else "cand_scored"].take_ms()) * 1e3)
                    res[arm]["select_us"].append(sum(timers["select" if G == 1 else "group_select"].take_ms()) * 1e3)
            row = {}
            for arm, v in res.items():
                total, pre = statistics.median(v["total_ms"]), statistics.median(v["prefill_ms"])
                row[arm] = {"ms_per_step": round((total - pre) / N, 3), "candidates_us_per_step": round(statistics.median(v["cand_us"]) / N, 1),
                            "select_us_per_step": round(statistics.median(v["select_us"]) / N, 1)}
            for arm in arms:
                if arm != "plain":
                    row[arm]["vs_plain"] = round(row[arm]["ms_per_step"] / row["plain"]["ms_per_step"], 3)
            out["runs"][f"k{k}_B{B}"] = row
            print(f"k={k} B={B}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
