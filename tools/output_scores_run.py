"""Measure what output_scores costs the decode step (generate(return_dict_in_generate=True, output_scores=True)) at Llama-3-8B shapes:
the full-depth decoder of config c2 with seeded random weights, 259-row prompts, every request run with and without the flag,
alternating, after a warm-up of each:
  * batch 1, greedy and sampled (generate_from_embeds);
  * B = 32, greedy and sampled (generate_batch, the batched step);
  * beams, 42 prompts x 3 beams (generate_beam_batch).
Per mode: ms per generated step without and with scores (host clock around the call, ending in a device synchronise, minus the same
call at max_new_tokens = 1, over the remaining steps; medians over the repetitions), the difference, and the ids equal with and without.
The card name, power limit and SM clocks are read in the same run.

    python tools/output_scores_run.py [--reps 3] [--steps 64]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.nf4_run import card, timed  # noqa: E402

S = 259
SAMPLING = dict(temperature=0.7, top_p=0.9, top_k=50, seed=3)


def ids_of(r):
    r = r[0] if isinstance(r, tuple) else r
    return [t.tolist() for t in r] if isinstance(r, list) else r.tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("output_scores_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(d, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)

    def prompts(n):
        return dec.embed_tokens(torch.randint(1000, 30000, (n * S,), generator=g))

    one, b32, b42 = prompts(1), prompts(32), prompts(42)
    modes = {
        "batch1_greedy": lambda n, sc: dec.generate_from_embeds(one, n, output_scores=sc),
        "batch1_sampled": lambda n, sc: dec.generate_from_embeds(one, n, sampling=SAMPLING, output_scores=sc),
        "b32_greedy": lambda n, sc: dec.generate_batch(b32, [S] * 32, n, output_scores=sc),
        "b32_sampled": lambda n, sc: dec.generate_batch(b32, [S] * 32, n, sampling=SAMPLING, output_scores=sc),
        "beams_42x3": lambda n, sc: dec.generate_beam_batch(b42, [S] * 42, 3, n, output_scores=sc),
    }
    res = {"card": card(), "steps": args.steps, "prompt_rows": S}
    for name, run in modes.items():
        per = {False: [], True: []}
        same = True
        for sc in (False, True):  # warm-up: graphs captured, buffers allocated
            run(args.steps, sc)
        for _ in range(args.reps):
            ids = {}
            for sc in (False, True):
                t1, _ = timed(lambda: run(1, sc))
                tn, r = timed(lambda: run(args.steps, sc))
                per[sc].append((tn - t1) * 1e3 / (args.steps - 1))
                ids[sc] = ids_of(r)
                del r
            same &= ids[False] == ids[True]
        off, on = statistics.median(per[False]), statistics.median(per[True])
        res[name] = {"ms_per_step": round(off, 3), "ms_per_step_scores": round(on, 3), "overhead_ms": round(on - off, 3),
                     "overhead_pct": round(100 * (on - off) / off, 2), "ids_equal": same}
        print(name, res[name], file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
