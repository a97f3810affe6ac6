"""Measure batch-invariant decoding at c2 shapes: the full-depth Llama-3-8B decoder with seeded random weights (packed decode weights
unless SRGPT_DECODE_PACK=0), B prompts of 259 rows each, 128 greedy tokens per prompt, for B = 1, 2, 4, 8:

  * rows: LlamaDecoder.generate_rows over the B prompts (the rows step, graph-replayed);
  * sequential: the same B prompts one after another through batch-1 generate_from_embeds;
  * batched: generate_batch over the same B prompts (the stream-K GEMM step, which is not batch-invariant);
Each is timed as the decode phase, (t(128 tokens) - t(1 token)) with a host clock around work that ends in a device synchronise, so
prefill and the first token drop out; step_ms = decode time / 127 and tokens_per_s = B * 127 / decode time.  ids_identical compares
every row of the rows run with its sequential run.  The three modes alternate over --reps rounds after a warm-up round; medians.  The
card name, power limit and max SM clock are read in the same run.

    python tools/batch_invariant_run.py [--reps 3] [--new-tokens 128]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402

PROMPT_ROWS = 259  # c2: 256 image rows + the question
ROWS = (1, 2, 4, 8)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:
        q = f"unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batch_invariant_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (PROMPT_ROWS,), generator=g)) for _ in range(max(ROWS))]
    N = args.new_tokens
    modes = {
        "rows": lambda B, n: dec.generate_rows(prompts[:B], n),
        "sequential": lambda B, n: [dec.generate_from_embeds(p, n) for p in prompts[:B]],
        "batched": lambda B, n: dec.generate_batch(torch.cat(prompts[:B]), [PROMPT_ROWS] * B, n),
    }
    times = {(m, B): [] for m in modes for B in ROWS}
    ids = {}
    for _ in range(1 + args.reps):  # round 0 warms every graph and shape up
        for B in ROWS:
            for m, fn in modes.items():
                t1, _ = timed(lambda: fn(B, 1))
                tn, r = timed(lambda: fn(B, N))
                times[(m, B)].append(tn - t1)
                ids[(m, B)] = [o.tolist() for o in r]
    out = {"card": card(), "decode_pack": "packed" if any(v == "packed" for v in dec.decode_pack.values()) else "bf16",
           "prompt_rows": PROMPT_ROWS, "new_tokens": N, "reps": args.reps}
    for B in ROWS:
        row = {}
        for m in modes:
            t = statistics.median(times[(m, B)][1:])
            row[m] = {"step_ms": round(t * 1e3 / (N - 1), 3), "tokens_per_s": round(B * (N - 1) / t, 1)}
        row["rows_ids_identical_to_sequential"] = ids[("rows", B)] == ids[("sequential", B)]
        row["batched_ids_identical_to_sequential"] = ids[("batched", B)] == ids[("sequential", B)]
        out[f"B{B}"] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
