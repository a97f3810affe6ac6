#!/usr/bin/env python
"""Per-launch device time of the sampler at Llama-3's vocabulary (V = 128256), top_k 50: sample_top_p over one fp32 row and
sample_rows over R = 1 and R = 32 element-type rows (the batched lm_head's), at the sampled workload of DESIGN.md §5 (T 0.7, top_p 0.9)
and at the reference's default (T 0.2, top_p 1).  CUDA events around back-to-back launches after a warm-up; the median of --reps
windows.  The card's name, power limit and maximum SM clock are read in the same run.  One JSON line.

    python tools/sampler_time.py [--lib OTHER/libsrgpt_b200.so] [--launches 200] [--reps 5]

--lib times another build of the library (e.g. the parent commit's, for a before / after comparison); it is loaded as is, never rebuilt.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

V = 128256
SETTINGS = {"T0.7_p0.9_k50": (0.7, 0.9, 50.0), "T0.2_p1_k50": (0.2, 1.0, 50.0)}


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return {"name": torch.cuda.get_device_name(0), "power.limit, clocks.max.sm": q}


def time_us(fn, launches, reps):
    import torch
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / launches)
    return round(statistics.median(out), 1), round(max(out) - min(out), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    from spatialrgpt_b200 import _build, _lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("sampler_time: needs a CUDA device")
    if args.lib:
        _build.VARIANTS["bf16"] = (os.path.abspath(args.lib), [])
        _lib.load(build_if_missing=False)
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rows = torch.randn(32, V, generator=g, device=dev) * 2.5
    row, rows16 = rows[0].contiguous(), rows.to(ops.ELEM())
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    seeds = torch.arange(32, dtype=torch.int64, device=dev)
    out = torch.empty(32, dtype=torch.int64, device=dev)
    res = {"card": card(), "lib": args.lib or _lib.lib_path(), "V": V, "launches": args.launches, "reps": args.reps, "us_per_launch": {}}
    for name, (T, p, k) in SETTINGS.items():
        params = torch.tensor([T, p, k], dtype=torch.float32, device=dev)
        r = {"sample_top_p": time_us(lambda: ops.sample_top_p(row, params, seeds[:1], step, 0, out), args.launches, args.reps)}
        for R in (1, 32):
            r[f"sample_rows_R{R}"] = time_us(lambda R=R: ops.sample_rows(rows16[:R], params, seeds[:R], step, 0, out[:R]), args.launches,
                                             args.reps)
        res["us_per_launch"][name] = {kname: {"median": v[0], "spread": v[1]} for kname, v in r.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
