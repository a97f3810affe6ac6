"""Measure generate(prefix_cache=True) on a multi-turn line: c2 shapes (SigLIP-so400m@448px + Llama-3-8B, seeded random weights,
one image, 8 regions, depth on), three questions asked one after the other with the conversation growing, as the SpatialRGPT-Bench
driver asks them.  The cache-off and cache-on lines alternate in one process after a warm-up.

Per turn: TTFT (generate with max_new_tokens=1) and request time (max_new_tokens=--new-tokens), both host clocks around work that
ends in a device synchronise (median over --reps), model.last_prefix_reuse, and the on-vs-off logit deviation relative to the
logits' standard deviation (up to the first diverging greedy step; where the ids diverge, the top-1 / top-2 margin of the cache-off
logits at that step).  Also the paged attention kernel alone (CUDA events over many launches): a 30-row chunk over 259 and over
1024 cached positions at Llama-3-8B heads.  The card name and power limit are read in the same run.

    python tools/prefix_cache_run.py [--reps 5] [--new-tokens 32] [--out DIR]   (one JSON line on stdout)
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

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llava_llama import LlavaLlamaModel  # noqa: E402
from spatialrgpt_b200.synth import synth_request  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402

QUESTION_ROWS = 24  # tokens per follow-up question, two of them region references


def turns(cfg, seed=1234):
    """Three prompts, each the previous one with a question appended (the assistant slots stay empty, as in the driver)."""
    ids, im, de, mk = synth_request(cfg, 8, 64, seed)
    g = torch.Generator().manual_seed(seed + 1)
    prompts = [ids]
    for k in range(2):
        q = torch.randint(1000, 30000, (1, QUESTION_ROWS), generator=g)
        q[0, 3], q[0, 4] = cfg.llm_mask_token_id, cfg.llm_depth_token_id
        q[0, 9], q[0, 10] = cfg.llm_mask_token_id, cfg.llm_depth_token_id
        prompts.append(torch.cat([prompts[-1], q], 1))
    # every <mask> token consumes one mask row: the driver passes the masks of all the line's references in every turn
    return prompts, im, de, torch.cat([mk[0], mk[0][:4]])


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, with the reason the limit is missing
        q = f"unavailable ({e})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def run_line(model, prompts, args, cache: bool, **kw):
    """One annotation: the three turns in order.  Returns per turn (seconds, output, last_prefix_reuse)."""
    if cache:
        model._prefix_state = None  # a new annotation: nothing from the previous line is reused
    out = []
    for ids in prompts:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = model.generate(ids, prefix_cache=cache, **args, **kw) if cache else model.generate(ids, **args, **kw)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0, r, model.last_prefix_reuse if cache else None))
    return out


def paged_kernel(rows, start, iters=500):
    nh, nkv, hd, page = 32, 8, 128, 16
    dev = "cuda"
    n_pg = (start + rows + page - 1) // page
    pages = torch.randn(n_pg + 1, 2, page, nkv, hd, device=dev).to(torch.bfloat16)
    pt = torch.randperm(n_pg + 1, device=dev)[None].to(torch.int32)
    qkv = torch.randn(rows, (nh + 2 * nkv) * hd, device=dev).to(torch.bfloat16)
    sp = torch.tensor([start], dtype=torch.int32, device=dev)
    cu = torch.tensor([0, rows], dtype=torch.int32, device=dev)
    out = torch.empty(rows, nh * hd, dtype=torch.bfloat16, device=dev)
    call = lambda: ops.attention_prefill_paged(qkv[:, :nh * hd], pages, pt, page, sp, cu, rows, nh, nkv, hd, hd ** -0.5, out=out)  # noqa: E731
    for _ in range(20):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    visible = sum(start + r + 1 for r in range(rows))  # causal: row r sees start + r + 1 positions
    flops = 4 * nh * hd * visible  # QK^T and PV
    kv_bytes = 2 * (start + rows) * nkv * hd * 2  # K and V of every visible position, read once per kv head
    return {"rows": rows, "cached_positions": start, "us": round(ms * 1e3, 2), "tflops": round(flops / ms / 1e9, 3),
            "kv_gbps": round(kv_bytes / ms / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--new-tokens", type=int, default=32)
    ap.add_argument("--out", default=None, help="also write the result to DIR/prefix_cache_run.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    cfg = baseline_config("c2")
    dev = torch.device("cuda", 0)
    model = LlavaLlamaModel(cfg, random_init(cfg, dev, seed=0, n_tower_layers=cfg.vision.num_hidden_layers - 1), max_seq_len=1024)
    prompts, im, de, mk = turns(cfg)
    prompts = [p.to(dev) for p in prompts]
    base = dict(images=im.to(dev), depths=de.to(dev), masks=[mk.to(dev)], do_sample=False)
    ttft_args, req_args = dict(base, max_new_tokens=1), dict(base, max_new_tokens=a.new_tokens)
    for cache in (False, True, False, True):  # warm-up of every shape
        run_line(model, prompts, ttft_args, cache)
        run_line(model, prompts, req_args, cache)
    times = {k: [[] for _ in prompts] for k in ("ttft_off", "ttft_on", "req_off", "req_on")}
    reuse = None
    for _ in range(a.reps):
        for cache in (False, True):
            tag = "on" if cache else "off"
            for i, (t, _, info) in enumerate(run_line(model, prompts, ttft_args, cache)):
                times["ttft_" + tag][i].append(t * 1e3)
            line = run_line(model, prompts, req_args, cache)
            for i, (t, _, info) in enumerate(line):
                times["req_" + tag][i].append(t * 1e3)
            if cache:
                reuse = [info for _, _, info in line]
    # on-vs-off deviation of the per-step logits (eager decode with logits)
    lg_args = dict(base, max_new_tokens=16, output_logits=True)
    off = run_line(model, prompts, lg_args, False)
    on = run_line(model, prompts, lg_args, True)
    dev_rows = []
    for k, ((_, (ids_off, lg_off), _), (_, (ids_on, lg_on), _)) in enumerate(zip(off, on)):
        a_ids, b_ids = ids_off[0].tolist(), ids_on[0].tolist()
        n = min(len(a_ids), len(b_ids))
        div = next((i for i in range(n) if a_ids[i] != b_ids[i]), None)
        upto = n if div is None else div + 1
        lo, ln = lg_off[0][:upto].float(), lg_on[0][:upto].float()
        sigma = float(lo.std())
        row = {"turn": k + 1, "max_dev_over_sigma": round(float((ln - lo).abs().max()) / sigma, 5), "steps_compared": upto,
               "first_diverging_step": div}
        if div is not None:
            t2 = lo[div].topk(2).values
            row["top1_top2_margin_over_sigma_at_divergence"] = round(float(t2[0] - t2[1]) / sigma, 5)
        dev_rows.append(row)
    med = {k: [round(statistics.median(v), 2) for v in vs] for k, vs in times.items()}
    res = {"card": card(), "workload": "c2 shapes, seeded random weights, 1 image 448px + depth, 8 regions, 3 questions "
                                       f"(64-token first prompt, +{QUESTION_ROWS} tokens per follow-up)",
           "reps": a.reps, "new_tokens": a.new_tokens, "median_ms": med, "last_prefix_reuse": reuse, "logit_deviation": dev_rows,
           "paged_kernel": [paged_kernel(30, 259), paged_kernel(30, 1024)]}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "prefix_cache_run.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
