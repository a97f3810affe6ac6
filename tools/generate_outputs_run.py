"""Measure generate(output_hidden_states=, output_attentions=, return_dict_in_generate=True) at Llama-3-8B shapes: the full-depth
decoder (32 layers, 32 query / 8 kv heads of 128) with seeded random weights, a 259-row text prompt (the c2 request's length) and 128
greedy tokens, at B = 1 and B = 8.

  * ms per decode step with no flags, hidden states, attentions and both: (generate of 128 tokens - generate of 1 token) / 127, host
    clock around synchronised calls, median over the repetitions after a warm-up.  The ids of every arm must equal the no-flag ids.
  * The decode probability kernel alone (srgpt_attention_probs_decode_bf16, both launches, over one layer's paged cache at 387 and 4096
    keys, CUDA events around one CUDA-graph replay of --iters launches): us per layer, and the bytes it moves over that time (K read by both launches, the
    probabilities written).
The card name, power limit and SM clocks are read in the same run.

    python tools/generate_outputs_run.py [--reps 3] [--iters 50]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llava_llama import LlavaLlamaModel  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.nf4_run import card, timed  # noqa: E402

HBM_TBS = 3.35
ARMS = {"none": {}, "hidden": dict(output_hidden_states=True), "attn": dict(output_attentions=True),
        "both": dict(output_hidden_states=True, output_attentions=True)}


def kernel_row(d, R, P, iters):
    nh, nkv, hd, ps = d.num_attention_heads, d.num_key_value_heads, d.head_dim, 16
    g = torch.Generator(device="cuda").manual_seed(P + R)
    cap = (P + ps - 1) // ps
    kv = torch.randn(R * cap, 2, ps, nkv, hd, generator=g, device="cuda").to(torch.bfloat16)
    pt = torch.arange(R * cap, dtype=torch.int32, device="cuda").view(R, cap)
    q = torch.randn(R, nh * hd, generator=g, device="cuda").to(torch.bfloat16)
    n = P - 128  # 128 generated keys after the prompt
    pos = torch.full((R,), P - 1, dtype=torch.int32, device="cuda")
    off = torch.zeros(R, dtype=torch.int32, device="cuda")
    n_prompt = torch.full((R,), n, dtype=torch.int32, device="cuda")
    step = torch.ones(1, dtype=torch.int32, device="cuda")
    out = torch.empty((1, R, nh, P), dtype=torch.bfloat16, device="cuda")
    ws = ops.attention_probs_decode_ws(R, nh, P, "cuda")
    run = lambda: ops.attention_probs_decode(q, kv, pt, ps, pos, nh, nkv, hd, hd ** -0.5, off, n_prompt, n, step, -1, out, ws)  # noqa: E731
    run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()  # the launches replayed as in a decode step's graph, without the Python launch path
    with torch.cuda.graph(graph):
        for _ in range(iters):
            run()
    graph.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    graph.replay()
    b.record()
    torch.cuda.synchronize()
    s = a.elapsed_time(b) / iters * 1e-3
    moved = 2 * R * P * nkv * hd * 2 + R * nh * P * 2
    return {"us_per_layer": round(s * 1e6, 1), "bytes": moved, "TBps": round(moved / s / 1e12, 3), "share_of_hbm": round(moved / s / 1e12 / HBM_TBS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--prompt", type=int, default=259)
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--kernel-only", action="store_true", help="time the probability kernel only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generate_outputs_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    model = LlavaLlamaModel(cfg, random_init(cfg, "cuda", seed=0), max_seq_len=4096)
    d = cfg.llama
    out = {"card": card(), "layers": d.num_hidden_layers, "prompt": args.prompt, "tokens": args.tokens, "reps": args.reps, "runs": {}}
    g = torch.Generator().manual_seed(7)
    N = args.tokens
    for B in [int(b) for b in args.batches.split(",") if not args.kernel_only]:
        ids = torch.randint(1000, 30000, (B, args.prompt), generator=g).cuda()
        row, ref = {}, None
        for arm, kw in ARMS.items():
            ts = []
            for rep in range(1 + args.reps):
                t1, _ = timed(lambda: model.generate(ids, max_new_tokens=1, eos_token_id=None, return_dict_in_generate=True, **kw))
                tN, r = timed(lambda: model.generate(ids, max_new_tokens=N, eos_token_id=None, return_dict_in_generate=True, **kw))
                if ref is None:
                    ref = r.sequences.clone()
                row.setdefault("ids_equal", True)
                row["ids_equal"] = row["ids_equal"] and torch.equal(r.sequences, ref)
                del r
                if rep:
                    ts.append((tN - t1) * 1e3 / (N - 1))
            row[arm + "_ms_per_step"] = round(statistics.median(ts), 3)
            torch.cuda.empty_cache()
        out["runs"][f"B{B}"] = row
        print(f"B={B}: {row}", file=sys.stderr, flush=True)
    for P in (args.prompt + N, 4096):
        for R in [int(b) for b in args.batches.split(",")]:
            out["runs"][f"kernel_P{P}_R{R}"] = kernel_row(d, R, P, args.iters)
            print(f"kernel P={P} R={R}: {out['runs'][f'kernel_P{P}_R{R}']}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
