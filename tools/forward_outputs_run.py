"""Measure forward(output_hidden_states=, output_attentions=) at Llama-3-8B shapes: the full-depth decoder (32 layers, 32 query / 8 kv
heads of 128) with seeded random weights, prompts of 259 rows (the c2 request's length) and text prompts of 1024, 2048 and 4096 rows, at
B = 1 and B = 8.

  * forward() wall time (host clock around a synchronised call, median over the repetitions after a warm-up) with no flags, with each
    flag alone and with both.  A configuration whose outputs do not fit in device memory reports the bytes forward() asked for (its
    RuntimeError is raised before any GPU work).
  * The probability kernel alone (srgpt_attention_probs_bf16 over random rotated Q / K of one layer, CUDA events over --iters launches):
    us per layer; the bytes it writes (B * 32 * S * S * 2) per second against the H100 SXM's 3.35 TB/s; and its Q K^T TFLOP/s, counted
    as 2 passes x 2 * 128 FLOP over the S (S + 1) / 2 causal (query, key) pairs of each head.
The card name, power limit and SM clocks are read in the same run.

    python tools/forward_outputs_run.py [--reps 3] [--iters 20]   (one JSON line on stdout)
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


def kernel_row(d, B, S, iters):
    nh, nkv, hd = d.num_attention_heads, d.num_key_value_heads, d.head_dim
    g = torch.Generator(device="cuda").manual_seed(S + B)
    q = torch.randn(B * S, nh * hd, generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn(B * S, nkv * hd, generator=g, device="cuda").to(torch.bfloat16)
    cu = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device="cuda")
    out = torch.empty((B, nh, S, S), dtype=torch.bfloat16, device="cuda")
    run = lambda: ops.attention_probs(q, k, nh, nkv, hd, hd ** -0.5, out, cu_seqlens=cu, max_seqlen=S)  # noqa: E731
    run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    s = a.elapsed_time(b) / iters * 1e-3
    written = B * nh * S * S * 2
    flop = 2 * 2 * hd * (S * (S + 1) // 2) * nh * B
    del out
    return {"us_per_layer": round(s * 1e6, 1), "write_TBps": round(written / s / 1e12, 3), "write_share_of_hbm": round(written / s / 1e12 / HBM_TBS, 3),
            "qk_TFLOPs": round(flop / s / 1e12, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--lens", default="259,1024,2048,4096")
    ap.add_argument("--batches", default="1,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("forward_outputs_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    model = LlavaLlamaModel(cfg, random_init(cfg, "cuda", seed=0), max_seq_len=4096)
    d = cfg.llama
    out = {"card": card(), "layers": d.num_hidden_layers, "reps": args.reps, "runs": {}}
    g = torch.Generator().manual_seed(7)
    for S in [int(s) for s in args.lens.split(",")]:
        for B in [int(b) for b in args.batches.split(",")]:
            ids = torch.randint(1000, 30000, (B, S), generator=g).cuda()
            emb = model.llm.embed_tokens(ids).view(B, S, -1)
            row = {}
            for arm, kw in ARMS.items():
                try:
                    ts = []
                    for rep in range(1 + args.reps):
                        t, r = timed(lambda: model.forward(inputs_embeds=emb, **kw))
                        del r
                        if rep:
                            ts.append(t * 1e3)
                    row[arm + "_ms"] = round(statistics.median(ts), 2)
                except RuntimeError as e:
                    row[arm + "_ms"] = f"not run: {e}"
                torch.cuda.empty_cache()
            try:
                row["probs_kernel"] = kernel_row(d, B, S, args.iters)
            except torch.OutOfMemoryError:
                row["probs_kernel"] = "not run: one layer's output does not fit"
            torch.cuda.empty_cache()
            out["runs"][f"S{S}_B{B}"] = row
            print(f"S={S} B={B}: {row}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
