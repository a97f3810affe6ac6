"""Measure prompt-lookup speculative decoding at c2 shapes: the full-depth Llama-3-8B decoder with seeded random weights (packed decode
weights unless SRGPT_DECODE_PACK=0), a 259-row prompt, batch 1, greedy.

  * the plain one-token graph step and the verify pass for T = 2 .. 8 (graph replays, CUDA events, warmed up, median);
  * decode-phase tokens/s of one 128-token request ((t(128 tokens) - t(1 token)) / 127, host clock around work that ends in a device
    synchronise): plain greedy, prompt lookup with perfect drafts (the plain continuation planted as the lookup history: the upper
    bound), with drafts that are never accepted (a lookup history the model's choices never follow), and with real prompt lookup on the
    synthetic prompt (random weights: the acceptance says nothing about a trained checkpoint);
  * every speculative line carries ids_identical (its ids against the plain request's) and last_speculation.
Plain and speculative requests alternate over --reps rounds; medians.  The card name, power limit and max SM clock are read in
the same run.

    python tools/spec_decode_run.py [--reps 3] [--k 4] [--new-tokens 128]   (one JSON line on stdout)
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
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402

PROMPT_ROWS = 259  # c2: 256 image rows + the question


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


def replay_ms(dec, graph, S, n=30):
    """Median time of one graph replay starting at position S (pos / step reset before each, outside the timed window)."""
    ts = []
    for i in range(n + 5):
        dec.pos.fill_(S)
        dec.step.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        b.synchronize()
        if i >= 5:
            ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_decode_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    prompt_ids = torch.randint(1000, 30000, (PROMPT_ROWS,), generator=g)
    x = dec.embed_tokens(prompt_ids)
    N, k = args.new_tokens, args.k
    plain_ids = dec.generate_from_embeds(x, N + 2 * ops.SPEC_T_MAX)
    ref = plain_ids[:N]
    cases = {
        "perfect": torch.cat([prompt_ids, plain_ids.cpu()]),
        "never_accepted": torch.cat([prompt_ids, (plain_ids.cpu() + 1) % cfg.llama.vocab_size]),
        "prompt_lookup": prompt_ids,
    }
    runs = {"plain": []}
    runs.update({c: [] for c in cases})
    spec = {}
    for _ in range(1 + args.reps):  # round 0 warms every graph and shape up
        t1, _ = timed(lambda: dec.generate_from_embeds(x, 1))
        tn, r = timed(lambda: dec.generate_from_embeds(x, N))
        assert torch.equal(r, ref)
        runs["plain"].append((tn - t1) * 1e3)
        for c, hist in cases.items():
            t1, _ = timed(lambda: dec.generate_from_embeds(x, 1, lookup_ids=hist, lookup_k=k))
            tn, r = timed(lambda: dec.generate_from_embeds(x, N, lookup_ids=hist, lookup_k=k))
            runs[c].append((tn - t1) * 1e3)
            spec[c] = dict(ids_identical=bool(torch.equal(r, ref)), last_speculation=list(dec.last_speculation))
    out = {"card": card(), "decode_pack": "packed" if any(v == "packed" for v in dec.decode_pack.values()) else "bf16", "prompt_rows": PROMPT_ROWS, "new_tokens": N,
           "k": k}
    med = {c: statistics.median(v[1:]) for c, v in runs.items()}
    out["decode_tokens_per_s"] = {c: round((N - 1) / (m / 1e3), 1) for c, m in med.items()}
    out["speedup_vs_plain"] = {c: round(med["plain"] / m, 3) for c, m in med.items() if c != "plain"}
    out["spec"] = spec
    # graph replay times of one step / one verify pass
    dec.generate_from_embeds(x, N, lookup_ids=cases["perfect"], lookup_k=k)  # reserves the pages a pass at position S may write
    dec._ensure_graph(0)
    steps = {"plain_step_ms": round(replay_ms(dec, dec._graph, PROMPT_ROWS), 4)}
    for T in range(2, ops.SPEC_T_MAX + 1):
        dec._verify_buffers()["state"].zero_()
        steps[f"verify_T{T}_ms"] = round(replay_ms(dec, dec._verify_graph(T, 2), PROMPT_ROWS), 4)
    out["graph_replay"] = steps
    print(json.dumps(out))


if __name__ == "__main__":
    main()
