"""Measure the logits processors at c2 shapes: the full-depth Llama-3-8B decoder with seeded random weights (packed decode weights unless
SRGPT_DECODE_PACK=0), a 259-row prompt, batch 1, greedy, 128 new tokens.

  * decode-phase tokens/s ((t(128 tokens) - t(1 token)) / 127, host clock around work that ends in a device synchronise) with the
    processors off and on (repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=8), alternating over --reps rounds; medians;
  * the graph-replayed decode step with processing off and on (CUDA events, warmed up, median);
  * the processing kernels alone (processing + key unpack + pick, as the greedy step runs them) at history 0 / 128 / 4096, CUDA events
    over many launches.
The card name, power limit and max SM clock are read in the same run.

    python tools/logits_processors_run.py [--reps 3] [--new-tokens 128]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, logits_processors, ops  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.spec_decode_run import PROMPT_ROWS, card, replay_ms, timed  # noqa: E402

PROCESSORS = dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=8)
EOS = 128009  # Llama-3's <|eot_id|>: the minimum length bans it on the device (the request itself is not cut at EOS)


def kernel_us(dec, hist_len: int, n: int = 2000) -> float:
    """Processing + unpack + pick of the one-token step over a history of hist_len tokens, per launch."""
    V = dec.dims.vocab_size
    raw = torch.randn(V, device="cuda")
    dec.out_ids[:hist_len].copy_(torch.randint(0, V, (hist_len,)))
    step = torch.tensor([hist_len + 1], dtype=torch.int32, device="cuda")
    w = dec.w

    def once():
        ops.logits_process(raw, dec.out_ids, 0, 1, step, -1, dec.proc_fparams, dec.proc_spec, ids=dec.proc_ids)
        ops.logits_pick_token(dec.proc_ids, step, -1, dec.out_ids, w.embed, dec.h)

    for _ in range(50):
        once()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        once()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logits_processors_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=8192, max_new_tokens_cap=4608)
    g = torch.Generator().manual_seed(7)
    x = dec.embed_tokens(torch.randint(1000, 30000, (PROMPT_ROWS,), generator=g))
    spec = logits_processors.resolve_min_length(logits_processors.parse(**PROCESSORS, eos_token_id=EOS,
                                                                         vocab_size=cfg.llama.vocab_size), PROMPT_ROWS)
    N = args.new_tokens
    runs = {"off": [], "on": []}
    ids = {}
    for _ in range(1 + args.reps):  # round 0 captures both graphs
        for mode, p in (("off", None), ("on", spec)):
            t1, _ = timed(lambda: dec.generate_from_embeds(x, 1, processors=p))
            tn, r = timed(lambda: dec.generate_from_embeds(x, N, processors=p))
            runs[mode].append((tn - t1) * 1e3)
            ids[mode] = r
    med = {m: statistics.median(v[1:]) for m, v in runs.items()}
    out = {"card": card(), "decode_pack": "packed" if any(v == "packed" for v in dec.decode_pack.values()) else "bf16", "prompt_rows": PROMPT_ROWS, "new_tokens": N,
           "processors": PROCESSORS, "decode_tokens_per_s": {m: round((N - 1) / (t / 1e3), 1) for m, t in med.items()},
           "ids_differ": bool(not torch.equal(ids["off"], ids["on"]))}
    dec.generate_from_embeds(x, N, processors=spec)
    g_off, g_on = dec._ensure_graph(0), dec._ensure_graph(0, proc=True)
    off_ms, on_ms = replay_ms(dec, g_off, PROMPT_ROWS, 60), replay_ms(dec, g_on, PROMPT_ROWS, 60)
    out["graph_replay_ms"] = {"off": round(off_ms, 4), "on": round(on_ms, 4), "delta_pct": round(100 * (on_ms - off_ms) / off_ms, 2)}
    out["processing_kernels_us"] = {f"history_{n}": round(kernel_us(dec, n), 2) for n in (0, 128, 4096)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
