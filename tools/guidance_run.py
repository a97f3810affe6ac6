"""Measure classifier-free guidance at c2 shapes: the full-depth Llama-3-8B decoder with seeded random weights (packed decode weights
unless SRGPT_DECODE_PACK=0), B prompts of 259 rows each, a 64-token image-free negative prompt per prompt, 128 greedy tokens, for
B = 1, 2, 4.  Three modes alternate:

  * generate: what an unguided generate() of the B prompts runs - batch 1's one-token step (generate_from_embeds) at B = 1, the
    batched step (generate_batch) at B > 1;
  * rows: generate_rows over the B prompts (the batch-invariant rows step over B rows, what generate(batch_invariant=True) runs);
  * guided: the same prompts with the negative prompts and guidance_scale 3 (the rows step over 2B rows plus the guidance kernel),
    what generate(guidance_scale=3, negative_prompt_ids=...) runs;
guided_vs_generate / guided_vs_rows: the guided step time over the generate / rows step time, the cost of turning guidance on against
either baseline.
Each is timed as the decode phase, (t(128 tokens) - t(1 token)) with a host clock around work that ends in a device synchronise, so
prefill and the first token drop out; step_ms = decode time / 127 and tokens_per_s = B * 127 / decode time (new tokens of the prompts;
the unconditional rows are not counted).  prefill_ms = t(1 token), the prefills and the first token.  Medians of --reps rounds after a
warm-up round.  guidance_kernel_us: device time of one srgpt_guidance_rows launch over the 2B logits rows (greedy), from CUDA events
around 200 launches.  The card's name, power limit and maximum SM clock are read in the same run, and the SM clock is sampled with
nvidia-smi every 2 s while the modes run (sm_clock_mhz_under_load: min / median / max of the samples).

    python tools/guidance_run.py [--reps 3] [--new-tokens 128]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import random_init  # noqa: E402
from tools.batch_invariant_run import card, timed  # noqa: E402

PROMPT_ROWS = 259  # c2: 256 image rows + the question
NEG_ROWS = 64
ROWS = (1, 2, 4)
SCALE = 3.0


def kernel_us(dec, B: int, n: int = 200) -> float:
    st = dec._guidance_state()
    lg, ids = st["logits"][:2 * B], st["ids"][:2 * B]
    ops.guidance_rows(lg, st["scale"], st["guided"][:B], ids=ids)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        ops.guidance_rows(lg, st["scale"], st["guided"][:B], ids=ids)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("guidance_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    dec = LlamaDecoder(cfg.llama, w, max_seq_len=1024)
    g = torch.Generator().manual_seed(7)
    prompts = [dec.embed_tokens(torch.randint(1000, 30000, (PROMPT_ROWS,), generator=g)) for _ in range(max(ROWS))]
    negs = [dec.embed_tokens(torch.randint(1000, 30000, (NEG_ROWS,), generator=g)) for _ in range(max(ROWS))]
    N = args.new_tokens
    modes = {
        "generate": lambda B, n: ([dec.generate_from_embeds(prompts[0], n)] if B == 1 else
                                  dec.generate_batch(torch.cat(prompts[:B]), [PROMPT_ROWS] * B, n)),
        "rows": lambda B, n: dec.generate_rows(prompts[:B], n),
        "guided": lambda B, n: dec.generate_rows(prompts[:B], n, guidance_scale=SCALE, negative_embeds=negs[:B]),
    }
    clocks, stop = [], threading.Event()

    def sample_clock():
        while not stop.wait(2.0):
            try:
                q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                                   text=True, timeout=10).stdout.strip()
                clocks.append(float(q))
            except Exception:
                pass
    sampler = threading.Thread(target=sample_clock, daemon=True)
    sampler.start()
    times = {(m, B): [] for m in modes for B in ROWS}
    pre = {(m, B): [] for m in modes for B in ROWS}
    for _ in range(1 + args.reps):  # round 0 warms every graph and shape up
        for B in ROWS:
            for m, fn in modes.items():
                t1, _ = timed(lambda: fn(B, 1))
                tn, _ = timed(lambda: fn(B, N))
                times[(m, B)].append(tn - t1)
                pre[(m, B)].append(t1)
    stop.set()
    sampler.join()
    under_load = [min(clocks), statistics.median(clocks), max(clocks)] if clocks else "no samples"
    out = {"card": dict(card(), sm_clock_mhz_under_load=under_load),
           "decode_pack": "packed" if any(v == "packed" for v in dec.decode_pack.values()) else "bf16",
           "prompt_rows": PROMPT_ROWS, "negative_rows": NEG_ROWS, "guidance_scale": SCALE, "new_tokens": N, "reps": args.reps}
    for B in ROWS:
        row = {}
        for m in modes:
            t = statistics.median(times[(m, B)][1:])
            row[m] = {"step_ms": round(t * 1e3 / (N - 1), 3), "tokens_per_s": round(B * (N - 1) / t, 1),
                      "prefill_ms": round(statistics.median(pre[(m, B)][1:]) * 1e3, 2)}
        row["guided_vs_generate"] = round(row["guided"]["step_ms"] / row["generate"]["step_ms"], 3)
        row["guided_vs_rows"] = round(row["guided"]["step_ms"] / row["rows"]["step_ms"], 3)
        row["guidance_kernel_us"] = round(kernel_us(dec, B), 1)
        out[f"B{B}"] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
