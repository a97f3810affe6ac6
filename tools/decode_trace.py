"""In-graph timeline of one decode step (c2, Llama-3-8B) from the kernels' own %globaltimer marks
(srgpt_trace_begin/end) — shows how much of the step is streaming and how much is kernel boundaries."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from spatialrgpt_b200 import _lib, baseline_config, ops
from spatialrgpt_b200.llava_llama import LlavaLlamaModel
from spatialrgpt_b200.synth import synth_request
from spatialrgpt_b200.weights import random_init

cfg = baseline_config("c2")
dev = torch.device("cuda", 0)
model = LlavaLlamaModel(cfg, random_init(cfg, dev, seed=0, n_tower_layers=cfg.vision.num_hidden_layers - 1), max_seq_len=1024)
ids, im, de, mk = synth_request(cfg, 8, 64, 1234)
model.generate(ids.to(dev), images=im.to(dev), depths=de.to(dev), masks=[mk[0].to(dev)], do_sample=False, max_new_tokens=8)
llm = model.llm
n = 5 * cfg.llama.num_hidden_layers + 1   # traced launches per step (the 1-CTA finalize kernel is not traced)
buf = torch.zeros(2 * n + 8, 4, dtype=torch.int64, device=dev)
lib = _lib.load()
llm._drop_graphs()
lib.srgpt_trace_begin(buf.data_ptr(), 2 * n + 8)
llm._ensure_graph(0)           # capture with trace records baked into the kernel parameters
used = lib.srgpt_trace_end()
BIG = torch.iinfo(torch.int64).max


def reset():
    buf[:, 0:2] = BIG
    buf[:, 2:4] = 0


names = []
for l in range(cfg.llama.num_hidden_layers):
    names += [f"L{l}.qkv_rope", f"L{l}.attn", f"L{l}.o_proj", f"L{l}.gateup", f"L{l}.down"]
names += ["lm_head"]
best = None
for it in range(6):
    reset()
    torch.cuda.synchronize()
    llm._graph.replay()
    torch.cuda.synchronize()
    rec = buf.cpu()[n: n + len(names)].clone()   # records [0,n) belong to the eager warm-up step, [n,2n) to the graph
    total = int(rec[:, 2].max() - rec[:, 0].min())
    if it >= 2 and (best is None or total < best[0]):
        best = (total, rec)
total, rec = best
t0 = int(rec[0, 0])
print(f"records used by capture: {used} (eager warm-up + capture), kernels per step: {n}")
print(f"decode step (first CTA start -> last CTA end): {total/1e3:.1f} us")
kinds = {}
rows = []
prev_end = None
for i, nm in enumerate(names):
    s, w, e, c = (int(v) for v in rec[i])
    kind = nm.split(".")[-1]
    gap = (s - prev_end) if prev_end is not None else 0      # <0: started before the previous kernel ended (PDL)
    wait_gap = (w - prev_end) if prev_end is not None else 0  # dependency release -> first CTA past the wait
    d = kinds.setdefault(kind, dict(n=0, dur=0, busy=0, early=0, rel=0))
    d["n"] += 1; d["dur"] += e - s; d["busy"] += e - max(w, prev_end or w); d["early"] += -gap; d["rel"] += wait_gap
    rows.append((nm, (s - t0) / 1e3, (w - t0) / 1e3, (e - t0) / 1e3, c))
    prev_end = e
print("first layer timeline (us): name start after_wait end ctas")
for r in rows[:10] + rows[-6:]:
    print("  %-14s %8.2f %8.2f %8.2f %6d" % r)
print("per kernel kind: count, mean start->end, mean (end - max(after_wait, prev_end)) = exposed time, mean early start before prev end, mean prev_end->after_wait")
summary = {}
for k, d in kinds.items():
    summary[k] = {kk: round(v / d["n"] / 1e3, 2) for kk, v in d.items() if kk != "n"}
    summary[k]["n"] = d["n"]
    print("  %-10s n=%3d  dur=%7.2f  exposed=%7.2f  early=%6.2f  release=%6.2f" % (k, d["n"], *(summary[k][x] for x in ("dur", "busy", "early", "rel"))))
print(json.dumps({"step_us": total / 1e3, "kinds": summary}))
# JSON lines for tools/ab.py (microseconds in the ms_median field)
print(json.dumps({"kernel": "decode_step_us", "ms_median": round(total / 1e3, 2)}))
for k, d in summary.items():
    print(json.dumps({"kernel": f"exposed_us {k}", "ms_median": d["busy"]}))
    print(json.dumps({"kernel": f"release_us {k}", "ms_median": d["rel"]}))
