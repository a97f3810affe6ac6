"""Measure NF4 decode at c2 shapes: the full-depth Llama-3-8B decoder with seeded random weights, a 259-row prompt, batch 1, 128 greedy
tokens, in three arms that alternate in one run: bf16 (SRGPT_DECODE_PACK=0), the lossless 12-bit packing (the default) and NF4 (the same
weights quantized at load; lm_head packed as in the packed arm).

  * decode-phase ms per token and tokens/s of one request ((t(128 tokens) - t(1 token)) / 127, host clock around work that ends in a
    device synchronise), and the graph-replayed decode step (CUDA events, median);
  * per-GEMV time of layer 0's four matrices, NF4 against packed-12 (CUDA events, L2 flushed before each launch, median), with the
    bytes each streams;
  * weight bytes streamed per token by each arm's decode step;
  * the card name, power limit and SM clocks, read in the same run.

    python tools/nf4_run.py [--reps 3] [--new-tokens 128]   (one JSON line on stdout)
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
from spatialrgpt_b200.weights import LlamaW, _nf4_layer, random_init  # noqa: E402

PROMPT_ROWS = 259  # c2: 256 image rows + the question
MATS = ("qkv", "o", "gateup", "down")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        smi = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in smi.split(","))))
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "nvidia-smi": f"unavailable ({e})"}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def replay_ms(dec, S, n=30):
    dec._ensure_graph(0)
    ts = []
    for i in range(n + 5):
        dec.pos.fill_(S)
        dec.step.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dec._graph.replay()
        b.record()
        b.synchronize()
        if i >= 5:
            ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def kernel_us(fn, flush, n=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return statistics.median(ts)


def nf4_weights(w: LlamaW, dims) -> LlamaW:
    """The same layer matrices, NF4-quantized per original matrix (the fused qkv / interleaved gate-up split back)."""
    qd, kd = dims.num_attention_heads * dims.head_dim, dims.num_key_value_heads * dims.head_dim
    layers = []
    for lw in w.layers:
        sd = {"input_layernorm.weight": lw.in_norm, "post_attention_layernorm.weight": lw.post_norm,
              "self_attn.q_proj.weight": lw.qkv_w[:qd], "self_attn.k_proj.weight": lw.qkv_w[qd:qd + kd],
              "self_attn.v_proj.weight": lw.qkv_w[qd + kd:], "self_attn.o_proj.weight": lw.o_w,
              "mlp.gate_proj.weight": lw.gateup_w[0::2], "mlp.up_proj.weight": lw.gateup_w[1::2], "mlp.down_proj.weight": lw.down_w}
        layers.append(_nf4_layer(sd, "", lambda d, k: d[k].contiguous(), w.embed.dtype))
    return LlamaW(embed=w.embed, norm=w.norm, lm_head=w.lm_head, layers=layers, quantization="nf4")


def stream_bytes(dec) -> int:
    """Weight bytes one decode step streams: each layer matrix from its NF4 planes, packed planes or element-type copy, and lm_head."""
    total = 0
    for l, lw in enumerate(dec.w.layers):
        for i, m in enumerate(MATS):
            if dec.decode_quant.get(f"layers.{l}.{m}") == "nf4":
                total += lw.nf4[m].nbytes()
            elif dec.decode_pack.get(f"layers.{l}.{m}") == "packed":
                total += dec.stack.packed_layers[l][m].nbytes()
            else:
                t = getattr(lw, m + "_w")
                total += t.numel() * t.element_size()
    return total + (dec.stack.lm_packed.nbytes() if dec.stack.lm_packed is not None else dec.w.lm_head.numel() * dec.w.lm_head.element_size())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nf4_run.py measures on the GPU; no CUDA device found")
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    os.environ["SRGPT_DECODE_PACK"] = "0"
    decs = {"bf16": LlamaDecoder(d, w, max_seq_len=1024)}
    os.environ["SRGPT_DECODE_PACK"] = "1"
    decs["packed12"] = LlamaDecoder(d, w, max_seq_len=1024)
    t_q, wq = timed(lambda: nf4_weights(w, d))
    decs["nf4"] = LlamaDecoder(d, wq, max_seq_len=1024)
    assert "packed" in decs["packed12"].decode_pack.values() and "nf4" in decs["nf4"].decode_quant.values()
    prompt_ids = torch.randint(1000, 30000, (PROMPT_ROWS,), generator=torch.Generator().manual_seed(7))
    x = decs["bf16"].embed_tokens(prompt_ids)
    N = args.new_tokens
    runs = {a: [] for a in decs}
    ids = {}
    for _ in range(1 + args.reps):  # round 0 warms every graph up
        for a, dec in decs.items():
            t1, _ = timed(lambda: dec.generate_from_embeds(x, 1))
            tn, r = timed(lambda: dec.generate_from_embeds(x, N))
            runs[a].append((tn - t1) * 1e3 / (N - 1))
            ids[a] = r.cpu()
    out = {"card": card(), "prompt_rows": PROMPT_ROWS, "new_tokens": N, "reps": args.reps, "nf4_quantize_s": round(t_q, 2)}
    out["decode_ms_per_token"] = {a: [round(v, 4) for v in r[1:]] for a, r in runs.items()}
    out["decode_tokens_per_s"] = {a: round(1e3 / statistics.median(r[1:]), 1) for a, r in runs.items()}
    out["graph_step_ms"] = {a: round(replay_ms(dec, PROMPT_ROWS), 4) for a, dec in decs.items()}
    out["weight_GB_per_token"] = {a: round(stream_bytes(dec) / 1e9, 3) for a, dec in decs.items()}
    out["packed12_ids_equal_bf16"] = bool(torch.equal(ids["bf16"], ids["packed12"]))
    out["nf4_ids_equal_bf16"] = int((ids["nf4"] == ids["bf16"]).long().cumprod(0).sum())  # leading tokens in common (lossy weights)
    # per-GEMV: layer 0 of each arm, L2 flushed before each launch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    pk, nf = decs["packed12"].stack.packed_layers[0], wq.layers[0].nf4
    H, I, nh, nkv, hd = d.hidden_size, d.intermediate_size, d.num_attention_heads, d.num_key_value_heads, d.head_dim
    dec = decs["nf4"]
    xh = torch.randn(H, device="cuda").to(w.embed.dtype)
    xi = torch.randn(I, device="cuda").to(w.embed.dtype)
    pages = torch.zeros(64, 2, 16, nkv, hd, dtype=w.embed.dtype, device="cuda")
    pt = torch.arange(64, dtype=torch.int32, device="cuda")
    pos = torch.tensor([300], dtype=torch.int32, device="cuda")
    gemvs = {}
    for m in MATS:
        if m == "qkv":
            y = torch.empty(nh * hd, dtype=w.embed.dtype, device="cuda")
            kw = dict(x=xh, y=y, norm_weight=w.layers[0].in_norm, eps=d.rms_norm_eps, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd,
                      cos_tab=dec.cos, sin_tab=dec.sin, pos=pos, kv_pages=pages, page_table=pt, page_size=16)
        elif m == "gateup":
            kw = dict(x=xh, y=torch.empty(I, dtype=w.embed.dtype, device="cuda"), norm_weight=w.layers[0].post_norm, eps=d.rms_norm_eps,
                      mode=ops.GEMV_SWIGLU)
        else:
            xin = xh if m == "o" else xi
            kw = dict(x=xin, y=torch.empty(H, dtype=w.embed.dtype, device="cuda"), residual=torch.randn(H, device="cuda").to(w.embed.dtype))
        x_, y_ = kw.pop("x"), kw.pop("y")
        us_p = kernel_us(lambda: ops.gemv_packed(x_, pk[m], y_, **kw), flush)
        us_n = kernel_us(lambda: ops.gemv_nf4(x_, nf[m], y_, **kw), flush)
        gemvs[m] = {"packed12_us": round(us_p, 2), "nf4_us": round(us_n, 2), "packed12_GBps": round(pk[m].nbytes() / us_p / 1e3, 1),
                    "nf4_GBps": round(nf[m].nbytes() / us_n / 1e3, 1)}
    out["layer0_gemv"] = gemvs
    print(json.dumps(out))


if __name__ == "__main__":
    main()
