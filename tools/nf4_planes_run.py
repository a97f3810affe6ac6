"""Measure NF4 without the dequantized copy (nf4_dequantized_copy=False) against NF4 with it, at Llama-3-8B shapes: the full-depth decoder with
seeded random weights (as tools/nf4_run.py builds them), both arms built from the same weights and timed alternately in one run.

  * resident bytes of the layer matrices and the load peak of bf16, NF4 copy and NF4 planes-only;
  * layer 0's four NF4 GEMMs (srgpt_gemm_nf4_bf16) against srgpt_gemm_bf16 on the dequantized matrix at M = 32, 128, 259 and 8288 (32 x 259):
    microseconds (CUDA events, median, L2 flushed before each launch), TFLOP/s and GB/s of the bytes moved (A, the weights as stored, C);
  * the c2 prefill (259 rows), the c3 prefill (32 x 259 rows), the batched decode step at B = 32, the verify pass at T = 5 and the one-token
    step (graph replay), per arm;
  * the card name, power limit and SM clocks, read in the same run.

    python tools/nf4_planes_run.py [--reps 3]   (one JSON line on stdout)
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from spatialrgpt_b200 import baseline_config, ops  # noqa: E402
from spatialrgpt_b200.llama_decoder import LlamaDecoder  # noqa: E402
from spatialrgpt_b200.weights import LlamaW, _nf4_layer, random_init  # noqa: E402
from tools.nf4_run import PROMPT_ROWS, card, kernel_us, replay_ms, timed  # noqa: E402

MATS = ("qkv", "o", "gateup", "down")
B = 32


def nf4_weights(w: LlamaW, dims, copy: bool) -> LlamaW:
    """The same layer matrices, NF4-quantized per original matrix (the fused qkv / interleaved gate-up split back)."""
    qd, kd = dims.num_attention_heads * dims.head_dim, dims.num_key_value_heads * dims.head_dim
    layers = []
    for lw in w.layers:
        sd = {"input_layernorm.weight": lw.in_norm, "post_attention_layernorm.weight": lw.post_norm,
              "self_attn.q_proj.weight": lw.qkv_w[:qd], "self_attn.k_proj.weight": lw.qkv_w[qd:qd + kd],
              "self_attn.v_proj.weight": lw.qkv_w[qd + kd:], "self_attn.o_proj.weight": lw.o_w,
              "mlp.gate_proj.weight": lw.gateup_w[0::2], "mlp.up_proj.weight": lw.gateup_w[1::2], "mlp.down_proj.weight": lw.down_w}
        layers.append(_nf4_layer(sd, "", lambda d, k: d[k].contiguous(), w.embed.dtype, dequantized_copy=copy))
    return LlamaW(embed=w.embed, norm=w.norm, lm_head=w.lm_head, layers=layers, quantization="nf4", nf4_dequantized_copy=copy)


def layer_bytes(w: LlamaW) -> int:
    total = 0
    for lw in w.layers:
        for n in MATS:
            m = getattr(lw, n + "_w")
            total += m.nbytes() if not isinstance(m, torch.Tensor) else m.numel() * m.element_size()
            if isinstance(m, torch.Tensor) and lw.nf4 is not None and lw.nf4[n] is not None:
                total += lw.nf4[n].nbytes()
    return total


def load(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t, w = timed(fn)
    return w, {"load_s": round(t, 1), "layers_GB": round(layer_bytes(w) / 1e9, 3),
               "load_peak_over_start_GB": round((torch.cuda.max_memory_allocated() - base) / 1e9, 3),
               "growth_GB": round((torch.cuda.memory_allocated() - base) / 1e9, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nf4_planes_run.py measures on the GPU; no CUDA device found")
    out = {"card": card()}
    cfg = baseline_config("c2")
    d = cfg.llama
    w = random_init(cfg, "cuda", seed=0, n_tower_layers=0).llama
    out["bf16"] = {"layers_GB": round(layer_bytes(w) / 1e9, 3)}
    wc, out["nf4_copy"] = load(lambda: nf4_weights(w, d, True))
    wp, out["nf4_planes_only"] = load(lambda: nf4_weights(w, d, False))
    decs = {"copy": LlamaDecoder(d, wc, max_seq_len=1024, max_seqs=B), "planes": LlamaDecoder(d, wp, max_seq_len=1024, max_seqs=B)}
    dt = w.embed.dtype

    # layer 0's GEMMs
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    gemms = {}
    for m in MATS:
        deq, p = getattr(wc.layers[0], m + "_w"), wp.layers[0].nf4[m]
        N, K = deq.shape
        epi = ops.EPI_SWIGLU if m == "gateup" else ops.EPI_NONE
        n_out = N // 2 if m == "gateup" else N
        for M in (32, 128, 259, 8288):
            a = torch.randn(M, K, device="cuda").to(dt)
            c = torch.empty(M, n_out, dtype=dt, device="cuda")
            us_b = kernel_us(lambda: ops.gemm(a, deq, epilogue=epi, out=c), flush)
            us_n = kernel_us(lambda: ops.gemm_nf4(a, p, epilogue=epi, out=c), flush)
            ref = ops.gemm(a, deq, epilogue=epi)
            same = bool(torch.equal(ref.view(torch.int16), ops.gemm_nf4(a, p, epilogue=epi).view(torch.int16)))
            flop = 2.0 * M * N * K
            io = (M * K + M * n_out) * 2
            gemms[f"{m}_M{M}"] = {"bf16_us": round(us_b, 1), "nf4_us": round(us_n, 1), "nf4_over_bf16_time": round(us_n / us_b, 3),
                                  "bf16_TFLOPs": round(flop / us_b / 1e6, 1), "nf4_TFLOPs": round(flop / us_n / 1e6, 1),
                                  "bf16_GBps": round((io + deq.numel() * 2) / us_b / 1e3, 1), "nf4_GBps": round((io + p.nbytes()) / us_n / 1e3, 1),
                                  "bit_identical": same}
    out["layer0_gemm"] = gemms

    g = torch.Generator().manual_seed(7)
    prompt_ids = torch.randint(1000, 30000, (PROMPT_ROWS,), generator=g)
    x = decs["copy"].embed_tokens(prompt_ids)
    packed = decs["copy"].embed_tokens(torch.randint(1000, 30000, (B * PROMPT_ROWS,), generator=g))
    lens = [PROMPT_ROWS] * B
    runs = {a: {k: [] for k in ("c2_prefill_ms", "c3_prefill_ms", "batched_step_ms", "verify_ms_per_token", "step_ms")} for a in decs}
    res = {}
    for rep in range(1 + args.reps):  # round 0 warms up every shape and graph
        for a, dec in decs.items():
            r = runs[a]
            t, _ = timed(lambda: dec.prefill_hidden(x))
            r["c2_prefill_ms"].append(t * 1e3)
            dec.cache.reserve_many(lens)
            t, _ = timed(lambda: dec.prefill_packed(packed, lens))
            r["c3_prefill_ms"].append(t * 1e3)
            t1, _ = timed(lambda: dec.generate_batch(packed, lens, 1))
            t17, ids_b = timed(lambda: dec.generate_batch(packed, lens, 17))
            r["batched_step_ms"].append((t17 - t1) * 1e3 / 16)
            t1, _ = timed(lambda: dec.generate_from_embeds(x, 1))
            t65, ids_v = timed(lambda: dec.generate_from_embeds(x, 65, lookup_ids=prompt_ids, lookup_k=4))
            r["verify_ms_per_token"].append((t65 - t1) * 1e3 / 64)
            r["step_ms"].append(replay_ms(dec, PROMPT_ROWS))
            res[a] = (torch.stack([t.cpu() for t in ids_b]) if isinstance(ids_b, (list, tuple)) else ids_b.cpu(), ids_v.cpu())
    out["timings_median"] = {a: {k: round(statistics.median(v[1:]), 3) for k, v in r.items()} for a, r in runs.items()}
    out["timings_all"] = {a: {k: [round(x, 3) for x in v[1:]] for k, v in r.items()} for a, r in runs.items()}
    out["ids_equal"] = bool(all(torch.equal(p, q) for p, q in zip(res["copy"], res["planes"])))
    out["speculation_last"] = list(decs["planes"].last_speculation)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
