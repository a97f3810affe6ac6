"""FP8 (E4M3) W8A8 decoder measurement on one GPU; prints one JSON line.

Seeded random weights of config c2's Llama-3-8B decoder, resident at once in four formats: bf16 (plain one-token step), packed (the 12-bit
lossless decode stream), NF4 and FP8.  Reports
  * the GPU name and power limit (read-only nvidia-smi query);
  * one-token decode step time and tokens/s per format, rounds alternating between the formats: (time of generate(128 tokens) - time of
    generate(1 token)) / 127 after a 64-row prompt, graph replay, CUDA events;
  * GB/s of the FP8 decode GEMV per layer matrix of layer 0 (plain mode, codes + row scales over time, graph replay);
  * the packed 32 x 259-row prefill of all layers, FP8 against bf16 (ms, and TFLOP/s of the layer linears' algorithmic FLOPs);
  * FP8-vs-bf16 greedy agreement over the 128 tokens (random weights: for information only, not an accuracy measurement).
Needs a CUDA GPU; there is no CPU fallback.  Usage: python tools/fp8_run.py [--rounds R]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if out.returncode != 0:
        return None, None
    name, power = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return name, power


def llama_weights(d, dev, seed=0, std=0.02):
    """The same seeded layer matrices as plain bf16 layers, NF4 layers and FP8 layers; embeddings and lm_head shared."""
    from spatialrgpt_b200.weights import LlamaLayerW, LlamaW, _fp8_layer, _nf4_layer, interleave_rows
    gen = torch.Generator(device=dev).manual_seed(seed)
    H, I, hd = d.hidden_size, d.intermediate_size, d.head_dim

    def rn(*shape, s=std):
        return (torch.randn(*shape, generator=gen, device=dev) * s).to(torch.bfloat16)

    embed, lm_head, norm = rn(d.vocab_size, H, s=0.3), rn(d.vocab_size, H, s=0.08), (1 + 0.05 * torch.randn(H, generator=gen, device=dev)).to(torch.bfloat16)
    plain, nf4, fp8 = [], [], []
    g = lambda dd, k: dd[k]  # noqa: E731
    for i in range(d.num_hidden_layers):
        p = f"model.layers.{i}."
        sd = {p + "input_layernorm.weight": norm.clone(), p + "post_attention_layernorm.weight": norm.clone(),
              p + "self_attn.q_proj.weight": rn(d.num_attention_heads * hd, H), p + "self_attn.k_proj.weight": rn(d.num_key_value_heads * hd, H),
              p + "self_attn.v_proj.weight": rn(d.num_key_value_heads * hd, H), p + "self_attn.o_proj.weight": rn(H, d.num_attention_heads * hd),
              p + "mlp.gate_proj.weight": rn(I, H), p + "mlp.up_proj.weight": rn(I, H), p + "mlp.down_proj.weight": rn(H, I)}
        a = p + "self_attn."
        plain.append(LlamaLayerW(in_norm=sd[p + "input_layernorm.weight"],
                                 qkv_w=torch.cat([sd[a + n + ".weight"] for n in ("q_proj", "k_proj", "v_proj")]).contiguous(),
                                 o_w=sd[a + "o_proj.weight"], post_norm=sd[p + "post_attention_layernorm.weight"],
                                 gateup_w=interleave_rows(sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]), down_w=sd[p + "mlp.down_proj.weight"]))
        nf4.append(_nf4_layer(sd, p, g, torch.bfloat16))
        fp8.append(_fp8_layer(sd, p, g, torch.bfloat16))
        del sd
    mk = lambda layers, q: LlamaW(embed=embed, norm=norm, lm_head=lm_head, layers=layers, quantization=q)  # noqa: E731
    return mk(plain, None), mk(nf4, "nf4"), mk(fp8, "fp8")


def elapsed_ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_run.py needs a CUDA GPU")
    from spatialrgpt_b200 import ops
    from spatialrgpt_b200.config import baseline_config
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    d = baseline_config("c2").llama
    w_plain, w_nf4, w_fp8 = llama_weights(d, dev)
    os.environ["SRGPT_DECODE_PACK"] = "0"
    decs = {"bf16": LlamaDecoder(d, w_plain, max_seq_len=1024)}
    os.environ["SRGPT_DECODE_PACK"] = "1"
    decs["packed"] = LlamaDecoder(d, w_plain, max_seq_len=1024)
    decs["nf4"] = LlamaDecoder(d, w_nf4, max_seq_len=1024)
    decs["fp8"] = LlamaDecoder(d, w_fp8, max_seq_len=1024)
    assert "packed" in decs["packed"].decode_pack.values() and "nf4" in decs["nf4"].decode_quant.values() and decs["fp8"].fp8
    x = (torch.randn(64, d.hidden_size, generator=torch.Generator().manual_seed(1)) * 0.3).to(torch.bfloat16).to(dev)
    n = args.tokens
    ids = {k: dec.generate_from_embeds(x, n) for k, dec in decs.items()}  # warm-up: graphs captured
    step_ms = {k: [] for k in decs}
    for _ in range(args.rounds):
        for k, dec in decs.items():
            t_all = elapsed_ms(lambda: dec.generate_from_embeds(x, n))
            t_one = elapsed_ms(lambda: dec.generate_from_embeds(x, 1))
            step_ms[k].append((t_all - t_one) / (n - 1))
    decode = {k: dict(step_ms=round(statistics.median(v), 4), tokens_per_s=round(1000.0 / statistics.median(v), 1)) for k, v in step_ms.items()}
    # the FP8 decode GEMV over every layer matrix of layer 0
    lw, H = w_fp8.layers[0], d.hidden_size
    qd, I = d.num_attention_heads * d.head_dim, d.intermediate_size
    gbps = {}
    for name in ("qkv", "o", "gateup", "down"):
        wt = getattr(lw, name + "_w")
        N, K = wt.shape
        xin = torch.randn(K, device=dev).to(torch.bfloat16)
        out = torch.empty(N, dtype=torch.bfloat16, device=dev)
        run = lambda: ops.gemv_fp8(xin, wt, out)  # noqa: E731
        run()  # kernel attributes set outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()  # timed as the step runs it: replayed, without the Python launch path
        with torch.cuda.graph(graph):
            for _ in range(20):
                run()
        graph.replay()
        ms = elapsed_ms(graph.replay, reps=10) / 20
        gbps[name] = dict(N=N, K=K, us=round(ms * 1000, 2), GBps=round(wt.nbytes() / (ms * 1e-3) / 1e9, 1))
    # packed 32 x 259-row prefill
    B, S = 32, 259
    emb = (torch.randn(B * S, H, generator=torch.Generator().manual_seed(2)) * 0.3).to(torch.bfloat16).to(dev)
    flops = 2.0 * B * S * d.num_hidden_layers * (H * (qd + 2 * d.num_key_value_heads * d.head_dim) + qd * H + H * 2 * I + I * H)
    prefill = {}
    for k in ("bf16", "fp8"):
        dec = decs[k]
        dec.ensure_capacity(B, S)
        dec.cache.reserve_many([S] * B)
        dec.prefill_packed(emb, [S] * B)
        ms = statistics.median(elapsed_ms(lambda: dec.prefill_packed(emb, [S] * B)) for _ in range(args.rounds))
        prefill[k] = dict(ms=round(ms, 3), layer_linear_TFLOPs=round(flops / (ms * 1e-3) / 1e12, 1))
    a, b = ids["fp8"].cpu(), ids["bf16"].cpu()
    name, power = gpu_name_and_power()
    print(json.dumps(dict(gpu=name, power_limit=power, config="c2 Llama-3-8B decoder, seeded random weights, bf16 activations",
                          decode_64_row_prompt_128_tokens=decode, fp8_gemv_layer0=gbps, prefill_32x259=prefill,
                          fp8_vs_bf16_greedy=dict(leading_agreement=int((a == b).long().cumprod(0).sum()), equal_positions=int((a == b).sum()), tokens=n))))


if __name__ == "__main__":
    main()
