"""Bit-identity of the Llama decoder's generation paths across a code change, in every weight format.

Builds seeded 4-layer decoders (hidden 2048, vocabulary 32003) over the same state dict in five formats - element type with the
decode step over the plain matrices (SRGPT_DECODE_PACK=0), 12-bit packed decode weights (bf16 only), NF4 with its dequantized copy,
NF4 planes only, and FP8 - in bf16 and fp16, and runs on each: greedy, sampled and processor-on generate_from_embeds (ids and
logits), prompt-lookup decoding (not FP8), generate_batch (one sequence at a time with logits, and the batched step greedy, with
processors and sampled), generate_beam_batch and score_candidates.  Every result array goes into one .npz:

    python tools/format_parity.py --save /tmp/parity_parent.npz      (at the old commit)
    python tools/format_parity.py --compare /tmp/parity_parent.npz   (at the new one: every array must be bitwise equal)
"""
import argparse
import dataclasses
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

DEV = "cuda"
DIMS = dict(hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16, num_key_value_heads=4, head_dim=128,
            vocab_size=32003)
FORMATS = ("plain", "packed", "nf4_copy", "nf4_planes", "fp8")
SPEC = dict(repetition_penalty=1.15, no_repeat_ngram_size=2, min_new_tokens=6)
SMP = dict(temperature=0.9, top_p=0.95, seed=11)


def state_dict(d, seed=21):
    g = torch.Generator().manual_seed(seed)
    H, I, hd = d.hidden_size, d.intermediate_size, d.head_dim
    rn = lambda *s, std=0.02: torch.randn(*s, generator=g) * std  # noqa: E731
    sd = {"model.embed_tokens.weight": rn(d.vocab_size, H, std=0.3), "model.norm.weight": 1 + rn(H, std=0.05),
          "lm_head.weight": rn(d.vocab_size, H, std=0.08)}
    for l in range(d.num_hidden_layers):
        p = f"model.layers.{l}."
        sd.update({p + "input_layernorm.weight": 1 + rn(H, std=0.05), p + "post_attention_layernorm.weight": 1 + rn(H, std=0.05),
                   p + "self_attn.q_proj.weight": rn(d.num_attention_heads * hd, H), p + "self_attn.k_proj.weight": rn(d.num_key_value_heads * hd, H),
                   p + "self_attn.v_proj.weight": rn(d.num_key_value_heads * hd, H), p + "self_attn.o_proj.weight": rn(H, d.num_attention_heads * hd),
                   p + "mlp.gate_proj.weight": rn(I, H), p + "mlp.up_proj.weight": rn(I, H), p + "mlp.down_proj.weight": rn(H, I)})
    return sd


def decoder(d, sd, fmt, dtype):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.weights import LlamaLayerW, LlamaW, _fp8_layer, _nf4_layer, interleave_rows
    g = lambda dd, k: dd[k].to(device=DEV, dtype=dtype)  # noqa: E731
    os.environ["SRGPT_DECODE_PACK"] = "0" if fmt == "plain" else "1"
    layers = []
    for l in range(d.num_hidden_layers):
        p = f"model.layers.{l}."
        if fmt.startswith("nf4"):
            layers.append(_nf4_layer(sd, p, g, dtype, dequantized_copy=fmt == "nf4_copy"))
        elif fmt == "fp8":
            layers.append(_fp8_layer(sd, p, g, dtype))
        else:
            layers.append(LlamaLayerW(
                in_norm=g(sd, p + "input_layernorm.weight"),
                qkv_w=torch.cat([g(sd, p + f"self_attn.{n}.weight") for n in ("q_proj", "k_proj", "v_proj")], 0).contiguous(),
                o_w=g(sd, p + "self_attn.o_proj.weight").contiguous(), post_norm=g(sd, p + "post_attention_layernorm.weight"),
                gateup_w=interleave_rows(g(sd, p + "mlp.gate_proj.weight"), g(sd, p + "mlp.up_proj.weight")),
                down_w=g(sd, p + "mlp.down_proj.weight").contiguous()))
    quant = {"nf4_copy": "nf4", "nf4_planes": "nf4", "fp8": "fp8"}.get(fmt)
    w = LlamaW(embed=g(sd, "model.embed_tokens.weight").contiguous(), norm=g(sd, "model.norm.weight"), lm_head=g(sd, "lm_head.weight").contiguous(),
               layers=layers, quantization=quant, nf4_dequantized_copy=fmt != "nf4_planes")
    return LlamaDecoder(d, w, max_seq_len=512, max_seqs=8)


def runs(dec, dtype):
    """name -> numpy array of every path's output on this decoder."""
    gen = torch.Generator().manual_seed(5)
    x = (torch.randn(24, DIMS["hidden_size"], generator=gen) * 0.3).to(dtype).to(DEV)
    lens = [12, 20, 7]
    xb = (torch.randn(sum(lens), DIMS["hidden_size"], generator=gen) * 0.3).to(dtype).to(DEV)
    out = {}
    ids, lg = dec.generate_from_embeds(x, 24, use_graph=False, return_logits=True)
    out["greedy_eager_ids"], out["greedy_eager_logits"] = ids, lg
    out["greedy_graph_ids"] = dec.generate_from_embeds(x, 24)
    ids, lg = dec.generate_from_embeds(x, 24, use_graph=False, return_logits=True, sampling=SMP)
    out["sampled_eager_ids"], out["sampled_eager_logits"] = ids, lg
    out["sampled_graph_ids"] = dec.generate_from_embeds(x, 24, sampling=SMP)
    ids, lg = dec.generate_from_embeds(x, 24, use_graph=False, return_logits=True, processors=SPEC)
    out["proc_eager_ids"], out["proc_eager_logits"] = ids, lg
    out["proc_graph_ids"] = dec.generate_from_embeds(x, 24, processors=SPEC)
    if not dec.fp8:
        hist = torch.tensor(out["greedy_graph_ids"].tolist() * 2)
        ids, lg = dec.generate_from_embeds(x, 24, use_graph=False, return_logits=True, lookup_ids=hist, lookup_k=3)
        out["lookup_eager_ids"], out["lookup_eager_logits"] = ids, lg
        out["lookup_graph_ids"] = dec.generate_from_embeds(x, 24, lookup_ids=hist, lookup_k=3)
    ids, lg = dec.generate_batch(xb, lens, 12, return_logits=True)  # one sequence at a time, through the one-token step
    for b in range(len(lens)):
        out[f"batch_seq_{b}_ids"], out[f"batch_seq_{b}_logits"] = ids[b], lg[b]
    for graph in (False, True):  # the batched step
        for b, t in enumerate(dec.generate_batch(xb, lens, 12, use_graph=graph)):
            out[f"batch_{graph}_{b}"] = t
        for b, t in enumerate(dec.generate_batch(xb, lens, 12, use_graph=graph, processors=SPEC)):
            out[f"batch_proc_{graph}_{b}"] = t
        for b, t in enumerate(dec.generate_batch(xb, lens, 12, use_graph=graph, sampling=SMP)):
            out[f"batch_sampled_{graph}_{b}"] = t
        for b, t in enumerate(dec.generate_beam_batch(xb, lens, 3, 10, use_graph=graph)):
            out[f"beam_{graph}_{b}"] = t
    cands = [[5], [17, 40], [3, 4, 5], [900, 901, 902, 903, 904]]
    out["score"] = dec.score_candidates(xb, lens, cands, 8)
    return {k: (v.float() if v.dtype in (torch.bfloat16, torch.float16) else v).cpu().numpy() for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    grp = ap.add_mutually_exclusive_group(required=True)
    grp.add_argument("--save")
    grp.add_argument("--compare")
    args = ap.parse_args()
    from spatialrgpt_b200.config import LlamaDims
    d = dataclasses.replace(LlamaDims(), **DIMS)
    sd = state_dict(d)
    res = {}
    for dtype, dname in ((torch.bfloat16, "bf16"), (torch.float16, "f16")):
        for fmt in FORMATS:
            if fmt == "packed" and dtype != torch.bfloat16:
                continue  # the 12-bit packing is a bf16 format
            dec = decoder(d, sd, fmt, dtype)
            info = (sorted(set(dec.decode_pack.values())), sorted(set(dec.decode_quant.values())), dec.kernels_per_decode_step)
            print(dname, fmt, info, flush=True)
            for k, v in runs(dec, dtype).items():
                res[f"{dname}/{fmt}/{k}"] = v
            del dec
            torch.cuda.empty_cache()
    if args.save:
        os.makedirs(os.path.dirname(os.path.abspath(args.save)), exist_ok=True)
        np.savez(args.save, **res)
        print(f"saved {len(res)} arrays to {args.save}")
        return
    ref = np.load(args.compare)
    bad = sorted(set(ref.files) ^ set(res))
    for k in sorted(set(ref.files) & set(res)):
        a, b = ref[k], res[k]
        if a.shape != b.shape or a.dtype != b.dtype or a.tobytes() != b.tobytes():
            bad.append(k)
    print(f"{len(res)} arrays, {len(bad)} differ" + (": " + ", ".join(bad[:40]) if bad else ""))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
