"""NF4 weight-only quantization on the H100, in both element types: the device quantizer against the numpy restatement
(tests/nf4_ref.py) bit for bit, every NF4 GEMV mode against the plain kernel on the dequantized matrix bit for bit, graph decode with the
NF4 step against the plain step over the dequantized copy, generate() on the tiny fixtures against the fp32 oracle run on the
numpy-dequantized weights, and the loader."""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import srgpt_oracle as O
from tests import nf4_ref as R
from tests.golden.make_golden import CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
ELEM = {torch.bfloat16: "bf16", torch.float16: "f16"}
DTYPES = [torch.bfloat16, torch.float16]


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def matrix(N, K, seed, dtype, std=0.02):
    """[N, K] ~ N(0, std) with an all-zero block, a block of subnormals beside zeros, and single large outliers."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * std
    w[0, :64] = 0
    tiny = torch.finfo(dtype).tiny
    w[1, 64:128] = 0
    w[1, 64:72] = torch.tensor([tiny / 2, -tiny / 4, tiny / 8, 0, -tiny / 2, tiny / 16, 0, tiny / 2])
    rows = torch.randint(2, N, (6,), generator=g)
    cols = torch.randint(0, K, (6,), generator=g)
    w[rows, cols] = torch.tensor([3.0, -2.5, 1.7, -4.0, 2.2, 6.0])
    return w.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [256, 640, 4096, 14336])
def test_device_quantizer_matches_the_numpy_restatement(ops, dtype, K):
    N = 96 if K > 4096 else 160
    w = matrix(N, K, K, dtype)
    with ops.elem_dtype(dtype):
        codes, scale = ops.nf4_quantize(w.to(DEV))
        deq = ops.nf4_dequantize(codes, scale)
        q, s_ref, deq_ref = R.quantize_all(w.float().numpy(), ELEM[dtype])
        assert np.array_equal(codes.cpu().numpy(), R.pack_natural(q))
        assert np.array_equal(scale.cpu().numpy().view(np.uint32), s_ref.view(np.uint32))
        assert np.array_equal(deq.float().cpu().numpy().view(np.uint32), deq_ref.view(np.uint32))
        if K % 1024 == 0:
            p, why = ops.nf4_planes(codes, scale, deq)
            assert why is None and np.array_equal(p.q.cpu().numpy(), R.lane_order(q))
        else:
            assert ops.nf4_planes(codes, scale, deq) == (None, f"K = {K} is not a multiple of 1024")


def test_quantizer_rejects_inf_nan_and_odd_widths(ops):
    w = matrix(64, 1024, 1, torch.bfloat16).to(DEV)
    for bad in (float("inf"), float("nan")):
        v = w.clone()
        v[3, 100] = bad
        with pytest.raises(ops.SrgptError, match="Inf or NaN"):
            ops.nf4_quantize(v)
    with pytest.raises(NotImplementedError):
        ops.nf4_quantize(torch.zeros(8, 96, dtype=torch.bfloat16, device=DEV))


def test_round_trip_check_raises_on_a_corrupted_plane(ops):
    w = matrix(64, 2048, 2, torch.bfloat16).to(DEV)
    codes, scale = ops.nf4_quantize(w)
    deq = ops.nf4_dequantize(codes, scale)
    p, _ = ops.nf4_planes(codes, scale, deq)
    assert _same(ops.nf4_unpack(p), deq)
    bad = deq.clone()
    bad[5, 7] = bad[5, 7] + 1
    with pytest.raises(ops.SrgptError):
        ops.nf4_planes(codes, scale, bad)


def _quantized(ops, w, dtype):
    codes, scale = ops.nf4_quantize(w)
    deq = ops.nf4_dequantize(codes, scale)
    return ops.nf4_planes(codes, scale, deq)[0], deq


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [1024, 2048, 4096, 5120, 14336])
def test_plain_and_swiglu_modes_are_bit_identical(ops, dtype, K):
    N = 1024
    with ops.elem_dtype(dtype):
        p, deq = _quantized(ops, matrix(N, K, K + 1, dtype).to(DEV), dtype)
        g = torch.Generator().manual_seed(3)
        x = (torch.randn(K, generator=g) * 0.5).to(dtype).to(DEV)
        res = torch.randn(N, generator=g).to(dtype).to(DEV)
        y0, y1 = torch.empty(N, dtype=dtype, device=DEV), torch.empty(N, dtype=dtype, device=DEV)
        ops.gemv(x, deq, y0, residual=res)
        ops.gemv_nf4(x, p, y1, residual=res)
        assert _same(y0, y1) and y0.float().abs().sum() > 0
        nw = (1 + 0.1 * torch.randn(K, generator=g)).to(dtype).to(DEV)
        a0, a1 = torch.empty(N // 2, dtype=dtype, device=DEV), torch.empty(N // 2, dtype=dtype, device=DEV)
        ops.gemv(x, deq, a0, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
        ops.gemv_nf4(x, p, a1, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
        assert _same(a0, a1)


@pytest.mark.parametrize("dtype", DTYPES)
def test_qkv_rope_mode_and_kv_pages_are_bit_identical(ops, dtype):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, K, page = 32, 8, 128, 4096, 16
    N = (nh + 2 * nkv) * hd
    with ops.elem_dtype(dtype):
        p, deq = _quantized(ops, matrix(N, K, 7, dtype).to(DEV), dtype)
        cos, sin = build_rope_tables(LlamaDims(), 512, DEV, dtype)
        x = torch.randn(K, generator=torch.Generator().manual_seed(8)).to(dtype).to(DEV)
        nw = torch.ones(K, dtype=dtype, device=DEV)
        pos = torch.tensor([300], dtype=torch.int32, device=DEV)
        pt = torch.arange(40, dtype=torch.int32, device=DEV).flip(0).contiguous()
        outs = []
        for nf4 in (False, True):
            pages = torch.zeros(40, 2, page, nkv, hd, dtype=dtype, device=DEV)
            y = torch.empty(nh * hd, dtype=dtype, device=DEV)
            kw = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, cos_tab=cos, sin_tab=sin, pos=pos,
                      kv_pages=pages, page_table=pt, page_size=page)
            (ops.gemv_nf4(x, p, y, **kw) if nf4 else ops.gemv(x, deq, y, **kw))
            outs.append((y, pages))
        assert _same(outs[0][0], outs[1][0]) and _same(outs[0][1], outs[1][1])
        assert outs[0][1].float().abs().sum() > 0


def _llm_state_dict(d, seed):
    g = torch.Generator().manual_seed(seed)
    H, I, hd = d.hidden_size, d.intermediate_size, d.head_dim
    rn = lambda *s, std=0.02: torch.randn(*s, generator=g) * std  # noqa: E731
    sd = {"model.embed_tokens.weight": rn(d.vocab_size, H, std=0.3), "model.norm.weight": 1 + rn(H, std=0.05), "lm_head.weight": rn(d.vocab_size, H, std=0.08)}
    for l in range(d.num_hidden_layers):
        p = f"model.layers.{l}."
        sd.update({p + "input_layernorm.weight": 1 + rn(H, std=0.05), p + "post_attention_layernorm.weight": 1 + rn(H, std=0.05),
                   p + "self_attn.q_proj.weight": rn(d.num_attention_heads * hd, H), p + "self_attn.k_proj.weight": rn(d.num_key_value_heads * hd, H),
                   p + "self_attn.v_proj.weight": rn(d.num_key_value_heads * hd, H), p + "self_attn.o_proj.weight": rn(H, d.num_attention_heads * hd),
                   p + "mlp.gate_proj.weight": rn(I, H), p + "mlp.up_proj.weight": rn(I, H), p + "mlp.down_proj.weight": rn(H, I)})
    return sd


def _quantized_llama(d, dtype, seed=11):
    from spatialrgpt_b200.weights import LlamaW, _nf4_layer
    sd = _llm_state_dict(d, seed)
    g = lambda dd, k: dd[k].to(device=DEV, dtype=dtype)  # noqa: E731
    return LlamaW(embed=g(sd, "model.embed_tokens.weight").contiguous(), norm=g(sd, "model.norm.weight"), lm_head=g(sd, "lm_head.weight").contiguous(),
                  layers=[_nf4_layer(sd, f"model.layers.{l}.", g, dtype) for l in range(d.num_hidden_layers)], quantization="nf4")


@pytest.mark.parametrize("dtype", DTYPES)
def test_graph_decode_with_nf4_matches_the_plain_step(monkeypatch, dtype):
    from spatialrgpt_b200 import logits_processors
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    d = dataclasses.replace(LlamaDims(), hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16, num_key_value_heads=4,
                            head_dim=128, vocab_size=32003)
    w = _quantized_llama(d, dtype)
    decs = {}
    for knob in ("1", "0"):
        monkeypatch.setenv("SRGPT_DECODE_NF4", knob)
        decs[knob] = LlamaDecoder(d, w, max_seq_len=512)
    on, off = decs["1"], decs["0"]
    assert on._nf4_array is not None and set(on.decode_quant.values()) == {"nf4"} and len(on.decode_quant) == 16
    assert off._nf4_array is None and off.decode_quant == {}
    if dtype == torch.bfloat16:
        assert on.decode_pack == {"lm_head": "packed"}
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(24, 2048, generator=g) * 0.3).to(dtype).to(DEV)
    follow = (torch.randn(9, 2048, generator=g) * 0.3).to(dtype).to(DEV)
    lookup = torch.randint(0, 32003, (24,), generator=g)
    proc = logits_processors.resolve_min_length(logits_processors.parse(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5,
                                                                        eos_token_id=2), 24)
    res = {}
    for knob, dec in decs.items():
        r = [dec.generate_from_embeds(x, 40)]
        r += list(dec.generate_from_embeds(x, 40, use_graph=False, return_logits=True))
        r.append(dec.generate_from_embeds(x, 40, sampling=dict(temperature=0.8, top_p=0.9, seed=7)))
        r.append(dec.generate_from_embeds(x, 40, processors=proc))
        r.append(dec.generate_from_embeds(x, 40, lookup_ids=torch.cat([lookup, r[0][:10].cpu()]), lookup_k=4))
        r.append(dec.generate_from_embeds(x, 12))
        r.append(dec.generate_from_embeds(torch.cat([x, follow]), 20, reuse_rows=24))
        res[knob] = r
    for a, b in zip(res["1"], res["0"]):
        assert torch.equal(a, b)
    assert res["1"][0].numel() == 40 and torch.equal(res["1"][0], res["1"][1])


def _dequantized_llm(sd_llm, elem):
    out = dict(sd_llm)
    for k, v in sd_llm.items():
        if k.endswith(("q_proj.weight", "k_proj.weight", "v_proj.weight", "o_proj.weight", "gate_proj.weight", "up_proj.weight", "down_proj.weight")):
            out[k] = torch.from_numpy(R.quantize_all(v.float().numpy(), elem)[2])
    return out


def _build(case_kw, sd, dtype, quantization):
    from spatialrgpt_b200 import LlavaConfig, LlamaDims, VisionConfig
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    from spatialrgpt_b200.weights import from_state_dicts
    oc = O.OracleConfig(**case_kw)
    cfg = LlavaConfig(
        vision=VisionConfig(image_size=oc.image_size, patch_size=oc.patch_size, hidden_size=oc.v_hidden, num_hidden_layers=oc.v_layers,
                            num_attention_heads=oc.v_heads, intermediate_size=oc.v_inter, layer_norm_eps=oc.v_eps),
        llama=LlamaDims(hidden_size=oc.hidden, num_hidden_layers=oc.layers, num_attention_heads=oc.heads, num_key_value_heads=oc.kv_heads,
                        head_dim=oc.head_dim, intermediate_size=oc.inter, vocab_size=oc.vocab, rope_theta=oc.rope_theta, rms_norm_eps=oc.rms_eps),
        enable_region=oc.enable_region, enable_depth=oc.enable_depth, mm_vision_select_layer=oc.select_layer)
    cfg.llm_mask_token_id, cfg.llm_depth_token_id = oc.mask_token_id, oc.depth_token_id
    return oc, LlavaLlamaModel(cfg, from_state_dicts(cfg, sd, DEV, dtype=dtype, quantization=quantization), max_seq_len=512)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(CASES))
def test_generate_matches_the_oracle_on_the_dequantized_weights(dtype, name):
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    if name == "tiny_nodepth" and dtype == torch.float16:
        pytest.skip("the unquantized fp16 model's inputs_embeds already hold NaN on this fixture's weights (no quantization involved)")
    oc0 = O.OracleConfig(**kw)
    sd = O.make_weights(oc0, seed=3, dtype=dtype)
    oc, mq = _build(kw, sd, dtype, "nf4")
    _, mp = _build(kw, sd, dtype, None)
    assert all(v.startswith("K = ") for v in mq.llm.decode_quant.values()) and len(mq.llm.decode_quant) == 4 * oc.layers
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    depths = depths if depth_on else None
    args = (input_ids.to(DEV), None, None, None, None, images.to(DEV), [m.to(DEV) for m in masks], None if depths is None else depths.to(DEV))
    eq, ep = mq.prepare_inputs_labels_for_multimodal(*args)[4], mp.prepare_inputs_labels_for_multimodal(*args)[4]
    assert _same(eq, ep)  # everything up to inputs_embeds is unquantized
    ids, logits = mq.generate(input_ids.to(DEV), images=args[5], depths=args[7], masks=args[6], do_sample=False, max_new_tokens=n_new,
                              output_logits=True)
    ids2 = mq.generate(input_ids.to(DEV), images=args[5], depths=args[7], masks=args[6], do_sample=False, max_new_tokens=n_new)
    assert torch.equal(ids, ids2)
    enc = O.encode_multimodal(oc, sd, images, depths, masks)
    emb = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), input_ids, enc["image_features"], enc["mask_embeds"],
                              enc["depth_embeds"])[0]
    ref, rlg = O.greedy_generate(oc, _dequantized_llm(sd["llm"], ELEM[dtype]), emb, n_new, return_logits=True)
    got = ids[0].cpu()
    agree = int((got == ref).long().cumprod(0).sum())
    rows = min(agree + 1, n_new)  # logits row k follows ids[:k]
    lg = logits[0][:rows].cpu()
    sigma = float(rlg.std())
    assert (lg - rlg[:rows]).abs().max().item() <= 0.06 * sigma
    noise = float((lg - rlg[:rows]).pow(2).mean().sqrt())
    top2 = rlg.topk(2, -1).values
    safe = int(((top2[:, 0] - top2[:, 1]) > 4 * noise).long().cumprod(0).sum())
    assert safe >= 1 and agree >= min(safe, n_new)


def test_loader_and_the_paths_that_keep_raising(tmp_path):
    from spatialrgpt_b200 import builder
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    from tests.util import write_synthetic_checkpoint
    oc = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    root = str(tmp_path / "SpatialRGPT-tiny")
    write_synthetic_checkpoint(root, oc, O.make_weights(oc, seed=3), generation_eos=[2])
    tok, model, _, _ = builder.load_pretrained_model(root, "SpatialRGPT-tiny", None, quantization="nf4")
    assert model.dtype == torch.float16 and model.weights.llama.quantization == "nf4"
    assert len(model.llm.decode_quant) == 4 * oc.layers
    ids = model.generate(torch.tensor([[1, 20, 30, 40]], device=DEV), max_new_tokens=6)
    assert ids.shape == (1, 6)
    with pytest.raises(NotImplementedError):
        model.to(dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        builder.load_pretrained_model(root, "SpatialRGPT-tiny", None, load_4bit=True)
    with pytest.raises(NotImplementedError):
        TPLlamaDecoder(model.config.llama, model.weights.llama, 0, 2)
    d = dataclasses.replace(LlamaDims(), hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1,
                            head_dim=128, vocab_size=64)
    with pytest.raises(NotImplementedError):  # in_features % 64
        _quantized_llama(dataclasses.replace(d, intermediate_size=520), torch.bfloat16)
