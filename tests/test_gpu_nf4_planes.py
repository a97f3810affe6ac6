"""NF4 planes without a dequantized copy (nf4_dequantized_copy=False) on the H100, in both element types.  Every comparison is on the bits:
the NF4 GEMM against the 16-bit GEMM over the dequantized matrix (every epilogue, stream-K and whole-tile, a forced rasterisation group),
the multi-token NF4 GEMV against the element-type one, a 4-layer decoder loaded in copy mode against the same decoder loaded planes-only on
every generation path, the residency of a planes-only load, and the paths that raise."""
import dataclasses
import functools
import os
import subprocess
import sys

import pytest
import torch

from oracle import srgpt_oracle as O
from tests.golden.make_golden import CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def _same(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
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


@functools.lru_cache(maxsize=2)
def _planes(N, K, dtype):
    from spatialrgpt_b200 import ops
    with ops.elem_dtype(dtype):
        codes, scale = ops.nf4_quantize(matrix(N, K, N + K, dtype).to(DEV))
        deq = ops.nf4_dequantize(codes, scale)
        return ops.nf4_planes(codes, scale, deq)[0], deq


MS = [1, 7, 32, 128, 129, 259, 1000, 2100]


def _gemm_cases(ops, N, K, dtype, ms=MS):
    """Every M and epilogue: gemm_nf4 over the planes against gemm over the dequantized matrix."""
    p, deq = _planes(N, K, dtype)
    g = torch.Generator().manual_seed(N * 7 + K)
    with ops.elem_dtype(dtype):
        for M in ms:
            a = (torch.randn(M, K, generator=g) * 0.5).to(dtype).to(DEV)
            res = torch.randn(M, N, generator=g).to(dtype).to(DEV)
            h = (N // 2 + 7) // 8 * 8  # SwiGLU output rows padded to 16 bytes (N / 2 = 500)
            for epi, kw in ((ops.EPI_NONE, {}), (ops.EPI_BIAS_RESIDUAL, {"residual": res}), (ops.EPI_SWIGLU, {})):
                outs = [torch.empty(M, h, dtype=dtype, device=DEV)[:, :N // 2] if epi == ops.EPI_SWIGLU else None for _ in range(2)]
                ref = ops.gemm(a, deq, epilogue=epi, out=outs[0], **kw)
                got = ops.gemm_nf4(a, p, epilogue=epi, out=outs[1], **kw)
                assert _same(ref, got), (M, N, K, epi)
                assert ref.float().abs().sum() > 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [1024, 4096, 14336])
@pytest.mark.parametrize("N", [1000, 4096, 6144])
def test_nf4_gemm_is_bit_identical_to_the_gemm_over_the_dequantized_matrix(ops, N, K, dtype):
    _gemm_cases(ops, N, K, dtype)


def _subprocess_cases():
    """Run in a fresh process: the GEMM reads SRGPT_GEMM_TSK / SRGPT_GEMM_GM once per process."""
    from spatialrgpt_b200 import ops
    for dtype in DTYPES:
        for N, K in ((1000, 4096), (4096, 14336)):
            _gemm_cases(ops, N, K, dtype, ms=[1, 32, 128, 259, 2100])
    torch.cuda.synchronize()
    print("subprocess cases ok")


@pytest.mark.parametrize("env", [{"SRGPT_GEMM_TSK": "-1"}, {"SRGPT_GEMM_GM": "3"}])
def test_nf4_gemm_whole_tile_and_forced_group_order(env):
    code = "import sys; sys.path.insert(0, %r); from tests.test_gpu_nf4_planes import _subprocess_cases; _subprocess_cases()" % ROOT
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env={**os.environ, **env}, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "subprocess cases ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("dtype", DTYPES)
def test_multi_token_nf4_gemv_is_bit_identical_in_every_mode(ops, dtype):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, H, I, page = 16, 4, 128, 2048, 5120, 16
    nqkv = (nh + 2 * nkv) * hd
    pq, dq = _planes(nqkv, H, dtype)
    g = torch.Generator().manual_seed(4)
    with ops.elem_dtype(dtype):
        def planes(N, K, seed):
            codes, scale = ops.nf4_quantize(matrix(N, K, seed, dtype).to(DEV))
            deq = ops.nf4_dequantize(codes, scale)
            return ops.nf4_planes(codes, scale, deq)[0], deq
        pg, dg = planes(2 * I, H, 9)
        pd, dd = planes(H, I, 10)
        cos, sin = build_rope_tables(LlamaDims(), 512, DEV, dtype)
        nw = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(DEV)
        pt = torch.arange(40, dtype=torch.int32, device=DEV).flip(0).contiguous()
        for T in range(1, 9):
            xh = (torch.randn(T, H, generator=g) * 0.5).to(dtype).to(DEV)
            xi = (torch.randn(T, I, generator=g) * 0.5).to(dtype).to(DEV)
            res = torch.randn(T, H, generator=g).to(dtype).to(DEV)
            pos = torch.tensor([200 + T], dtype=torch.int32, device=DEV)
            out = {}
            for nf in (False, True):
                pages = torch.zeros(40, 2, page, nkv, hd, dtype=dtype, device=DEV)
                yq = torch.empty(T, nh * hd, dtype=dtype, device=DEV)
                ya = torch.empty(T, I, dtype=dtype, device=DEV)
                yd = torch.empty(T, H, dtype=dtype, device=DEV)
                kq = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, cos=cos, sin=sin, pos=pos,
                          kv_pages=pages, page_table=pt, page_size=page)
                ka = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
                if nf:
                    ops.gemv_multi_nf4(xh, pq, yq, **kq)
                    ops.gemv_multi_nf4(xh, pg, ya, **ka)
                    ops.gemv_multi_nf4(xi, pd, yd, residual=res)
                else:
                    ops.gemv_multi(xh, dq, yq, **kq)
                    ops.gemv_multi(xh, dg, ya, **ka)
                    ops.gemv_multi(xi, dd, yd, residual=res)
                out[nf] = (yq, ya, yd, pages)
            for a, b in zip(out[False], out[True]):
                assert _same(a, b), T
            assert out[True][3].float().abs().sum() > 0


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


def _llama(d, sd, dtype, copy: bool):
    from spatialrgpt_b200.weights import LlamaW, _nf4_layer
    g = lambda dd, k: dd[k].to(device=DEV, dtype=dtype)  # noqa: E731
    return LlamaW(embed=g(sd, "model.embed_tokens.weight").contiguous(), norm=g(sd, "model.norm.weight"), lm_head=g(sd, "lm_head.weight").contiguous(),
                  layers=[_nf4_layer(sd, f"model.layers.{l}.", g, dtype, dequantized_copy=copy) for l in range(d.num_hidden_layers)],
                  quantization="nf4", nf4_dequantized_copy=copy)


DIMS = dict(hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16, num_key_value_heads=4, head_dim=128, vocab_size=32003)


@pytest.mark.parametrize("dtype", DTYPES)
def test_planes_only_decoder_matches_copy_mode_on_every_path(dtype):
    from spatialrgpt_b200 import logits_processors
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.weights import Nf4W
    d = dataclasses.replace(LlamaDims(), **DIMS)
    sd = _llm_state_dict(d, 21)
    decs = {copy: LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512, max_seqs=4) for copy in (True, False)}
    po = decs[False]
    assert po.nf4_planes_only and not decs[True].nf4_planes_only
    assert all(isinstance(getattr(lw, n + "_w"), Nf4W) for lw in po.w.layers for n in ("qkv", "o", "gateup", "down"))
    assert set(po.decode_quant.values()) == {"nf4"} and po.decode_quant == decs[True].decode_quant
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(24, d.hidden_size, generator=g) * 0.3).to(dtype).to(DEV)
    follow = (torch.randn(9, d.hidden_size, generator=g) * 0.3).to(dtype).to(DEV)
    lookup = torch.randint(0, d.vocab_size, (24,), generator=g)
    lens = [37, 5, 130, 64]
    packed = (torch.randn(sum(lens), d.hidden_size, generator=g) * 0.3).to(dtype).to(DEV)
    proc = logits_processors.resolve_min_length(logits_processors.parse(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5,
                                                                        eos_token_id=2), 24)
    res = {}
    for copy, dec in decs.items():
        r = [dec.generate_from_embeds(x, 40)]
        r += list(dec.generate_from_embeds(x, 40, use_graph=False, return_logits=True))
        r.append(dec.generate_from_embeds(x, 40, sampling=dict(temperature=0.8, top_p=0.9, seed=7)))
        r.append(dec.generate_from_embeds(x, 40, processors=proc))
        r += list(dec.generate_from_embeds(x, 40, lookup_ids=torch.cat([lookup, r[0][:10].cpu()]), lookup_k=4, use_graph=False, return_logits=True))
        r.append(dec.generate_from_embeds(x, 40, lookup_ids=torch.cat([lookup, r[0][:10].cpu()]), lookup_k=4))
        r.append(dec.generate_from_embeds(x, 12))
        r.append(dec.generate_from_embeds(torch.cat([x, follow]), 20, reuse_rows=24))
        eos = [int(r[0][3]), int(r[0][17])]
        r += [t for t in dec.generate_batch(packed, lens, 24, eos_token_ids=eos)]
        r += [t for t in dec.generate_batch(packed, lens, 10, use_graph=False)]
        r.append(dec.generate_beam(x, 3, 16))
        dec.cache.reserve_many(lens)
        r.append(dec.logits_all(dec.prefill_packed(packed, lens)))
        res[copy] = r
    assert len(res[True]) == len(res[False])
    for i, (a, b) in enumerate(zip(res[True], res[False])):
        assert a.shape == b.shape and _same(a, b), i
    assert res[False][0].numel() == 40 and torch.equal(res[False][0], res[False][1])


@pytest.mark.parametrize("dtype", DTYPES)
def test_planes_only_residency_and_load_peak(dtype):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.weights import Nf4W
    d = dataclasses.replace(LlamaDims(), **DIMS)
    sd = _llm_state_dict(d, 22)
    small = dataclasses.replace(d, num_hidden_layers=1)
    _llama(small, _llm_state_dict(small, 23), dtype, copy=False)  # first-use tables of the quantizer stay out of the measurement
    H, I, nqkv = d.hidden_size, d.intermediate_size, (d.num_attention_heads + 2 * d.num_key_value_heads) * d.head_dim
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    w = _llama(d, sd, dtype, copy=False)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - base
    peak = torch.cuda.max_memory_allocated() - base
    planes = norms = 0
    for lw in w.layers:
        for n in ("qkv", "o", "gateup", "down"):
            m = getattr(lw, n + "_w")
            assert isinstance(m, Nf4W) and lw.nf4[n] is m  # no element-type [N, K] tensor is kept
            planes += m.nbytes()
        norms += lw.in_norm.numel() * 2 + lw.post_norm.numel() * 2
    other = sum(t.numel() * t.element_size() for t in (w.embed, w.norm, w.lm_head))
    layer_bytes = sum(t.numel() * t.element_size() for lw in w.layers for t in (lw.in_norm, lw.post_norm)) + planes
    assert layer_bytes == planes + norms
    fused = 2 * (nqkv * H + H * d.num_attention_heads * d.head_dim + 2 * I * H + H * I)  # one layer's fused element-type matrices
    # the caching allocator hands out a large block whole when less than 1 MB would be left over: up to 1 MB of slack per tensor
    slack = (1 << 20) * (10 * d.num_hidden_layers + 3)
    assert planes + norms + other <= grown <= planes + norms + other + slack, (grown, planes + norms + other)
    assert peak <= grown + 2 * fused + slack, (peak, grown, fused)


def _build(case_kw, sd, dtype, copy):
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
    return oc, LlavaLlamaModel(cfg, from_state_dicts(cfg, sd, DEV, dtype=dtype, quantization="nf4", nf4_dequantized_copy=copy), max_seq_len=512)


@pytest.mark.parametrize("dtype", DTYPES)
def test_tiny_fixture_keeps_its_copies_and_matches_copy_mode(dtype):
    kw, n_regions, t_text, kind, n_new, depth_on = CASES["tiny_masks_gqa"]
    sd = O.make_weights(O.OracleConfig(**kw), seed=3, dtype=dtype)
    oc, mc = _build(kw, sd, dtype, True)
    _, mp = _build(kw, sd, dtype, False)
    assert mp.llm.nf4_planes_only and all(v.startswith("K = ") for v in mp.llm.decode_quant.values())
    assert mp.llm.decode_quant == mc.llm.decode_quant and len(mp.llm.decode_quant) == 4 * oc.layers
    assert all(isinstance(lw.qkv_w, torch.Tensor) for lw in mp.weights.llama.layers)
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    args = dict(images=images.to(DEV), depths=depths.to(DEV) if depth_on else None, masks=[m.to(DEV) for m in masks], do_sample=False,
                max_new_tokens=n_new, output_logits=True)
    ic, lc = mc.generate(input_ids.to(DEV), **args)
    ip, lp = mp.generate(input_ids.to(DEV), **args)
    assert torch.equal(ic, ip) and _same(lc, lp)


def test_full_model_loader_planes_only_matches_copy_mode(tmp_path):
    from spatialrgpt_b200 import builder
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    from tests.util import write_synthetic_checkpoint
    kw = dict(CASES["tiny_masks_gqa"][0])
    kw.update(hidden=1024, inter=2048, heads=8, kv_heads=2, head_dim=128)
    oc = O.OracleConfig(**kw)
    root = str(tmp_path / "SpatialRGPT-nf4")
    write_synthetic_checkpoint(root, oc, O.make_weights(oc, seed=3), generation_eos=[2])
    models = {copy: builder.load_pretrained_model(root, "SpatialRGPT-nf4", None, quantization="nf4", nf4_dequantized_copy=copy)[1]
              for copy in (True, False)}
    assert models[False].llm.nf4_planes_only and set(models[False].llm.decode_quant.values()) == {"nf4"}
    ids = torch.tensor([[1, 20, 30, 40, 50, 60, 70]], device=DEV)
    out = {copy: m.generate(ids, do_sample=False, max_new_tokens=12, output_logits=True) for copy, m in models.items()}
    assert torch.equal(out[True][0], out[False][0]) and _same(out[True][1], out[False][1])
    po = models[False]
    with pytest.raises(NotImplementedError):
        po.to(dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        TPLlamaDecoder(po.config.llama, po.weights.llama, 0, 2)
    with pytest.raises(ValueError):
        builder.load_pretrained_model(root, "SpatialRGPT-nf4", None, nf4_dequantized_copy=False)


def test_decode_nf4_off_raises_for_a_planes_only_decoder(monkeypatch):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    d = dataclasses.replace(LlamaDims(), hidden_size=1024, intermediate_size=2048, num_hidden_layers=1, num_attention_heads=8, num_key_value_heads=2,
                            head_dim=128, vocab_size=64)
    w = _llama(d, _llm_state_dict(d, 1), torch.bfloat16, copy=False)
    monkeypatch.setenv("SRGPT_DECODE_NF4", "0")
    with pytest.raises(ValueError, match="SRGPT_DECODE_NF4"):
        LlamaDecoder(d, w, max_seq_len=128)
