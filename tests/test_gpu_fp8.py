"""FP8 (E4M3) W8A8 quantization on the H100, in both element types: the device quantizers against the CPU restatement (tests/fp8_ref.py)
bit for bit, the FP8 GEMM against an fp64 restatement from the exact codes and scales, the decoder's paths on FP8 weights, generate() on
the tiny fixtures against the fp32 oracle with FP8 linears, and the loader."""
import dataclasses

import pytest
import torch

from oracle import srgpt_oracle as O
from tests import fp8_ref as R
from tests.golden.make_golden import CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
MANT = {torch.bfloat16: 7, torch.float16: 10}
LAYER_LINEARS = ("q_proj.weight", "k_proj.weight", "v_proj.weight", "o_proj.weight", "gate_proj.weight", "up_proj.weight", "down_proj.weight")


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def matrix(N, K, seed, dtype, std=0.02):
    """[N, K] ~ N(0, std) with adversarial rows: all zero; subnormals of the element type beside one normal value; single large outliers;
    and a row whose maximum is 448, so that inv = 1 and the exact E4M3 ties 17, 19, 2^-10 and 3 2^-10 reach the rounding unchanged."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * std
    w[0] = 0
    tiny = torch.finfo(dtype).tiny
    w[1] = 0
    w[1, :7] = torch.tensor([tiny / 2, -tiny / 4, tiny, 0, -tiny / 8, tiny * 3, 0.01])
    w[2, :8] = torch.tensor([448.0, 17.0, 19.0, -17.0, 2.0 ** -10, 3 * 2.0 ** -10, -2.0 ** -10, 464.0 / 2])
    rows = torch.randint(3, N, (6,), generator=g)
    cols = torch.randint(0, K, (6,), generator=g)
    w[rows, cols] = torch.tensor([3.0, -2.5, 1.7, -4.0, 2.2, 6.0])
    return w.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [256, 640, 4096, 14336])
def test_quantizers_match_the_restatement(ops, dtype, K):
    w = matrix(96, K, K, dtype)
    with ops.elem_dtype(dtype):
        q, s = ops.fp8_quantize_weight(w.to(DEV))
        q_ref, s_ref = R.quantize_rows(w)
        assert torch.equal(q.cpu(), q_ref) and torch.equal(s.cpu().view(torch.int32), s_ref.view(torch.int32))
        assert s[0].item() == 1.0 and q[0].abs().sum().item() == 0  # the all-zero row
        assert R.decode(q[2, :4].cpu()).tolist() == [448.0, 16.0, 20.0, -16.0]
        # the activation quantizer: same definition, into a strided code buffer
        x = matrix(33, K, K + 1, dtype).to(DEV)
        qbuf = torch.full((33, K + 32), 0x55, dtype=torch.uint8, device=DEV)
        qa, sa = ops.fp8_quantize_act(x, q=qbuf[:, :K])
        qa_ref, sa_ref = R.quantize_rows(x.cpu())
        assert torch.equal(qa.cpu(), qa_ref) and torch.equal(sa.cpu().view(torch.int32), sa_ref.view(torch.int32))
        assert (qbuf[:, K:] == 0x55).all()


def test_quantizer_rejects_inf_nan_and_odd_widths(ops):
    w = matrix(64, 1024, 1, torch.bfloat16).to(DEV)
    for bad in (float("inf"), float("nan")):
        v = w.clone()
        v[3, 100] = bad
        with pytest.raises(ops.SrgptError, match="Inf or NaN"):
            ops.fp8_quantize_weight(v, name="model.layers.3.self_attn.o_proj.weight")
    with pytest.raises(NotImplementedError, match="has 1000"):
        ops.fp8_quantize_weight(torch.zeros(8, 1000, dtype=torch.bfloat16, device=DEV))


def _ulp(v: torch.Tensor, dtype) -> torch.Tensor:
    """The element type's unit in the last place at |v| (fp32 tensor), its subnormal step below the normal range."""
    a = v.abs().to(dtype).float().clamp_min(torch.finfo(dtype).tiny)
    return torch.ldexp(torch.ones_like(a), torch.frexp(a).exponent - 1 - MANT[dtype])


# (M, N, K, epilogue): M = 1, 32, 128 take stream-K (N K >= 4 MB), 259 and 8288 whole tiles; N = 1040 and 2 x 520 are not multiples of 128
GEMM_CASES = [(1, 1040, 4096, 0), (32, 1040, 4096, 0), (128, 1040, 4096, 0), (259, 1040, 4096, 0), (8288, 1040, 4096, 0),
              (1, 1040, 4096, 4), (259, 1040, 4096, 4), (8288, 1040, 4096, 4), (1, 1040, 4096, 5), (128, 1040, 4096, 5), (259, 1040, 4096, 5),
              (1, 1040, 14336, 4), (128, 1040, 14336, 4), (259, 1040, 14336, 4), (33, 272, 256, 0), (33, 272, 384, 4), (33, 1280, 512, 5),
              (259, 1040, 640, 4)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K,epi", GEMM_CASES)
def test_gemm_matches_the_fp64_restatement(ops, dtype, M, N, K, epi):
    """Each output within 1 ulp of the element type of the restatement from the exact codes and scales (acc summed exactly in fp64), once
    the tensor cores' summation bound (fp8_ref.linear_q) is allowed for; the epilogue's rounding points (residual add, SwiGLU) are restated alike."""
    from spatialrgpt_b200.weights import Fp8W
    g = torch.Generator().manual_seed(M * 7 + K + epi)
    with ops.elem_dtype(dtype):
        w = Fp8W(*ops.fp8_quantize_weight((torch.randn(N, K, generator=g) * 0.02).to(dtype).to(DEV)))
        x = (torch.randn(M, K, generator=g)).to(dtype).to(DEV)
        qx, sx = ops.fp8_quantize_act(x)
        y, bound = R.linear_q(qx, sx, w.q, w.scale)
        tol_y = _ulp(y, dtype) + bound
        if epi == ops.EPI_NONE:
            got = ops.gemm_fp8(qx, sx, w).float()
            assert ((got - y).abs() <= tol_y).all(), float(((got - y).abs() / tol_y).max())
        elif epi == ops.EPI_BIAS_RESIDUAL:
            res = torch.randn(M, N, generator=g).to(dtype).to(DEV)
            got = ops.gemm_fp8(qx, sx, w, residual=res, epilogue=epi).float()
            ref = (y.to(dtype).float() + res.float()).to(dtype).float()
            tol = tol_y + _ulp(ref, dtype)
            assert ((got - ref).abs() <= tol).all(), float(((got - ref).abs() / tol).max())
        else:
            got = ops.gemm_fp8(qx, sx, w, epilogue=epi).float()
            gate, up = y[:, 0::2].to(dtype).float(), y[:, 1::2].to(dtype).float()
            act = torch.nn.functional.silu(gate).to(dtype).float()
            ref = (act * up).to(dtype).float()
            # first-order propagation of the gate / up tolerances through silu (slope <= 1.1) and the product
            tol = _ulp(ref, dtype) + 1.1 * up.abs() * (tol_y[:, 0::2] + _ulp(gate, dtype)) + act.abs() * tol_y[:, 1::2] + _ulp(act, dtype) * up.abs()
            assert ((got - ref).abs() <= tol).all(), float(((got - ref).abs() / tol).max())
        assert got.abs().sum() > 0
        # the elementwise bound grows with K * sum |products|; the rms error must stay at the element type's rounding level whatever K
        # (one missing stream-K partial of 7 k-blocks would be about 0.25 of the output's rms)
        y_ref = ref if epi != ops.EPI_NONE else y
        assert float((got - y_ref).pow(2).mean().sqrt()) <= 2.0 ** -7 * float(y_ref.pow(2).mean().sqrt())


def _integer_operands(M, N, K, seed, dtype):
    """x [M, K] with values in {0, +-1, +-2, +-4} (its row maximum 4: every x * 448 / 4 is an exact E4M3 value) and FP8 weights with
    8 non-zero codes per row in {+-1, +-2, +-4} and scale 1: every partial sum is a small multiple of the products, exact in any order
    and at any accumulator precision, so the result must equal the restatement bit for bit."""
    from spatialrgpt_b200.weights import Fp8W
    g = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, 1.0, -1.0, 2.0, -2.0, 4.0, -4.0])
    x = vals[torch.randint(0, 7, (M, K), generator=g)]
    x[:, 0] = 4.0
    w = torch.zeros(N, K)
    for r in range(N):
        w[r, torch.randperm(K, generator=g)[:8]] = vals[1 + torch.randint(0, 6, (8,), generator=g)]
    return x.to(dtype).to(DEV), Fp8W(q=R.e4m3(w).to(DEV), scale=torch.ones(N, device=DEV))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemm_and_gemv_are_exact_where_the_sum_is(ops, dtype):
    """Exact sums: the whole-tile GEMM (M = 259), the stream-K GEMM (M = 1 and 128, N K >= 4 MB) and the FP8 GEMV equal the restatement
    fl32(acc) * fl32(s_x * s_w), rounded to the element type, bit for bit."""
    N, K = 1040, 4096
    with ops.elem_dtype(dtype):
        for M in (1, 128, 259):
            x, w = _integer_operands(M, N, K, M, dtype)
            qx, sx = ops.fp8_quantize_act(x)
            y, _ = R.linear_q(qx, sx, w.q, w.scale)
            assert torch.equal(ops.gemm_fp8(qx, sx, w), y.to(dtype)), M
            if M == 1:
                out = torch.empty(N, dtype=dtype, device=DEV)
                assert torch.equal(ops.gemv_fp8(x[0], w, out), y[0].to(dtype))


def _gemv_case(ops, N, K, seed, dtype):
    from spatialrgpt_b200.weights import Fp8W
    g = torch.Generator().manual_seed(seed)
    w = Fp8W(*ops.fp8_quantize_weight((torch.randn(N, K, generator=g) * 0.02).to(dtype).to(DEV)))
    x = torch.randn(K, generator=g).to(dtype).to(DEV)
    return g, w, x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N,K", [(4096, 4096), (28672, 4096), (4096, 14336), (6144, 4096), (1040, 256), (768, 640)])
def test_gemv_plain_and_swiglu_match_the_restatement_and_the_gemm(ops, dtype, N, K):
    """PLAIN (+ residual) and SWIGLU without the RMSNorm prologue against the restatement from the activation quantizer's exact codes,
    within 1 ulp once the fp32 summation bound is allowed for; the GEMV and the M = 1 GEMM within 1 ulp of each other likewise."""
    with ops.elem_dtype(dtype):
        g, w, x = _gemv_case(ops, N, K, N + K, dtype)
        qx, sx = ops.fp8_quantize_act(x[None])
        y, bound = R.linear_q(qx, sx, w.q, w.scale)
        y, bound = y[0], bound[0]
        tol = _ulp(y, dtype) + bound
        res = torch.randn(N, generator=g).to(dtype).to(DEV)
        got = ops.gemv_fp8(x, w, torch.empty(N, dtype=dtype, device=DEV), residual=res).float()
        ref = (y.to(dtype).float() + res.float()).to(dtype).float()
        assert ((got - ref).abs() <= tol + _ulp(ref, dtype)).all()
        plain = ops.gemv_fp8(x, w, torch.empty(N, dtype=dtype, device=DEV)).float()
        assert ((plain - y).abs() <= tol).all()
        gemm = ops.gemm_fp8(qx, sx, w)[0].float()
        assert ((plain - gemm).abs() <= _ulp(gemm, dtype) + 2 * bound).all()
        act = ops.gemv_fp8(x, w, torch.empty(N // 2, dtype=dtype, device=DEV), mode=ops.GEMV_SWIGLU).float()
        gate, up = y[0::2].to(dtype).float(), y[1::2].to(dtype).float()
        a = torch.nn.functional.silu(gate).to(dtype).float()
        ref = (a * up).to(dtype).float()
        tol = _ulp(ref, dtype) + 1.1 * up.abs() * (tol[0::2] + _ulp(gate, dtype)) + a.abs() * tol[1::2] + _ulp(a, dtype) * up.abs()
        assert ((act - ref).abs() <= tol).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemv_qkv_rope_mode_and_its_kv_pages_match_the_restatement(ops, dtype):
    """QKV + RoPE + KV append: q and the K/V rows written to the pages against the restatement (RoPE as the rope kernel rounds it,
    applied by the bf16 path's own rope_kv_append to the restated projection), within 1 ulp of the rotated values plus the propagated
    summation bound."""
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, K, page = 32, 8, 128, 4096, 16
    N = (nh + 2 * nkv) * hd
    with ops.elem_dtype(dtype):
        g, w, x = _gemv_case(ops, N, K, 7, dtype)
        cos, sin = build_rope_tables(LlamaDims(), 512, DEV, dtype)
        pos = torch.tensor([300], dtype=torch.int32, device=DEV)
        pt = torch.arange(40, dtype=torch.int32, device=DEV).flip(0).contiguous()
        pages = torch.zeros(40, 2, page, nkv, hd, dtype=dtype, device=DEV)
        q = torch.empty(nh * hd, dtype=dtype, device=DEV)
        ops.gemv_fp8(x, w, q, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pages,
                     page_table=pt, page_size=page)
        qx, sx = ops.fp8_quantize_act(x[None])
        y, bound = R.linear_q(qx, sx, w.q, w.scale)
        qkv = y.to(dtype).contiguous()
        ref_pages = torch.zeros_like(pages)
        ops.rope_kv_append(qkv, nh, nkv, hd, cos, sin, pos, ref_pages, pt, page)
        tol_y = (_ulp(y, dtype) + bound)[0]
        # a rotated value mixes two projections with |cos|, |sin| <= 1, each rounded: 1 ulp of each input plus 2 ulp of the output
        pair = tol_y.view(-1, 2, hd // 2).flip(1).reshape(-1)
        ref_q = qkv[0, :nh * hd].float()
        assert ((q.float() - ref_q).abs() <= tol_y[:nh * hd] + pair[:nh * hd] + 2 * _ulp(ref_q, dtype)).all()
        slot = pages[pt[300 // page], :, 300 % page].float().reshape(-1)
        ref_slot = ref_pages[pt[300 // page], :, 300 % page].float().reshape(-1)
        tk = (tol_y + pair)[nh * hd:]
        assert ((slot - ref_slot).abs() <= tk + 2 * _ulp(ref_slot, dtype)).all() and slot.abs().sum() > 0
        assert int((pages != 0).sum()) == int((slot != 0).sum())  # one position written, nothing else


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemv_rmsnorm_prologue(ops, dtype):
    """With norm_weight the GEMV quantizes its own RMSNorm output.  The restatement from rmsnorm() may differ where one ulp of a normed
    element moves its E4M3 code, so the check is on the rms: at the level of the element type's rounding, not of a missing term."""
    N, K = 4096, 4096
    with ops.elem_dtype(dtype):
        g, w, x = _gemv_case(ops, N, K, 3, dtype)
        nw = (1 + 0.1 * torch.randn(K, generator=g)).to(dtype).to(DEV)
        got = ops.gemv_fp8(x, w, torch.empty(N, dtype=dtype, device=DEV), norm_weight=nw, eps=1e-5).float()
        xn = ops.rmsnorm(x[None], nw, 1e-5)
        y = R.linear(xn, w.q, w.scale)[0]
        assert float((got - y).pow(2).mean().sqrt()) <= 2.0 ** -6 * float(y.pow(2).mean().sqrt())


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


def _fp8_llama(d, dtype, seed=11):
    from spatialrgpt_b200.weights import LlamaW, _fp8_layer
    sd = _llm_state_dict(d, seed)
    g = lambda dd, k: dd[k].to(device=DEV, dtype=dtype)  # noqa: E731
    return LlamaW(embed=g(sd, "model.embed_tokens.weight").contiguous(), norm=g(sd, "model.norm.weight"), lm_head=g(sd, "lm_head.weight").contiguous(),
                  layers=[_fp8_layer(sd, f"model.layers.{l}.", g, dtype) for l in range(d.num_hidden_layers)], quantization="fp8")


@pytest.mark.parametrize("dtype", DTYPES)
def test_decoder_paths_on_fp8_weights(dtype):
    from spatialrgpt_b200 import logits_processors
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.weights import Fp8W
    d = dataclasses.replace(LlamaDims(), hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16, num_key_value_heads=4,
                            head_dim=128, vocab_size=32003)
    w = _fp8_llama(d, dtype)
    assert all(isinstance(getattr(lw, n + "_w"), Fp8W) for lw in w.layers for n in ("qkv", "o", "gateup", "down"))
    dec = LlamaDecoder(d, w, max_seq_len=512, max_seqs=2)
    assert set(dec.decode_quant.values()) == {"fp8"} and len(dec.decode_quant) == 16
    assert dec.kernels_per_decode_step == 5 * 4 + 2 and not dec.supports_prompt_lookup
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(24, 2048, generator=g) * 0.3).to(dtype).to(DEV)
    follow = (torch.randn(9, 2048, generator=g) * 0.3).to(dtype).to(DEV)
    n = 40
    ids = dec.generate_from_embeds(x, n)  # graph replay
    ids_eager = dec.generate_from_embeds(x, n, use_graph=False)
    ids_lg, lg = dec.generate_from_embeds(x, n, use_graph=False, return_logits=True)
    assert ids.numel() == n and torch.equal(ids, ids_eager) and torch.equal(ids, ids_lg)
    # The step's logits (FP8 GEMVs) against the prefill path (quantizer + FP8 GEMMs) over the same tokens (prompt + the first n - 1
    # generated ids).  Both quantize each activation row by one definition, but the decode and prefill attention and RMSNorm kernels round
    # differently, and an activation moved by one ulp of the element type across an E4M3 rounding boundary changes its code by an eighth
    # of its value.  Over 16 linears that makes the two paths differ by about 0.08 sigma rms (measured on H100: 0.089 bf16, 0.082 fp16;
    # max 0.44 sigma).  The bound catches a wrong step (a misplaced KV row or a missing scale moves the logits by
    # about sigma), not the rounding.
    full = torch.cat([x, dec.embed_tokens(ids[:-1])])
    ref = dec.logits_all(dec.prefill_hidden(full))[23:23 + n]
    sigma = float(ref.std())
    diff = (lg - ref).abs()
    print(f"fp8 decode-step vs prefill logits ({dtype}): max {float(diff.max()) / sigma:.4f} sigma, rms {float(diff.pow(2).mean().sqrt()) / sigma:.4f} sigma")
    assert float(diff.max()) <= 0.8 * sigma and float(diff.pow(2).mean().sqrt()) <= 0.15 * sigma
    # sampling, logits processors and prefix reuse run on the FP8 step
    proc = logits_processors.resolve_min_length(logits_processors.parse(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5,
                                                                        eos_token_id=2), 24)
    s1 = dec.generate_from_embeds(x, n, sampling=dict(temperature=0.8, top_p=0.9, seed=7))
    assert torch.equal(s1, dec.generate_from_embeds(x, n, sampling=dict(temperature=0.8, top_p=0.9, seed=7)))
    p1 = dec.generate_from_embeds(x, n, processors=proc)
    assert p1.numel() == n and 2 not in p1[:4].tolist()
    dec.generate_from_embeds(x, 12)
    r = dec.generate_from_embeds(torch.cat([x, follow]), 20, reuse_rows=24)
    assert r.numel() == 20
    with pytest.raises(NotImplementedError, match="FP8"):
        dec.generate_from_embeds(x, n, lookup_ids=torch.zeros(4, dtype=torch.int64), lookup_k=3)
    # batched greedy decode (graph and eager agree), batched processors and beam search
    packed = torch.cat([x, follow])
    b = dec.generate_batch(packed, [24, 9], 16)
    assert [t.numel() for t in b] == [16, 16]
    assert all(torch.equal(u, v) for u, v in zip(b, dec.generate_batch(packed, [24, 9], 16, use_graph=False)))
    bp = dec.generate_batch(packed, [24, 9], 16, processors=proc)
    assert [t.numel() for t in bp] == [16, 16]
    beam = dec.generate_beam(x, 3, 10)
    assert 1 <= beam.numel() <= 10


def _fp8_linear_shim(table, linear):
    """F.linear for the oracle: the decoder-layer weights named in `table` (by identity) run as the W8A8 linear of tests/fp8_ref.py."""
    def shim(x, weight, bias=None):
        entry = table.get(id(weight))
        if entry is None:
            return linear(x, weight, bias)
        y = R.linear(x.reshape(-1, x.shape[-1]), *entry)
        return y.reshape(*x.shape[:-1], y.shape[-1]).to(x.dtype)
    return shim


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
def test_generate_matches_the_fp8_oracle(monkeypatch, dtype, name):
    """The agreement rule of the NF4 parity test against the fp32 oracle whose decoder-layer linears are W8A8, and, on the rows compared,
    rms(GPU - FP8 oracle) <= r rms(FP8 oracle - unquantized oracle): the GPU implements this scheme, not merely something near it.
    r = 1/2 in fp16.  In bf16 the ratio measured 0.496 .. 0.539 on H100 (fp16: 0.28 .. 0.40): the oracle quantizes fp32 activations, the
    GPU the bf16-rounded ones, and bf16's coarser rounding flips more E4M3 codes; r = 0.6 there.  The 4-noise margin rule may find no
    token safely decided (FP8 noise is larger than NF4's); the agreement is then asserted only as far as the rule finds, and the ratio decides."""
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    if name == "tiny_nodepth" and dtype == torch.float16:
        pytest.skip("the unquantized fp16 model's inputs_embeds already hold NaN on this fixture's weights (no quantization involved)")
    sd = O.make_weights(O.OracleConfig(**kw), seed=3, dtype=dtype)
    oc, mq = _build(kw, sd, dtype, "fp8")
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    depths = depths if depth_on else None
    ids, logits = mq.generate(input_ids.to(DEV), images=images.to(DEV), depths=None if depths is None else depths.to(DEV),
                              masks=[m.to(DEV) for m in masks], do_sample=False, max_new_tokens=n_new, output_logits=True)
    enc = O.encode_multimodal(oc, sd, images, depths, masks)
    emb = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), input_ids, enc["image_features"], enc["mask_embeds"],
                              enc["depth_embeds"])[0]
    w32 = {k: v.float() for k, v in sd["llm"].items()}  # fp32 already: the oracle's .to(float32) hands these very tensors to F.linear
    table = {id(w32[k]): R.quantize_rows(sd["llm"][k]) for k in w32 if k.endswith(LAYER_LINEARS)}
    with monkeypatch.context() as m:
        m.setattr(O.F, "linear", _fp8_linear_shim(table, O.F.linear))
        ref, rlg = O.greedy_generate(oc, w32, emb, n_new, return_logits=True)
    got = ids[0].cpu()
    agree = int((got == ref).long().cumprod(0).sum())
    rows = min(agree + 1, n_new)  # logits row k follows ids[:k]
    lg = logits[0][:rows].cpu()
    sigma = float(rlg.std())
    noise = float((lg - rlg[:rows]).pow(2).mean().sqrt())
    top2 = rlg.topk(2, -1).values
    safe = int(((top2[:, 0] - top2[:, 1]) > 4 * noise).long().cumprod(0).sum())
    # the unquantized oracle over the same tokens (teacher-forced on the FP8 oracle's ids)
    full = torch.cat([emb, w32["model.embed_tokens.weight"][ref[:rows - 1]]]) if rows > 1 else emb
    plain = O.llama_forward(oc, w32, full, None)[0][emb.shape[0] - 1:emb.shape[0] - 1 + rows]
    quant_effect = float((rlg[:rows] - plain).pow(2).mean().sqrt())
    print(f"{name} {dtype}: agree {agree}/{n_new}, safe {safe}, max|gpu - fp8 oracle| = {float((lg - rlg[:rows]).abs().max()) / sigma:.4f} sigma, "
          f"rms(gpu - fp8 oracle) = {noise:.3e}, rms(fp8 oracle - oracle) = {quant_effect:.3e}, ratio {noise / quant_effect:.3f}")
    assert (lg - rlg[:rows]).abs().max().item() <= 0.1 * sigma
    assert agree >= min(safe, n_new)
    assert noise <= (0.6 if dtype == torch.bfloat16 else 0.5) * quant_effect


def test_loader_holds_only_the_fp8_planes_and_the_paths_that_raise(tmp_path):
    from spatialrgpt_b200 import builder
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    from tests.util import write_synthetic_checkpoint
    oc = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    root = str(tmp_path / "SpatialRGPT-tiny")
    write_synthetic_checkpoint(root, oc, O.make_weights(oc, seed=3), generation_eos=[2])
    tok, model, _, _ = builder.load_pretrained_model(root, "SpatialRGPT-tiny", None, quantization="fp8")
    assert model.dtype == torch.float16 and model.weights.llama.quantization == "fp8"
    H, I, qkv_rows = oc.hidden, oc.inter, (oc.heads + 2 * oc.kv_heads) * oc.head_dim
    shapes = [(qkv_rows, H), (H, oc.heads * oc.head_dim), (2 * I, H), (H, I)]
    expect = oc.layers * (sum(N * K + 4 * N for N, K in shapes) + 2 * H * 2)  # + the two fp16 norms
    held = 0
    for lw in model.weights.llama.layers:
        for f in dataclasses.fields(lw):
            v = getattr(lw, f.name)
            for t in ([v.q, v.scale] if hasattr(v, "q") else [v] if isinstance(v, torch.Tensor) else []):
                assert t.is_cuda
                held += t.numel() * t.element_size()
    assert held == expect
    ids = model.generate(torch.tensor([[1, 20, 30, 40]], device=DEV), max_new_tokens=6)
    assert ids.shape == (1, 6)
    with pytest.raises(NotImplementedError, match="fp8"):
        model.generate(torch.tensor([[1, 20, 30, 40]], device=DEV), max_new_tokens=6, prompt_lookup_num_tokens=3)
    with pytest.raises(NotImplementedError):
        model.to(dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        builder.load_pretrained_model(root, "SpatialRGPT-tiny", None, load_8bit=True)
    with pytest.raises(NotImplementedError):
        TPLlamaDecoder(model.config.llama, model.weights.llama, 0, 2)
