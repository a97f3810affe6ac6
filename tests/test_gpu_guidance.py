"""Classifier-free guidance on the H100: the guidance kernel against torch's fp32 log_softmax and the three-op combine, guided generate()
against the CPU oracle's guidance (tests/guidance_oracle.py) over plain, 12-bit packed and NF4 decode weights, and the bit identities of
the guided rows step: each prompt of a batch equals its guided call alone, graph replay equals eager, the conditional row is the one-token
arithmetic, guidance_scale=1 is plain generate(), and a draw is srgpt_sample_rows on the guided row."""
import pytest
import torch

from oracle import srgpt_oracle as O
from tests.guidance_oracle import argmax_rule, combine, guided_generate

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
V = 128259  # odd: rows b * V start off every 16-byte boundary


# ---- the kernel ----------------------------------------------------------------------------------------------------------------------
def _rows(P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2 * P, V, generator=g) * 4.0
    x[0, 5] = x[0, 77] = x[0].max() + 1.0  # a tie in the conditional row
    if P > 1:
        x[1, ::7] = float("-inf")  # -inf entries
        x[P + 1, 3::11] = float("-inf")
    if P > 2:
        x[2] *= 1e30  # huge magnitudes
        x[P + 2] *= 1e20
    if P > 3:
        x[P + 3] = x[3]  # identical rows: the guided row is the log-probs themselves, with their ties
        x[3, 100] = x[3, 900] = x[3].max() + 2.0
        x[P + 3, 100] = x[P + 3, 900] = x[3, 100]
    return x


@pytest.mark.parametrize("elem", ["bf16", "f16"])
@pytest.mark.parametrize("P,scale", [(1, 1.5), (2, 0.5), (3, 3.0), (4, -1.0), (4, 7.25)])
def test_guidance_kernel_against_torch(elem, P, scale):
    from spatialrgpt_b200 import _lib, ops
    prev = _lib.set_elem(elem)
    try:
        x = _rows(P, 10 * P + int(scale * 4)).to(DEV)
        g = torch.tensor([scale], dtype=torch.float32, device=DEV)
        guided = torch.full((P, V), 7.0, device=DEV)
        lse = torch.zeros(2 * P, 2, device=DEV)
        ids = torch.full((2 * P,), -5, dtype=torch.int64, device=DEV)
        ops.guidance_rows(x, g, guided, lse=lse, ids=ids)
        guided2 = torch.empty_like(guided)
        ops.guidance_rows(x, g, guided2)
        torch.cuda.synchronize()
    finally:
        _lib.set_elem(prev)
    assert torch.equal(guided.view(torch.int32), guided2.view(torch.int32))  # fixed reduction order; ids or not, the same rows
    xc = x.cpu().double()
    m = xc.max(-1).values
    ref_l = (xc - m[:, None]).exp().sum(-1).log()
    assert torch.equal(lse[:, 0].cpu(), x.cpu().max(-1).values)
    # the fp32 sum of exp over 128 K columns: within 64 ulp of the exact sum, i.e. 64 eps in log space
    assert torch.allclose(lse[:, 1].cpu().double(), ref_l, rtol=0, atol=64 * 2.0 ** -23), (lse[:, 1].cpu().double() - ref_l).abs().max()
    # the combine, bit for bit, given the kernel's own log-probs (x - m) - L in torch's fp32 ops
    lp = (x.cpu() - lse[:, :1].cpu()) - lse[:, 1:].cpu()
    want = combine(lp[:P], lp[P:], scale)
    got = guided.cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(got.nan_to_num(), want.nan_to_num())
    # against torch's own log_softmax: a few ulp
    ls = torch.log_softmax(x, -1).cpu()
    ref = combine(ls[:P], ls[P:], scale)
    fin = torch.isfinite(ref)
    assert torch.equal(fin, torch.isfinite(got))
    # a few ulp of the operands: the log-probs' sums are reduced in another order than torch's
    tol = 16 * torch.finfo(torch.float32).eps * (abs(scale) * (ls[:P].abs() + ls[P:].abs()) + ls[P:].abs() + ref.abs())
    assert bool(((got - ref).abs()[fin] <= tol[fin]).all()), ((got - ref).abs()[fin] - tol[fin]).max()
    for b in range(P):
        assert int(ids[b]) == int(ids[P + b]) == argmax_rule(got[b]), b
    if P > 3:
        assert int(ids[3]) == 100


# ---- guided generate() against the oracle --------------------------------------------------------------------------------------------
def _build(dtype, quantization=None, seed=3):
    from tests.golden.make_golden import CASES
    from tests.test_gpu_nf4 import _build as build_q
    kw = CASES["tiny_masks_gqa"][0]
    sd = O.make_weights(O.OracleConfig(**kw), seed=seed, dtype=dtype)
    oc, model = build_q(kw, sd, dtype, quantization)
    return oc, sd, model


def _text(oc, B, T, seed):
    return torch.randint(3, oc.vocab - 3, (B, T), generator=torch.Generator().manual_seed(seed))


FORMATS = [(torch.bfloat16, "plain"), (torch.bfloat16, "nf4"), (torch.float16, "plain"), (torch.float16, "nf4")]


@pytest.mark.parametrize("dtype,fmt", FORMATS)
@pytest.mark.parametrize("scale", [0.5, 3.0])
def test_guided_generate_matches_the_oracle(dtype, fmt, scale):
    """Ids agree up to the first step whose guided top-1 / top-2 margin the element type's noise could flip, as test_gpu_nf4.py's rule;
    the raw conditional logits stay within 0.06 sigma up to there.  NF4: the oracle runs the dequantized weights.  (The fixture's widths
    are too small for the 12-bit packing and the NF4 planes; test_packed_and_nf4_planes_equal_plain covers those streams.)"""
    from tests.test_gpu_nf4 import ELEM, _dequantized_llm
    oc, sd, model = _build(dtype, "nf4" if fmt == "nf4" else None)
    w = _dequantized_llm(sd["llm"], ELEM[dtype]) if fmt == "nf4" else sd["llm"]
    n_new = 10
    ids, neg = _text(oc, 2, 20, 1), _text(oc, 2, 9, 2)
    got, lg = model.generate(ids.to(DEV), guidance_scale=scale, negative_prompt_ids=neg.to(DEV), max_new_tokens=n_new, eos_token_id=None,
                             output_logits=True)
    emb = w["model.embed_tokens.weight"].float()
    for b in range(2):
        ref, raw, rows = guided_generate(oc, w, emb[ids[b]], neg[b], scale, n_new)
        g = got[b].cpu()
        agree = int((g == ref).long().cumprod(0).sum())
        k = min(agree + 1, n_new)
        err = (lg[b][:k].cpu() - raw[:k]).abs()
        sigma = float(raw.std())
        assert float(err.max()) <= 0.06 * sigma
        noise = float(err.pow(2).mean().sqrt())
        top2 = rows.topk(2, -1).values
        safe = int(((top2[:, 0] - top2[:, 1]) > 4 * max(1.0, scale) * 2 * noise).long().cumprod(0).sum())
        assert agree >= min(safe, n_new), (b, agree, safe)


# ---- bit identities ------------------------------------------------------------------------------------------------------------------
def _same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_equal_their_guided_call_alone_and_graph_equals_eager(dtype):
    """Five multimodal prompts (groups of 4 and 1) with padded negative prompts: row b equals prompt b's guided call alone, ids and
    output_logits; the captured step equals the eager one."""
    from tests.golden.make_golden import CASES
    oc, _, model = _build(dtype)
    _, n_regions, t_text, kind, _, _ = CASES["tiny_masks_gqa"]
    reqs = [O.synth_request(oc, n_regions, t_text, seed=s, kind=kind) for s in (1234, 77, 5, 9, 31)]
    h = lambda t: t.to(DEV, dtype)  # noqa: E731
    B, T = len(reqs), max(r[0].shape[1] for r in reqs)
    ids = torch.zeros(B, T, dtype=torch.int64)
    mask = torch.zeros(B, T, dtype=torch.int64)
    for b, r in enumerate(reqs):
        ids[b, :r[0].shape[1]] = r[0][0]
        mask[b, :r[0].shape[1]] = 1
    neg = _text(oc, B, 12, 4)
    nmask = torch.ones_like(neg)
    for b in range(B):
        nmask[b, :b] = 0  # left padding of b tokens
    args = dict(images=h(torch.cat([r[1] for r in reqs])), depths=h(torch.cat([r[2] for r in reqs])), masks=[h(m) for r in reqs for m in r[3]])
    kw = dict(max_new_tokens=12, eos_token_id=None, guidance_scale=2.5)
    got, lg = model.generate(ids.to(DEV), attention_mask=mask.to(DEV), negative_prompt_ids=neg.to(DEV), negative_prompt_attention_mask=nmask.to(DEV),
                             output_logits=True, **args, **kw)
    graph = model.generate(ids.to(DEV), attention_mask=mask.to(DEV), negative_prompt_ids=neg.to(DEV), negative_prompt_attention_mask=nmask.to(DEV),
                           **args, **kw)
    assert torch.equal(got, graph)
    for b, r in enumerate(reqs):
        one, l1 = model.generate(r[0].to(DEV), images=h(r[1]), depths=h(r[2]), masks=[h(m) for m in r[3]], negative_prompt_ids=neg[b:b + 1, b:].to(DEV),
                                 output_logits=True, **kw)
        assert got[b].tolist() == one[0].tolist(), b
        assert _same(lg[b], l1[0]), b


def test_packed_and_nf4_planes_equal_plain(monkeypatch):
    """The guided rows step streams every weight format of the rows step: at Llama-3-8B widths the 12-bit packed step (bf16) equals the
    plain one, and the NF4 planes equal their dequantized copies, ids and logits bit for bit; three prompts equal each alone."""
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_beam_batch import _dims
    from tests.test_gpu_batch_invariant import _prompts
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    from tests.test_gpu_packed_decode import _decoder
    kw = dict(guidance_scale=2.0, return_logits=True)

    def run(dec, P, N):
        three = dec.generate_rows(P, 10, negative_embeds=N, **kw)
        for b in range(3):
            one = dec.generate_rows(P[b:b + 1], 10, negative_embeds=N[b:b + 1], **kw)
            assert three[0][b].tolist() == one[0][0].tolist() and _same(three[1][b], one[1][0]), b
        assert [o.tolist() for o in dec.generate_rows(P, 10, negative_embeds=N, guidance_scale=2.0)] == [o.tolist() for o in three[0]]
        return three

    got = {}
    for pack in (True, False):
        dec = _decoder(monkeypatch, pack, layers=2)
        assert ("packed" in dec.decode_pack.values()) == pack
        H = dec.dims.hidden_size
        got[pack] = run(dec, _prompts([37, 5, 120], H, torch.bfloat16, 3), _prompts([9, 64, 3], H, torch.bfloat16, 4))
        del dec
    assert [o.tolist() for o in got[True][0]] == [o.tolist() for o in got[False][0]]
    assert all(_same(a, b) for a, b in zip(got[True][1], got[False][1]))
    d = _dims()
    sd = _llm_state_dict(d, 21)
    for dtype in DTYPES:
        P, N = _prompts([131, 150, 9], d.hidden_size, dtype, 5), _prompts([20, 7, 33], d.hidden_size, dtype, 6)
        nf = {}
        for copy in (True, False):
            dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512)
            nf[copy] = run(dec, P, N)
            del dec
        assert [o.tolist() for o in nf[True][0]] == [o.tolist() for o in nf[False][0]]
        assert all(_same(a, b) for a, b in zip(nf[True][1], nf[False][1]))


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_near_one_keeps_the_one_token_logits_and_scale_one_is_plain(dtype):
    from spatialrgpt_b200 import ops
    oc, _, model = _build(dtype)
    ids, neg = _text(oc, 2, 16, 7).to(DEV), _text(oc, 2, 6, 8).to(DEV)
    kw = dict(max_new_tokens=10, eos_token_id=None, output_logits=True)
    plain, pl = model.generate(ids, **kw)
    plain_rows = [model.generate(ids[b:b + 1], **kw) for b in range(2)]
    near, nl = model.generate(ids, guidance_scale=1.0 + 2 ** -20, negative_prompt_ids=neg, **kw)
    for b in range(2):
        one, l1 = plain_rows[b]
        n = int((near[b].cpu() == one[0].cpu()).long().cumprod(0).sum())
        assert n >= 1
        assert _same(nl[b][:n], l1[0][:n]), b  # the conditional row is the batch-1 one-token step's, bit for bit
    model.generate(ids, max_new_tokens=10, eos_token_id=None)  # captures the plain graphs
    before = ops.LAUNCHES
    p1 = model.generate(ids, max_new_tokens=10, eos_token_id=None)
    plain_launches = ops.LAUNCHES - before
    before = ops.LAUNCHES
    g1 = model.generate(ids, max_new_tokens=10, eos_token_id=None, guidance_scale=1.0, negative_prompt_ids=neg)
    assert ops.LAUNCHES - before == plain_launches and torch.equal(g1, p1) and torch.equal(p1, plain)


@pytest.mark.parametrize("dtype", DTYPES)
def test_sampled_guidance_reproduces_and_draws_from_the_guided_row(dtype):
    from spatialrgpt_b200 import _lib, ops
    oc, _, model = _build(dtype)
    ids, neg = _text(oc, 3, 14, 11).to(DEV), _text(oc, 3, 5, 12).to(DEV)
    kw = dict(max_new_tokens=9, eos_token_id=None, guidance_scale=1.8, negative_prompt_ids=neg, do_sample=True, temperature=0.9, top_p=0.95,
              top_k=40, seed=[5, 6, 7])
    a = model.generate(ids, **kw)
    one = model.generate(ids[1:2], **dict(kw, negative_prompt_ids=neg[1:2], seed=6))
    assert torch.equal(one[0], a[1])
    assert torch.equal(a, model.generate(ids, use_cuda_graph=False, **kw)) and torch.equal(a, model.generate(ids, **kw))
    # every draw: a call with a budget of n tokens leaves the guided rows of its last choice (token n - 1) and the counter it drew at;
    # srgpt_sample_rows on those rows, at that counter, with the prompts' seeds, draws token n - 1 again
    dec, P, N = model.llm, [model.llm.embed_tokens(ids[b]) for b in range(3)], [model.llm.embed_tokens(neg[b]) for b in range(3)]
    smp = dict(temperature=0.9, top_p=0.95, top_k=40)
    ids_re = torch.empty(3, dtype=torch.int64, device=DEV)
    prev = _lib.set_elem("bf16" if dtype == torch.bfloat16 else "f16")
    try:
        for n in range(1, 10):
            r = dec.generate_rows(P, n, sampling=smp, seeds=[5, 6, 7], guidance_scale=1.8, negative_embeds=N)
            assert [o.tolist() for o in r] == a[:, :n].tolist(), n
            st = dec._rstate
            ops.sample_rows(st["guided"][:3], dec.sample_params, st["seeds"][:3], (st["step"] - 1).clone(), 0, ids_re)
            assert ids_re.tolist() == a[:, n - 1].tolist(), n
    finally:
        _lib.set_elem(prev)


def test_refusals_on_the_device_model():
    """Beams and FP8 layers (a model built with quantization='fp8') raise, through generate() and through the decoder itself."""
    oc, _, model = _build(torch.bfloat16)
    ids, neg = _text(oc, 2, 8, 1).to(DEV), _text(oc, 2, 4, 2).to(DEV)
    with pytest.raises(NotImplementedError, match="beam"):
        model.generate(ids, guidance_scale=2.0, negative_prompt_ids=neg, num_beams=2, max_new_tokens=4)
    with pytest.raises(ValueError, match="1 .. 4 prompts"):  # the decoder itself: at most SPEC_T_MAX / 2 guided prompts per step
        model.llm.generate_rows([model.llm.embed_tokens(ids[0])] * 5, 4, guidance_scale=2.0, negative_embeds=[model.llm.embed_tokens(neg[0])] * 5)
    del model
    _, _, fp8 = _build(torch.bfloat16, "fp8")
    assert fp8.llm.fp8
    with pytest.raises(NotImplementedError, match="fp8"):
        fp8.generate(ids, guidance_scale=2.0, negative_prompt_ids=neg, max_new_tokens=4)
    with pytest.raises(NotImplementedError, match="FP8"):
        fp8.llm.generate_rows([fp8.llm.embed_tokens(ids[0])], 4, guidance_scale=2.0, negative_embeds=[fp8.llm.embed_tokens(neg[0])])
