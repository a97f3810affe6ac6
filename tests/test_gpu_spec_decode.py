"""Prompt-lookup speculative decoding on the H100: every multi-token kernel against T one-token calls bit for bit, the decoder's verify
loop against plain greedy decoding (ids, logits, stops, counts, untouched pages) with planted drafts, and generate() on the tiny
pipeline fixtures."""
import pytest
import torch

from tests.test_gpu_packed_decode import _decoder, _same, weights
from tests.test_spec_decode_cpu import simulate

pytestmark = pytest.mark.gpu
DEV = "cuda"
T_MAX = 8


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def _x(T, K, seed, scale=0.5):
    return (torch.randn(T, K, generator=torch.Generator().manual_seed(seed)) * scale).to(torch.bfloat16).to(DEV)


# ---- kernels ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("K", [4096, 14336])
def test_plain_and_swiglu_equal_one_token_calls(ops, packed, K):
    N = 1024
    w = weights(N, K, K + 1, n_planted=150)
    p = ops.pack12(w)[0] if packed else None
    assert not packed or p is not None
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(3))).to(torch.bfloat16).to(DEV)
    one = (lambda x, y, **kw: ops.gemv_packed(x, p, y, **kw)) if packed else (lambda x, y, **kw: ops.gemv(x, w, y, **kw))
    for T in range(1, T_MAX + 1):
        x = _x(T, K, T)
        res = _x(T, N, 50 + T)
        y = res.clone()
        ops.gemv_multi(x, w, y, residual=y, packed=p)
        swiglu = K == 4096  # the RMSNorm-fused modes run at the hidden size (the whole row of x is staged per token)
        a = torch.empty(T, N // 2, dtype=torch.bfloat16, device=DEV)
        if swiglu:
            ops.gemv_multi(x, w, a, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU, packed=p)
        for t in range(T):
            yr = torch.empty(N, dtype=torch.bfloat16, device=DEV)
            one(x[t], yr, residual=res[t])
            assert _same(y[t], yr), (T, t)
            if not swiglu:
                continue
            ar = torch.empty(N // 2, dtype=torch.bfloat16, device=DEV)
            one(x[t], ar, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
            assert _same(a[t], ar), (T, t)


@pytest.mark.parametrize("packed", [False, True])
def test_qkv_rope_equals_one_token_calls(ops, packed):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, K, page = 32, 8, 128, 4096, 16
    N = (nh + 2 * nkv) * hd
    w = weights(N, K, 7, n_planted=200)
    p = ops.pack12(w)[0] if packed else None
    cos, sin = build_rope_tables(LlamaDims(), 512, DEV)
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(4))).to(torch.bfloat16).to(DEV)
    pt = torch.randperm(40, generator=torch.Generator().manual_seed(5)).to(torch.int32).to(DEV)
    kw = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, page_table=pt, page_size=page)
    for T in range(1, T_MAX + 1):
        x = _x(T, K, 20 + T, 1.0)
        p0 = 301 - T  # the pass crosses a page boundary for T >= 4
        pm = torch.zeros(40, 2, page, nkv, hd, dtype=torch.bfloat16, device=DEV)
        y = torch.empty(T, nh * hd, dtype=torch.bfloat16, device=DEV)
        ops.gemv_multi(x, w, y, cos=cos, sin=sin, pos=torch.tensor([p0], dtype=torch.int32, device=DEV), kv_pages=pm, packed=p, **kw)
        pr = torch.zeros_like(pm)
        for t in range(T):
            yr = torch.empty(nh * hd, dtype=torch.bfloat16, device=DEV)
            pos = torch.tensor([p0 + t], dtype=torch.int32, device=DEV)
            one_kw = {k: v for k, v in kw.items() if k not in ("page_table", "page_size")}
            if packed:
                ops.gemv_packed(x[t], p, yr, cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pr, page_table=pt, page_size=page, **one_kw)
            else:
                ops.gemv(x[t], w, yr, cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pr, page_table=pt, page_size=page, **one_kw)
            assert _same(y[t], yr), (T, t)
        assert _same(pm, pr) and pm.abs().sum() > 0


@pytest.mark.parametrize("packed", [False, True])
def test_lm_head_logits_and_arg_maxes_equal_one_token_calls(ops, packed):
    V, K = 128259, 4096
    w = weights(V, K, 11, std=0.08, n_planted=500)
    p = ops.pack12(w)[0] if packed else None
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(6))).to(torch.bfloat16).to(DEV)
    ws1 = ops.lm_head_workspace(V, DEV)
    wsT = torch.empty(T_MAX * ws1.numel(), dtype=torch.uint8, device=DEV)
    for T in (1, 2, 5, T_MAX):
        x = _x(T, K, 70 + T, 1.0)
        lg = torch.empty(T, V, dtype=torch.float32, device=DEV)
        ops.lm_head_multi(x, w, nw, 1e-5, wsT, logits_out=lg, packed=p)
        ref_ids = []
        for t in range(T):
            ids = torch.zeros(1, dtype=torch.int64, device=DEV)
            step, pos = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
            lr = torch.empty(V, dtype=torch.float32, device=DEV)
            f = ops.lm_head_argmax_packed if packed else ops.lm_head_argmax
            f(x[t], p if packed else w, nw, 1e-5, ws1, ids, step, pos, logits_out=lr)
            assert torch.equal(lg[t], lr), (T, t)
            ref_ids.append(int(ids[0]))
        # the accept kernel's arg maxes: drafts planted equal to them are all accepted, and out_ids holds the T arg maxes
        draft = torch.tensor([-1] + ref_ids[:-1] + [-1] * (T_MAX - T), dtype=torch.int32, device=DEV)
        out = torch.full((16,), -5, dtype=torch.int64, device=DEV)
        step, pos, state = (torch.tensor([3], dtype=torch.int32, device=DEV), torch.tensor([40], dtype=torch.int32, device=DEV),
                            torch.zeros(8, dtype=torch.int32, device=DEV))
        ops.spec_accept(wsT, V, T, draft, out, step, pos, state)
        assert out[3:3 + T].tolist() == ref_ids and int(step) == 3 + T and int(pos) == 40 + T and int(state[2]) == T - 1
        # a wrong second draft: only the first is accepted
        if T >= 3:
            draft[2] = (ref_ids[1] + 1) % V
            out.fill_(-5); step.fill_(3); pos.fill_(40); state.zero_()
            ops.spec_accept(wsT, V, T, draft, out, step, pos, state)
            assert out[3:6].tolist() == ref_ids[:2] + [-5] and int(step) == 5 and int(state[5]) == 2


@pytest.mark.parametrize("nkv", [8, 32])
@pytest.mark.parametrize("p0", [37, 290])
def test_attention_equals_one_token_calls(ops, nkv, p0):
    nh, hd, page, n_pages = 32, 128, 16, 48
    g = torch.Generator().manual_seed(p0 + nkv)
    pages = torch.randn(n_pages, 2, page, nkv, hd, generator=g).to(torch.bfloat16).to(DEV)
    pt = torch.randperm(n_pages, generator=g).to(torch.int32).to(DEV)
    for T in range(1, T_MAX + 1):
        q = _x(T, nh * hd, 90 + T, 1.0)
        out = torch.empty(T, nh * hd, dtype=torch.bfloat16, device=DEV)
        rows = torch.arange(p0, p0 + T, dtype=torch.int32, device=DEV)
        ops.attention_decode_multi(q, out, pages, pt, page, rows, nh, nkv, hd, hd ** -0.5)
        for t in range(T):
            o = torch.empty(nh * hd, dtype=torch.bfloat16, device=DEV)
            ops.attention_decode(q[t].contiguous(), o, pages, pt, page, rows[t:t + 1].contiguous(), nh, nkv, hd, hd ** -0.5)
            assert _same(out[t], o), (T, t)


# ---- decoder ------------------------------------------------------------------------------------------------------------------
MAX_NEW = 40


def _plans(g):
    """Planted lookup histories: the continuation itself (perfect drafts), ids that never occur (garbage), and the continuation
    with every third id replaced (partly right)."""
    perfect = list(g)
    garbage = [3] * 5
    half = [v if i % 3 else 7 for i, v in enumerate(g)]
    return {"perfect": perfect, "garbage": garbage, "half": half}


@pytest.mark.parametrize("pack", [True, False])
def test_verify_loop_equals_plain_greedy(ops, monkeypatch, pack):
    dec = _decoder(monkeypatch, pack)
    assert (dec._packed_array is not None) == pack
    x = (torch.randn(20, 4096, generator=torch.Generator().manual_seed(5)) * 0.3).to(torch.bfloat16).to(DEV)
    g_long = dec.generate_from_embeds(x, MAX_NEW + 2 * T_MAX).tolist()
    g = torch.tensor(g_long[:MAX_NEW], device=DEV)
    ids_l, lg = dec.generate_from_embeds(x, MAX_NEW, use_graph=False, return_logits=True)
    assert torch.equal(ids_l, g)
    owned_before = set(dec.cache.owned[0])
    snapshot = dec.cache.pages.clone()
    for name, hist in _plans(g_long).items():
        for k in (1, 3, 7, 12):
            for graph in (True, False):
                ids = dec.generate_from_embeds(x, MAX_NEW, use_graph=graph, lookup_ids=torch.tensor(hist), lookup_k=k)
                assert torch.equal(ids, g), (name, k, graph)
                assert dec.last_speculation == simulate(hist, g_long, k, 2, MAX_NEW), (name, k, graph, dec.last_speculation)
        if name == "perfect":
            assert dec.last_speculation[2] > 0
        ids2, lg2 = dec.generate_from_embeds(x, MAX_NEW, use_graph=False, return_logits=True, lookup_ids=torch.tensor(hist), lookup_k=3)
        assert torch.equal(ids2, g) and torch.equal(lg2, lg), name
    # pages of no sequence: bitwise unchanged
    other = [pg for pg in range(dec.cache.n_pages) if pg not in owned_before and pg not in dec.cache.owned[0]]
    assert other and torch.equal(dec.cache.pages[:, other].view(torch.int16), snapshot[:, other].view(torch.int16))
    # stops: EOS inside an accepted run, a stopping criterion, and a budget that is not a multiple of T
    eos = g_long[11]
    first = g_long.index(eos)
    plain_eos = dec.generate_from_embeds(x, MAX_NEW, eos_token_ids=[eos])
    assert plain_eos.numel() == first + 1
    stop_fn = lambda ids: ids.numel() >= 13  # noqa: E731
    plain_stop = dec.generate_from_embeds(x, MAX_NEW, stopping_fn=stop_fn)
    for k in (3, 7):
        for graph in (True, False):
            kw = dict(use_graph=graph, lookup_ids=torch.tensor(g_long), lookup_k=k)
            assert torch.equal(dec.generate_from_embeds(x, MAX_NEW, eos_token_ids=[eos], **kw), plain_eos)
            assert torch.equal(dec.generate_from_embeds(x, MAX_NEW, stopping_fn=stop_fn, **kw), plain_stop)
            r = dec.generate_from_embeds(x, 23, **kw)
            assert torch.equal(r, g[:23])
            assert dec.last_speculation == simulate(g_long, g_long, k, 2, 23)
    # slack that does not fit max_seq_len: the one-token loop, reported as (0, 0, 0)
    r = dec.generate_from_embeds(x, 256 - 20 - 4, lookup_ids=torch.tensor(g_long), lookup_k=3)
    assert dec.last_speculation == (0, 0, 0) and torch.equal(r[:MAX_NEW], g)


# ---- model --------------------------------------------------------------------------------------------------------------------
def test_generate_with_prompt_lookup_equals_generate():
    from tests.test_gpu_prefix_cache import _requests
    oc, model, imgs, deps, turns, masks = _requests("tiny_masks_gqa")
    md = [masks.to(DEV, dtype=model.dtype)]
    args = dict(images=imgs, depths=deps, masks=md, do_sample=False, max_new_tokens=12)
    for ids in turns[:2]:
        ref = model.generate(ids.to(DEV), **args)
        ref_l, ref_lg = model.generate(ids.to(DEV), output_logits=True, **args)
        for k in (1, 4, 10):
            out = model.generate(ids.to(DEV), prompt_lookup_num_tokens=k, **args)
            assert torch.equal(out, ref), k
            assert model.last_speculation[0] > 0
            o2, lg2 = model.generate(ids.to(DEV), prompt_lookup_num_tokens=k, output_logits=True, use_cuda_graph=False, **args)
            assert torch.equal(o2, ref_l) and torch.equal(lg2[0], ref_lg[0])
    # a prefix-cached follow-up with the option equals the one without
    for opt in ({}, {"prompt_lookup_num_tokens": 3}):
        model.generate(turns[0].to(DEV), prefix_cache=True, **args)
        r = model.generate(turns[1].to(DEV), prefix_cache=True, **args, **opt)
        if not opt:
            base = r
    assert torch.equal(r, base)
    # text only
    tids = torch.tensor([[1, 5, 9, 5, 9, 5]], device=DEV)
    assert torch.equal(model.generate(tids, max_new_tokens=10, prompt_lookup_num_tokens=2), model.generate(tids, max_new_tokens=10))
    with pytest.raises(NotImplementedError):
        model.generate(ids.to(DEV), prompt_lookup_num_tokens=3, do_sample=True, temperature=0.5, **{k: v for k, v in args.items() if k != "do_sample"})
    with pytest.raises(NotImplementedError):
        model.generate(ids.to(DEV), prompt_lookup_num_tokens=3, num_beams=2, **args)
    with pytest.raises(NotImplementedError):
        model.generate(torch.cat([tids, tids]), max_new_tokens=4, prompt_lookup_num_tokens=2)
    with pytest.raises(TypeError):
        model.generate(tids, max_new_tokens=4, assistant_model=model)


def test_fp16_model_with_prompt_lookup():
    from tests.test_gpu_prefix_cache import _requests
    oc, model, imgs, deps, turns, masks = _requests("tiny_boxes")
    model.to(dtype=torch.float16)
    md = [masks.to(DEV, dtype=torch.float16)]
    args = dict(images=imgs.half(), depths=None if deps is None else deps.half(), masks=md, do_sample=False, max_new_tokens=10)
    ref = model.generate(turns[0].to(DEV), **args)
    assert torch.equal(model.generate(turns[0].to(DEV), prompt_lookup_num_tokens=4, **args), ref)
