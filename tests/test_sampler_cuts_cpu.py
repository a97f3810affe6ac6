"""The sampler's top-k and top-p selection rule without a GPU: a torch restatement of sample_row's key search (csrc/sampling.cu) against
transformers' TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper on the row families where a cut on the probability value
goes wrong: confident rows (the k-th probability below p_max * 2^-26, or exactly 0 in fp32), blocks of tokens straddling k, near-ties
at the k-th value, masked rows and 16-bit rows with many ties.  tests/test_gpu_sampler_cuts.py runs the same families on the kernels."""
import numpy as np
import pytest
import torch

INF = float("inf")
VS = (1000, 32000, 32002, 128256, 128259)
TS = (1.0, 0.7, 0.2, 0.05)
KS = (0, 1, 2, 50, 1000)
PS = (1.0, 0.95, 0.5)
GAPS = (10, 17, 19, 25, 40, 120)  # scaled gaps (nats): across the 26-halving resolution (18.02) and fp32 exp underflow (~104)
SIGMAS = (0.1, 0.5, 1.0)
THREADS = 1024  # sample_row's CTA: thread t walks the chunk [t * per, (t + 1) * per), per = ceil(V / 1024)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- row families ---------------------------------------------------------------------------------------------------------------
def confident(V, sigma, gap, T, seed=0):
    """One token ``gap`` scaled nats (gap * T raw) above an N(0, sigma) tail."""
    g = _gen(seed)
    x = torch.randn(V, generator=g) * sigma
    x[int(torch.randint(V, (1,), generator=g))] = float(x.max()) + gap * T
    return x


def straddled(V, n, T, seed=0):
    """``n`` tokens 25-29 scaled nats above an N(0, 1) tail."""
    g = _gen(seed)
    x = torch.randn(V, generator=g)
    x[torch.randperm(V, generator=g)[:n]] = float(x.max()) + T * (25 + 4 * torch.rand(n, generator=g))
    return x


def near_tie(V, k, ulps, seed=0):
    """The (k+1)-th largest logit ``ulps`` fp32 ulps below the k-th."""
    g = _gen(seed)
    x = torch.randn(V, generator=g)
    o = torch.argsort(x, descending=True)
    y = x[o[k - 1]].clone()
    for _ in range(ulps):
        y = torch.nextafter(y, torch.tensor(-INF))
    x[o[k]] = y
    return x


def div_tie(V, k, T, seed=0):
    """Distinct k-th and (k+1)-th logits with equal fl(x / T) (HF keeps both); None at T = 1, where no two logits share x / T."""
    if T == 1.0:
        return None
    g = _gen(seed)
    x = torch.randn(V, generator=g) * 0.3  # below 1.6
    v = torch.tensor(1.9)  # x / T lands in a binade with a coarser ulp than x's at every T < 1 of TS, so fl(x / T) has collisions
    while True:
        w = torch.nextafter(v, torch.tensor(-INF))
        if bool(w / T == v / T):
            break
        v = w
    idx = torch.randperm(V, generator=g)[:k + 1]
    x[idx[:k - 1]] = 2.0 + torch.rand(k - 1, generator=g)
    x[idx[k - 1]], x[idx[k]] = v, w
    return x


def chunk_ends(V):
    """The last index of each non-empty 1024-thread chunk of sample_row (every third token where a chunk holds one token)."""
    per = -(-V // THREADS)
    if per == 1:
        return torch.arange(2, V, 3)
    return torch.arange(per - 1, V + per - 1, per).clamp(max=V - 1).unique()


def masked(V, finite=None, seed=0):
    """-inf where the logits processors write it (bad words, n-gram bans, EOS below the minimum length): 5 % of the tokens and the
    last token of every 1024-thread chunk, so a chunk's walk ends on a -inf token.  With ``finite``, only that many entries are finite."""
    g = _gen(seed)
    x = torch.randn(V, generator=g) * 2
    x[torch.rand(V, generator=g) < 0.05] = -INF
    ends = chunk_ends(V)
    x[ends] = -INF
    if finite is not None:
        ok = torch.ones(V, dtype=torch.bool)
        ok[ends] = False
        cand = ok.nonzero().flatten()
        keep = cand[torch.randperm(cand.numel(), generator=g)[:finite]]
        y = torch.full((V,), -INF)
        y[keep] = torch.randn(finite, generator=g) * 2
        x = y
    return x


def elem_ties(V, k, dtype, seed=0):
    """A 16-bit row (many exact ties) with 8 more tokens tied at the k-th value."""
    g = _gen(seed)
    x = (torch.randn(V, generator=g) * 2).to(dtype)
    o = torch.argsort(x.float(), descending=True, stable=True)
    x[o[k:k + 8]] = x[o[k - 1]].clone()
    return x


def family_rows(V, T, k, n=32):
    """``n`` fp32 rows of every family at (V, T, k): confident (3 sigma x 6 gaps), straddled blocks of 2/49/50/51/60 tokens, k-th
    near-ties 1-4 ulps apart, a division tie, masked rows (some with fewer than k finite entries), then confident rows of new seeds."""
    kk = k if 0 < k < V - 1 else 50
    rows = [confident(V, s, gp, T, seed=i) for i, (s, gp) in enumerate((s, gp) for s in SIGMAS for gp in GAPS)]
    rows += [straddled(V, b, T, seed=b) for b in (2, 49, 50, 51, 60)]
    rows += [near_tie(V, kk, u, seed=u) for u in (1, 2, 4)]
    d = div_tie(V, kk, T, seed=7)
    rows += [d if d is not None else near_tie(V, kk, 3, seed=3)]
    rows += [masked(V, seed=1), masked(V, finite=max(kk // 2, 1), seed=2), masked(V, finite=3, seed=3)]
    s = 100
    while len(rows) < n:
        rows.append(confident(V, SIGMAS[s % 3], GAPS[s % 6], T, seed=s))
        s += 1
    return torch.stack(rows[:n])


# ---- references -----------------------------------------------------------------------------------------------------------------
def hf_warp(x, T, k, p):
    """transformers' warpers as generate() builds them (TopK only for top_k > 0, TopP only for top_p < 1) over fp32 rows [R, V]."""
    from transformers.generation import logits_process as lp
    s = lp.TemperatureLogitsWarper(T)(None, x.float().clone())
    if k > 0:
        s = lp.TopKLogitsWarper(k)(None, s)
    if p < 1.0:
        s = lp.TopPLogitsWarper(p)(None, s)
    return s


def key(x):
    """sample_row's order-preserving 32-bit key of fp32 values (-0 folded into +0), as int64."""
    b = (x.float() + 0.0).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, ~b & 0xFFFFFFFF, b | (1 << 31))


def unkey(k):
    """The fp32 values of keys [R] (int64)."""
    b = torch.where(k >= 1 << 31, k & 0x7FFFFFFF, ~k & 0xFFFFFFFF)
    return torch.from_numpy(b.numpy().astype(np.uint32).view(np.float32))


def _widen(x, c, T):
    """The smallest logit of each row whose fl(x / T) reaches that of the logit of key c: the cut moved over its ties in x / T."""
    xc = unkey(c)[:, None]
    return torch.where(x / T >= xc / T, x, INF).min(-1, keepdim=True).values


def select(x, T, k, p):
    """The kernel's kept mask over fp32 rows [R, V] (batched; each row's searches run independently): the k-th largest key by a count
    search over the 32 key bits, then the largest key whose mass reaches top_p of the top-k mass by a search over the bits below the
    common prefix of the top-k key and the top key, each cut widened over its ties in fl(x / T).  Masses in fp32, as the kernel."""
    x = x.float()
    R, V = x.shape
    t = torch.tensor(T, dtype=torch.float32)
    inv_t = 1.0 / t.clamp(min=1e-6)
    m = x.max(-1, keepdim=True).values
    e = torch.exp((x - m) * inv_t)
    pr = e * (1.0 / e.sum(-1, keepdim=True))
    kx = key(x)
    x_floor = torch.full((R, 1), -INF)
    mass_floor = torch.ones(R, 1)
    if 0 < k < V:
        c = torch.zeros(R, dtype=torch.int64)
        for b in range(31, -1, -1):
            cand = c | (1 << b)
            c = torch.where((kx >= cand[:, None]).sum(-1) >= k, cand, c)
        x_floor = _widen(x, c, t)
        mass_floor = torch.where(x >= x_floor, pr, 0.0).sum(-1, keepdim=True)
    if p >= 1.0:
        return x >= x_floor
    target = p * mass_floor
    kf, km = key(x_floor)[:, 0], key(m)[:, 0]
    c = kf.clone()
    for r in range(R):
        a, z = int(kf[r]), int(km[r])
        if a == z:
            continue
        hb = (a ^ z).bit_length() - 1
        cr = a & ~((2 << hb) - 1)
        for b in range(hb, -1, -1):
            cand = cr | (1 << b)
            if float(torch.where(kx[r] >= max(cand, a), pr[r], 0.0).sum()) >= float(target[r]):
                cr = cand
        c[r] = min(max(cr, a), z)
    return x >= _widen(x, c, t)


def bisection_topk_keeps(x, T, k):
    """How many tokens the 26-halving bisection on the probability value keeps at top-k (the rule sample_row used before the key
    search), in fp32 as it ran."""
    inv_t = 1.0 / max(T, 1e-6)
    p = torch.exp((x.float() - x.max()) * inv_t)
    p = p / p.sum()
    lo, hi = 0.0, float(p.max())
    for _ in range(26):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if int((p >= mid).sum()) >= k else (lo, mid)
    return int((p >= lo).sum())


def check_topk(got, ref, x, T, where=""):
    """The finite entries of ``got`` (kept masks or warped rows [R, V]) are HF's top-k set exactly."""
    gf = torch.isfinite(got) if got.dtype != torch.bool else got & torch.isfinite(x)
    bad = gf != torch.isfinite(ref)
    assert not bool(bad.any()), (where, bad.sum(-1).nonzero().flatten().tolist(), gf.sum(-1).tolist(), torch.isfinite(ref).sum(-1).tolist())


def check_top_p(gf, x, T, k, p, where=""):
    """Kept masks [R, V] against HF's top-p set: equal, or within DESIGN.md §7's tolerance (top_p moved by a relative 1e-4), or, where
    HF's sort splits tokens of equal score x / T at the nucleus threshold (equal logits, or distinct logits whose fl(x / T) are
    equal), HF's set plus tokens tied at the kept set's lowest score."""
    from tests.test_gpu_warpers import _near_cut
    ref = torch.isfinite(hf_warp(x, T, k, p))
    st = (T, k, p, 1.0, 0.0, 0.0)
    for r in torch.nonzero((gf != ref).any(-1)).flatten().tolist():
        g, s = gf[r], x[r] / T
        if set(s[ref[r]].tolist()) & set(s[~ref[r] & torch.isfinite(x[r])].tolist()):
            assert bool((ref[r] <= g).all()) and bool((s[g & ~ref[r]] == s[g].min()).all()), (where, r)
            continue
        lo, hi = _near_cut(x[r], st)
        assert bool((lo <= g).all() and (g <= hi).all()), (where, r, int(g.sum()), int(ref[r].sum()))


# ---- tests ----------------------------------------------------------------------------------------------------------------------
def test_families_reach_the_regimes_a_probability_bisection_misses():
    V = 128256
    assert bisection_topk_keeps(confident(V, 1.0, 19, 1.0), 1.0, 50) == V  # past 18.02 nats every probe counts < k
    x = confident(V, 0.5, 120, 0.2)
    p = torch.softmax(x / 0.2, -1)
    assert int((p > 0).sum()) == 1 and int(torch.isfinite(hf_warp(x[None], 0.2, 50, 1.0)).sum()) == 50  # exp underflows; HF keeps 50
    d = div_tie(V, 50, 0.2)
    o = torch.argsort(d, descending=True)
    assert d[o[49]] != d[o[50]] and d[o[49]] / 0.2 == d[o[50]] / 0.2
    assert int(torch.isfinite(hf_warp(d[None], 0.2, 50, 1.0)).sum()) == 51
    m = masked(32002, finite=10)
    assert int(torch.isfinite(m).sum()) == 10 and bool(torch.isinf(m[chunk_ends(32002)]).all())
    e = elem_ties(V, 50, torch.bfloat16)
    assert int(torch.isfinite(hf_warp(e.float()[None], 1.0, 50, 1.0)).sum()) >= 58


def test_key_is_order_preserving():
    x = torch.tensor([-INF, -3.5, -1e-30, -0.0, 0.0, 1e-45, 2.0, 3e38, INF])
    k = key(x)
    assert bool((k[1:] >= k[:-1]).all()) and int(k[3]) == int(k[4])
    assert torch.equal(unkey(k), x + 0.0)


@pytest.mark.parametrize("V", [1000, 32002, 128259])
@pytest.mark.parametrize("T", TS)
def test_top_k_rule_is_hf_exactly(V, T):
    for k in (1, 2, 50, 1000):
        x = family_rows(V, T, k)
        check_topk(select(x, T, k, 1.0), hf_warp(x, T, k, 1.0), x, T, (V, T, k))
        if k == 1:
            top = (x / T) == (x / T).max(-1, keepdim=True).values
            assert torch.equal(select(x, T, 1, 1.0), top)


@pytest.mark.parametrize("V", [1000, 128259])
@pytest.mark.parametrize("T", [0.7, 0.05])
def test_top_p_rule_is_hf_within_tolerance(V, T):
    for k in (0, 1, 2, 50, 1000):
        x = family_rows(V, T, k, n=24)
        for p in (0.95, 0.5):
            check_top_p(select(x, T, k, p), x, T, k, p, (V, T, k, p))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_top_k_rule_on_16_bit_rows_with_ties(dtype):
    for V, T, k in ((32000, 1.0, 50), (128256, 0.7, 2), (128259, 0.2, 1000)):
        x = torch.stack([elem_ties(V, k, dtype, seed=s) for s in range(4)]).float()
        check_topk(select(x, T, k, 1.0), hf_warp(x, T, k, 1.0), x, T, (V, T, k))
        check_top_p(select(x, T, k, 0.95), x, T, k, 0.95, (V, T, k))
