"""Exact checkers for attention over long paged contexts, and proof that they can fail.

The GPU tests in test_gpu_attention_context.py judge the attention kernels with three checks whose expected outputs are exact:
  * row census: q = 0, so every visible row has weight exactly 1.  Position j carries a random class c(j) and
    V[j, h, c(j)] = 1 + h (0 elsewhere), so channel ch of a head on kv head h must be (1 + h) * n_ch / L, where n_ch counts the
    visible rows of class ch.  No class holds more than 64 rows, so one dropped, doubled or foreign row moves its channel by more
    than two bf16 ulps; the 1 + h factor exposes a query head read against the wrong kv head.
  * needles: one row whose score exceeds every other by at least 40 nats; the output must be that row's V, bit for bit.
  * causal census: row r of a chunk at start s sees exactly positions [0, s + r].
Here the checkers run against numpy attention with planted bugs (a dropped row, a doubled row, a swapped page, a causal mask off by
one, a query head on the neighbouring kv head), each of which must be rejected, and against a correct one, which must pass.  The
numpy code keeps the kernels' arithmetic: fp32 running sums and one fp32 division (decode) or a product with 1 / l (prefill)."""
import numpy as np
import pytest
import torch

HD, PAGE = 128, 16
NEEDLE_POS = (0, 1, 15, 16, 31, 32, 255, 256, 257, 511, 2047)  # plus L - 2 and L - 1 (needle_positions)
MANT = {torch.bfloat16: 7, torch.float16: 10}
MIN_EXP = {torch.bfloat16: -126, torch.float16: -14}


# ---- construction ------------------------------------------------------------------------------------------------------------
def random_classes(L: int, n_classes: int, rng: np.random.Generator) -> np.ndarray:
    """A random class per position, every class used at most ceil(L / n_classes) times (and so in every prefix too)."""
    reps = -(-L // n_classes)
    return rng.permutation(np.tile(np.arange(n_classes), reps))[:L]


def census_values(cls: np.ndarray, n_kv: int, hd: int) -> np.ndarray:
    """V [L, n_kv, hd] float32: V[j, h, cls[j]] = 1 + h, 0 elsewhere."""
    v = np.zeros((cls.size, n_kv, hd), np.float32)
    v[np.arange(cls.size), :, cls] = 1.0 + np.arange(n_kv, dtype=np.float32)
    return v


def prefix_counts(cls: np.ndarray, hd: int, lens) -> np.ndarray:
    """counts[r, ch] = number of positions j < lens[r] with class ch."""
    cum = np.zeros((cls.size + 1, hd), np.int64)
    cum[1:] = np.cumsum(np.eye(hd, dtype=np.int64)[cls], axis=0)
    return cum[np.asarray(lens)]


def census_expected(counts: np.ndarray, lens, kv_of_head, dtype) -> torch.Tensor:
    """[R, n_heads, hd] in the element type: elem(float32((1 + kv) * n) / float32(L)), the decode kernels' exact result."""
    scale = 1.0 + np.asarray(kv_of_head, np.float32)
    a = (scale[None, :, None] * counts[:, None, :].astype(np.float32)).astype(np.float32)
    return torch.from_numpy(a / np.asarray(lens, np.float32)[:, None, None]).to(dtype)


def needle_positions(L: int):
    return sorted({j for j in NEEDLE_POS if j < L} | {j for j in (L - 2, L - 1) if j >= 0})


# ---- checks ------------------------------------------------------------------------------------------------------------------
def ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of the element type at |x| (float64)."""
    a = x.double().abs()
    e = torch.floor(torch.log2(torch.where(a > 0, a, torch.ones_like(a)))).clamp_min(MIN_EXP[dtype])
    return torch.pow(2.0, e - MANT[dtype])


def _first_bad(bad: torch.Tensor, out, want, what):
    idx = tuple(int(i) for i in bad.nonzero()[0])
    n = int(bad.sum())
    raise AssertionError(f"{what}: {n} of {bad.numel()} elements wrong, first at {idx}: got {float(out[idx])!r}, want {float(want[idx])!r}")


def assert_bits(out: torch.Tensor, want: torch.Tensor, what: str):
    """Bit-equal (NaN anywhere fails)."""
    out, want = out.cpu(), want.cpu().to(out.dtype).reshape(out.shape)
    bad = out.view(torch.int16) != want.view(torch.int16)
    if bool(bad.any()):
        _first_bad(bad, out, want, what)


def assert_within_ulp(out: torch.Tensor, want: torch.Tensor, dtype, what: str, floor: float = 0.0):
    """|out - want| <= one ulp of the element type at want (+ floor); NaN fails."""
    out, want = out.cpu().double(), want.cpu().double().reshape(out.shape)
    bad = ~((out - want).abs() <= ulp(want, dtype) + floor)
    if bool(bad.any()):
        _first_bad(bad, out, want, what)


# ---- numpy attention with planted bugs ---------------------------------------------------------------------------------------
BUGS = ["drop_row_256", "row_0_twice", "page_swapped", "causal_off_by_one", "neighbour_kv_head"]


def np_attention(q, pages, pt, rows_visible, group, dtype, bug=None, prefill=False):
    """q [R, nh, hd] float32; pages [P, 2, PAGE, nkv, hd] float32; rows_visible[r] = number of visible positions of query r.
    fp32 online-free softmax (scores, max, exp, sums in float32), then sum / l (decode) or sum * (1 / l) (prefill)."""
    R, nh, hd = q.shape
    nkv = pages.shape[3]
    out = np.zeros((R, nh, hd), np.float32)
    for r in range(R):
        n = int(rows_visible[r]) + (1 if bug == "causal_off_by_one" and prefill else 0)
        pos = np.arange(n)
        if bug == "drop_row_256":
            pos = pos[pos != 256]
        if bug == "row_0_twice":
            pos = np.concatenate([[0], pos])
        lp = pos // PAGE
        if bug == "page_swapped":
            lp = np.where(lp == 1, 2, lp)  # logical page 1 read from logical page 2's physical page
        phys = pt[lp]
        for h in range(nh):
            kvh = h // group
            if bug == "neighbour_kv_head":
                kvh = (kvh + 1) % nkv
            k = pages[phys, 0, pos % PAGE, kvh]
            v = pages[phys, 1, pos % PAGE, kvh]
            s = (k @ q[r, h]).astype(np.float32) * np.float32(hd ** -0.5)
            p = np.exp(s - s.max()).astype(np.float32)
            acc = (p[:, None] * v).sum(0, dtype=np.float32)
            l = p.sum(dtype=np.float32)
            out[r, h] = acc * (np.float32(1) / l) if prefill else acc / l
    return torch.from_numpy(out).to(dtype)


def paged(kv_rows: np.ndarray, rng):
    """kv_rows [L, 2, nkv, hd] -> (pages over a random permutation of physical pages with NaN spare pages, page table)."""
    L = kv_rows.shape[0]
    n_lp = -(-L // PAGE)
    n_phys = n_lp + 3
    pt = rng.permutation(n_phys)[:n_lp]
    pages = np.full((n_phys, 2, PAGE) + kv_rows.shape[2:], np.nan, np.float32)
    pad = np.zeros((n_lp * PAGE,) + kv_rows.shape[1:], np.float32)
    pad[:L] = kv_rows
    pages[pt] = pad.reshape(n_lp, PAGE, 2, *kv_rows.shape[2:]).transpose(0, 2, 1, 3, 4)
    return pages, pt


def decode_census_case(L, nh, nkv, rng):
    cls = random_classes(L, HD, rng)
    k = rng.standard_normal((L, nkv, HD)).astype(np.float32)
    pages, pt = paged(np.stack([k, census_values(cls, nkv, HD)], 1), rng)
    return pages, pt, cls


def needle_case(L, nh, nkv, where, rng, dtype):
    """q shared by the heads of a kv head; small random scores; kv head h plants its needle at where[h] (score + >= 40 nats)."""
    grp = nh // nkv
    qv = rng.standard_normal((nkv, HD)).astype(np.float32)
    k = (rng.standard_normal((L, nkv, HD)) * 0.05).astype(np.float32)
    v = rng.integers(1, 9, (L, nkv, HD)).astype(np.float32) * rng.choice([-1, 1], (L, nkv, HD))
    for h in range(nkv):
        k[where[h], h] = qv[h] * (45.0 / (float(qv[h] @ qv[h]) * HD ** -0.5))
    k = torch.from_numpy(k).to(dtype).float().numpy()
    q = torch.from_numpy(np.repeat(qv, grp, 0)).to(dtype).float().numpy()
    s = np.einsum("lhd,hd->lh", k.astype(np.float64), q[::grp].astype(np.float64)) * HD ** -0.5
    for h in range(nkv):  # the premise of the check: the needle leads by 40 nats, every other score is small
        others = np.delete(s[:, h], where[h])
        assert s[where[h], h] - others.max() >= 40 and np.abs(others).max() <= 1
    pages, pt = paged(np.stack([k, v], 1), rng)
    return q, pages, pt, v


# ---- the checkers against the numpy implementations -------------------------------------------------------------------------
def run_decode_census(bug, dtype, L=4096, nh=8, nkv=2, seed=0):
    rng = np.random.default_rng(seed)
    pages, pt, cls = decode_census_case(L, nh, nkv, rng)
    out = np_attention(np.zeros((1, nh, HD), np.float32), pages, pt, [L], nh // nkv, dtype, bug)
    want = census_expected(prefix_counts(cls, HD, [L]), [L], np.arange(nh) // (nh // nkv), dtype)
    assert_bits(out, want, f"census {bug}")


def run_decode_needles(bug, dtype, L=600, nh=4, nkv=2, seed=1):
    rng = np.random.default_rng(seed)
    js = needle_positions(L)
    for i in range(len(js)):
        where = [js[(i + h) % len(js)] for h in range(nkv)]
        q, pages, pt, v = needle_case(L, nh, nkv, where, rng, dtype)
        out = np_attention(q[None], pages, pt, [L], nh // nkv, dtype, bug)
        want = torch.from_numpy(np.stack([v[where[h // (nh // nkv)], h // (nh // nkv)] for h in range(nh)]))[None]
        assert_bits(out, want, f"needles {where} {bug}")


def run_causal_census(bug, dtype, start=250, n=40, nh=4, nkv=2, seed=2):
    rng = np.random.default_rng(seed)
    L = start + n
    pages, pt, cls = decode_census_case(L, nh, nkv, rng)
    vis = [start + r + 1 for r in range(n)]
    out = np_attention(np.zeros((n, nh, HD), np.float32), pages, pt, vis, nh // nkv, dtype, bug, prefill=True)
    want = census_expected(prefix_counts(cls, HD, vis), vis, np.arange(nh) // (nh // nkv), dtype)
    assert_within_ulp(out, want, dtype, f"causal census {bug}")


DTYPES = [torch.bfloat16, torch.float16]


@pytest.mark.parametrize("dtype", DTYPES)
def test_checkers_accept_a_correct_implementation(dtype):
    run_decode_census(None, dtype)
    run_decode_needles(None, dtype)
    run_causal_census(None, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bug", BUGS)
def test_checkers_reject_a_planted_bug(bug, dtype):
    checks = [run_causal_census] if bug == "causal_off_by_one" else [run_decode_census]
    if bug in ("drop_row_256", "page_swapped", "neighbour_kv_head"):  # a doubled row 0 next to a needle elsewhere weighs nothing
        checks.append(run_decode_needles)
    for check in checks:
        with pytest.raises(AssertionError):
            check(bug, dtype)


def test_a_nan_or_a_one_ulp_slip_fails_the_bit_check():
    want = torch.tensor([0.25, 1.5, -3.0], dtype=torch.bfloat16)
    slip = want.clone()
    slip.view(torch.int16)[1] += 1
    for bad in (slip, torch.tensor([0.25, float("nan"), -3.0], dtype=torch.bfloat16)):
        with pytest.raises(AssertionError):
            assert_bits(bad, want, "slip")
    assert_within_ulp(slip, want, torch.bfloat16, "one ulp")
    slip.view(torch.int16)[1] += 1
    with pytest.raises(AssertionError):
        assert_within_ulp(slip, want, torch.bfloat16, "two ulps")


def test_census_classes_are_bounded_and_not_periodic():
    rng = np.random.default_rng(3)
    cls = random_classes(4096, HD, rng)
    assert np.bincount(cls, minlength=HD).max() <= 64 and prefix_counts(cls, HD, range(1, 4097)).max() <= 64
    assert not np.array_equal(cls[:HD], np.arange(HD))
    pages, pt = paged(np.zeros((40, 2, 1, HD), np.float32), rng)
    assert np.isnan(pages[np.setdiff1d(np.arange(pages.shape[0]), pt)]).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
def test_rope_tables_match_transformers_over_4096_positions(dtype, theta):
    """The decoder's host-built cos / sin tables equal transformers' LlamaRotaryEmbedding bit for bit at every position of the
    default 4096-token context."""
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding

    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    cfg = LlamaConfig(hidden_size=4096, num_attention_heads=32, head_dim=HD, rope_theta=theta, max_position_embeddings=4096)
    cos, sin = LlamaRotaryEmbedding(config=cfg)(torch.zeros(1, 4096, HD, dtype=dtype), torch.arange(4096)[None])
    tc, ts = build_rope_tables(LlamaDims(head_dim=HD, rope_theta=theta), 4096, "cpu", dtype)
    assert tc.dtype == dtype and tc.shape == (4096, HD // 2)
    for half in (slice(0, HD // 2), slice(HD // 2, HD)):
        assert torch.equal(cos[0, :, half], tc) and torch.equal(sin[0, :, half], ts)
