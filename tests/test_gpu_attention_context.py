"""Every attention entry point over the full 4096-token context, in both element builds, with checks whose expected outputs are
exact (see test_attention_context_cpu.py for the checkers and for proof that they reject a dropped, doubled or foreign row):

  * row census (q = 0): decode kernels bit-equal to elem(float32((1 + h) n_ch) / float32(L)), prefill kernels within one ulp;
  * needles (one row 40+ nats above the rest): the output is that row's V bit for bit, and in causal prefill only from its position on;
  * random data against float64, the decode kernels within one ulp of the element type.

Caches sit on a random permutation of physical pages; every page a sequence does not own, and every page-table entry past its last
page, holds NaN, so a stray read turns an output into NaN.  Page ids and addresses always stay in range."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import test_attention_context_cpu as C
from tests.util import assert_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
HD, PAGE = 128, 16
SCALE = HD ** -0.5
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}
LENS = [1, 2, 16, 17, 255, 256, 257, 258, 511, 1000, 2048, 4095, 4096]
NAN = float("nan")
# decode entry points: (kernel, q heads, kv heads); the batched kernel has specialisations for groups 1, 2, 4, 8, others fall back
DECODE = {"decode": ("decode", 32, 8), "batched_g1": ("batched", 4, 4), "batched_g2": ("batched", 8, 4), "batched_g4": ("batched", 32, 8),
          "batched_g8": ("batched", 32, 4), "batched_g3": ("batched", 12, 4), "batched_g6": ("batched", 24, 4),
          "tp_rank1_of_2": ("tp", 32, 8), "tp_rank3_of_4": ("tp", 32, 8)}
TP = {"tp_rank1_of_2": (2, 1), "tp_rank3_of_4": (4, 3)}  # (world, rank): the rank's q heads [rank nh/world, ...), kv_head_off > 0
NEEDLE_PAIRS = [(255, 256), (15, 16), (40, 41), (7, 2500)]  # equal scores across the 256 boundary / a page edge / half-warps


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import _lib, ops as _ops
    _lib.load()
    assert _lib.device_info()[1:] == (9, 0), "these tests need an sm_90 device"
    return _ops


# ---- caches ------------------------------------------------------------------------------------------------------------------
def build_pool(kv_rows, dtype, seed, tail=NAN):
    """kv_rows: per sequence a float32 tensor [L_b, 2, nkv, HD].  Returns (pages [P, 2, PAGE, nkv, HD] elem, page tables [B, cap]
    int32, physical pages of each sequence).  Slots past L_b in a sequence's last page hold `tail` (NaN, or finite for the paged
    prefill kernel, which loads whole 64-row tiles and masks what is past the causal limit)."""
    g = torch.Generator().manual_seed(seed)
    n_lp = [-(-r.shape[0] // PAGE) for r in kv_rows]
    n_phys = sum(n_lp) + 3
    perm = torch.randperm(n_phys, generator=g)
    nkv = kv_rows[0].shape[2]
    cap = max(n_lp) + 2
    pt = torch.full((len(kv_rows), cap), int(perm[-1]), dtype=torch.int32)  # unused entries -> a NaN page
    pages = torch.full((n_phys, 2, PAGE, nkv, HD), NAN, dtype=dtype, device=DEV)
    owned, o = [], 0
    for b, r in enumerate(kv_rows):
        ids = perm[o:o + n_lp[b]]
        o += n_lp[b]
        pt[b, :n_lp[b]] = ids
        owned.append(ids)
        pad = torch.full((n_lp[b] * PAGE, 2, nkv, HD), tail, dtype=torch.float32, device=DEV)
        pad[:r.shape[0]] = r.to(DEV)
        pages[ids.to(DEV)] = pad.view(n_lp[b], PAGE, 2, nkv, HD).transpose(1, 2).to(dtype)
    return pages, pt.to(DEV), owned


def only(pages, owned, b):
    """A copy of the pool in which every page not owned by sequence b is NaN."""
    p = torch.full_like(pages, NAN)
    p[owned[b].to(DEV)] = pages[owned[b].to(DEV)]
    return p


def gather(pages, pt_row, L):
    pos = torch.arange(L, device=DEV)
    return pages[pt_row[pos // PAGE].long(), :, pos % PAGE].double()  # [L, 2, nkv, HD]


def census_rows(L, nkv, rng, tg, hd=HD, pad_to=None):
    n = pad_to or L
    cls = C.random_classes(n, hd, rng)
    k = torch.randn(n, nkv, hd, generator=tg) * 0.5
    v = torch.from_numpy(C.census_values(cls, nkv, hd))
    return torch.stack([k, v], 1), cls


def expected_census(cls, lens, kv_of_head, dtype, hd=HD):
    return C.census_expected(C.prefix_counts(cls, hd, lens), lens, kv_of_head, dtype)


# ---- decode launches ---------------------------------------------------------------------------------------------------------
def run_decode(ops, name, pages, pt, lens, q, owned=None):
    """q [B, nh * HD] (a column slice of a wider buffer for the batched kernel) -> out [B, heads served * HD]."""
    kind, nh, nkv = DECODE[name]
    B, dtype = len(lens), pages.dtype
    pos = torch.tensor([L - 1 for L in lens], dtype=torch.int32, device=DEV)
    if kind == "batched":
        out = torch.full((B, nh * HD), NAN, dtype=dtype, device=DEV)
        return ops.attention_decode_batched(q, out, pages, pt, PAGE, pos, nh, nkv, HD, SCALE)
    world, rank = TP.get(name, (1, 0))
    nhl, grp = nh // world, nh // nkv
    out = torch.full((B, nhl * HD), NAN, dtype=dtype, device=DEV)
    for b in range(B):
        pg = pages if owned is None else only(pages, owned, b)
        if kind == "decode":
            ops.attention_decode(q[b].contiguous(), out[b], pg, pt[b].contiguous(), PAGE, pos[b:b + 1], nh, nkv, HD, SCALE)
        else:
            ql = q[b, rank * nhl * HD:(rank + 1) * nhl * HD].contiguous()
            ops.attention_decode_tp(ql, out[b], pg, pt[b].contiguous(), PAGE, pos[b:b + 1], nhl, grp, nkv, rank * nhl // grp, HD, SCALE)
    return out


def served_heads(name):
    kind, nh, nkv = DECODE[name]
    world, rank = TP.get(name, (1, 0))
    heads = np.arange(rank * nh // world, (rank + 1) * nh // world)
    return heads, heads // (nh // nkv)


def q_rows(B, nh, nkv):
    """q as the q columns of a fused qkv buffer [B, (nh + 2 nkv) HD] (a strided view)."""
    buf = torch.zeros(B, (nh + 2 * nkv) * HD, device=DEV)
    return buf, buf[:, :nh * HD]


# ---- 1. row census -----------------------------------------------------------------------------------------------------------
def decode_census(ops, name, dtype, seed=0):
    kind, nh, nkv = DECODE[name]
    rng, tg = np.random.default_rng(seed), torch.Generator().manual_seed(seed)
    rows, classes = zip(*(census_rows(L, nkv, rng, tg) for L in LENS))
    pages, pt, owned = build_pool(list(rows), dtype, seed)
    buf, _ = q_rows(len(LENS), nh, nkv)
    out = run_decode(ops, name, pages, pt, LENS, buf.to(dtype)[:, :nh * HD], owned=None if kind == "batched" else owned)
    heads, kv_of = served_heads(name)
    for b, L in enumerate(LENS):
        C.assert_bits(out[b].view(len(heads), HD), expected_census(classes[b], [L], kv_of, dtype)[0], f"{name} census, L = {L}")


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("name", list(DECODE))
def test_decode_row_census_is_exact(ops, elem, name):
    with ops.elem_dtype(DTYPES[elem]):
        decode_census(ops, name, DTYPES[elem])


def multi_census(ops, dtype, seed=1):
    nh, nkv = 32, 8
    rng, tg = np.random.default_rng(seed), torch.Generator().manual_seed(seed)
    for L in LENS:
        rows, cls = census_rows(L, nkv, rng, tg)
        pages, pt, _ = build_pool([rows], dtype, seed + L)
        for T in range(1, 9):
            if T > L:
                break
            _, q = q_rows(T, nh, nkv)
            out = torch.full((T, nh * HD), NAN, dtype=dtype, device=DEV)
            pos_rows = torch.arange(L - T, L, dtype=torch.int32, device=DEV)
            ops.attention_decode_multi(q.to(dtype), out, pages, pt[0], PAGE, pos_rows, nh, nkv, HD, SCALE)
            lens = list(range(L - T + 1, L + 1))
            C.assert_bits(out.view(T, nh, HD), expected_census(cls, lens, np.arange(nh) // (nh // nkv), dtype), f"multi census, L = {L}, T = {T}")


@pytest.mark.parametrize("elem", list(DTYPES))
def test_decode_multi_row_census_is_exact(ops, elem):
    with ops.elem_dtype(DTYPES[elem]):
        multi_census(ops, DTYPES[elem])


# ---- 2. needles --------------------------------------------------------------------------------------------------------------
def needle_pool(nkv, dtype, seed, lens=None):
    """Small random K (|score| <= 1 against the q vectors), V entries in +-{1..8}; q head h of kv head g carries qv[g]."""
    tg = torch.Generator().manual_seed(seed)
    qv = torch.randn(nkv, HD, generator=tg).to(dtype)
    rows, lens = [], lens or LENS
    for L in lens:
        k = torch.randn(L, nkv, HD, generator=tg) * 0.05
        v = torch.randint(1, 9, (L, nkv, HD), generator=tg).float() * (torch.randint(0, 2, (L, nkv, HD), generator=tg) * 2 - 1)
        rows.append(torch.stack([k, v], 1))
    pages, pt, owned = build_pool(rows, dtype, seed)
    qf = qv.double()
    needle_k = (qf * (45.0 / ((qf * qf).sum(-1, keepdim=True) * SCALE))).to(dtype)  # score ~ 45 nats
    s_needle = (needle_k.double() * qf).sum(-1) * SCALE
    for b, L in enumerate(lens):
        s = torch.einsum("lhd,hd->lh", gather(pages, pt[b], L)[:, 0], qf.to(DEV)) * SCALE
        assert float(s.abs().max()) <= 1 and float(s_needle.min()) >= 42, "needle premise: the needle leads every row by 41+ nats"
    return qv, needle_k.to(DEV), pages, pt, owned


def plant(pages, pt, b, j, h, kvec, vvec=None):
    pg, sl = int(pt[b, j // PAGE]), j % PAGE
    pages[pg, 0, sl, h] = kvec
    if vvec is not None:
        pages[pg, 1, sl, h] = vvec


def decode_needles(ops, name, dtype, seed=2):
    kind, nh, nkv = DECODE[name]
    qv, nk, base, pt, owned = needle_pool(nkv, dtype, seed)
    buf, q = q_rows(len(LENS), nh, nkv)
    q[:] = qv.to(DEV).float().repeat_interleave(nh // nkv, 0).reshape(-1)
    q = buf.to(dtype)[:, :nh * HD]
    heads, kv_of = served_heads(name)
    sweeps = [C.needle_positions(L) for L in LENS]
    for i in range(max(len(s) for s in sweeps)):
        pages = base.clone()
        where = [[s[(i + h) % len(s)] for h in range(nkv)] for s in sweeps]  # a different position for every kv head
        for b in range(len(LENS)):
            for h in range(nkv):
                plant(pages, pt, b, where[b][h], h, nk[h])
        out = run_decode(ops, name, pages, pt, LENS, q, owned=None if kind == "batched" else owned)
        for b, L in enumerate(LENS):
            g = gather(pages, pt[b], L)[:, 1]
            want = torch.stack([g[where[b][h], h] for h in kv_of])
            C.assert_bits(out[b].view(len(heads), HD), want, f"{name} needles {where[b]}, L = {L}")
    # two needles of equal score: their exact mean
    for j1, j2 in NEEDLE_PAIRS:
        pages = base.clone()
        vpair = [torch.randint(1, 9, (nkv, HD), generator=torch.Generator().manual_seed(j1 + j2 + t)).float().to(DEV) for t in (0, 1)]
        seqs = [b for b, L in enumerate(LENS) if j2 < L]
        for b in seqs:
            for h in range(nkv):
                plant(pages, pt, b, j1, h, nk[h], vpair[0][h])
                plant(pages, pt, b, j2, h, nk[h], vpair[1][h])
        out = run_decode(ops, name, pages, pt, LENS, q, owned=None if kind == "batched" else owned)
        want = ((vpair[0] + vpair[1]) / 2)[torch.as_tensor(kv_of, device=DEV)]
        for b in seqs:
            C.assert_bits(out[b].view(len(heads), HD), want, f"{name} needle pair {j1}, {j2}, L = {LENS[b]}")


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("name", list(DECODE))
def test_decode_needles_are_exact(ops, elem, name):
    with ops.elem_dtype(DTYPES[elem]):
        decode_needles(ops, name, DTYPES[elem])


# ---- 3. random data against float64 -----------------------------------------------------------------------------------------
def ref_attention(q, kv, grp, causal_from=None):
    """q [R, nh, hd] float64, kv [L, 2, nkv, hd] float64 -> [R, nh, hd]; row r sees positions [0, causal_from + r] (all when None).
    Four heads at a time, so 32 heads x 4096 x 4096 scores stay small."""
    L, R, hd = kv.shape[0], q.shape[0], q.shape[2]
    k = kv[:, 0].repeat_interleave(grp, 1)
    v = kv[:, 1].repeat_interleave(grp, 1)
    out = []
    for h0 in range(0, q.shape[1], 4):
        s = torch.einsum("rhd,lhd->hrl", q[:, h0:h0 + 4], k[:, h0:h0 + 4]) * hd ** -0.5
        if causal_from is not None:
            s = s.masked_fill(torch.arange(L, device=DEV)[None, None, :] > (causal_from + torch.arange(R, device=DEV))[None, :, None], float("-inf"))
        out.append(torch.einsum("hrl,lhd->rhd", s.softmax(-1), v[:, h0:h0 + 4]))
    return torch.cat(out, 1)


def random_pool(nkv, dtype, seed, lens=None):
    tg = torch.Generator().manual_seed(seed)
    return build_pool([torch.randn(L, 2, nkv, HD, generator=tg) for L in lens or LENS], dtype, seed)


def decode_random(ops, name, dtype, seed=3):
    kind, nh, nkv = DECODE[name]
    pages, pt, owned = random_pool(nkv, dtype, seed)
    buf, q = q_rows(len(LENS), nh, nkv)
    buf[:] = torch.randn(buf.shape, generator=torch.Generator().manual_seed(seed + 1)).to(DEV)
    qe = buf.to(dtype)[:, :nh * HD]
    out = run_decode(ops, name, pages, pt, LENS, qe, owned=None if kind == "batched" else owned)
    heads, _ = served_heads(name)
    for b, L in enumerate(LENS):
        kv = gather(pages, pt[b], L)
        ref = ref_attention(qe[b].double().view(1, nh, HD), kv, nh // nkv)[0, torch.as_tensor(heads, device=DEV)]
        C.assert_within_ulp(out[b].view(len(heads), HD), ref, dtype, f"{name} random, L = {L}", floor=2.0 ** -20 * float(kv[:, 1].abs().max()))


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("name", list(DECODE))
def test_decode_random_within_one_ulp_of_fp64(ops, elem, name):
    with ops.elem_dtype(DTYPES[elem]):
        decode_random(ops, name, DTYPES[elem])


@pytest.mark.parametrize("elem", list(DTYPES))
def test_decode_multi_random_within_one_ulp_of_fp64(ops, elem):
    dtype, nh, nkv, T = DTYPES[elem], 32, 8, 8
    with ops.elem_dtype(dtype):
        pages, pt, _ = random_pool(nkv, dtype, 4, lens=[4096])
        kv = gather(pages, pt[0], 4096)
        for L in [l for l in LENS if l >= T]:
            q = torch.randn(T, nh * HD, generator=torch.Generator().manual_seed(L)).to(dtype).to(DEV)
            out = torch.full((T, nh * HD), NAN, dtype=dtype, device=DEV)
            ops.attention_decode_multi(q, out, pages, pt[0], PAGE, torch.arange(L - T, L, dtype=torch.int32, device=DEV), nh, nkv, HD, SCALE)
            for t in range(T):
                ref = ref_attention(q[t].double().view(1, nh, HD), kv[:L - T + t + 1], nh // nkv)[0]
                C.assert_within_ulp(out[t].view(nh, HD), ref, dtype, f"multi random, L = {L}, t = {t}", floor=2.0 ** -20 * float(kv[:, 1].abs().max()))


# ---- knobs read once per process: no pre-wait prefetch, no programmatic dependent launch -------------------------------------
def knob_checks():
    from spatialrgpt_b200 import ops
    for dtype in DTYPES.values():
        with ops.elem_dtype(dtype):
            for name in ("decode", "tp_rank1_of_2"):
                decode_census(ops, name, dtype)
                decode_needles(ops, name, dtype)
            multi_census(ops, dtype)
    print("KNOB_OK")


@pytest.mark.parametrize("knob", ["SRGPT_ATTN_NO_PREFETCH", "SRGPT_NO_PDL"])
def test_decode_census_and_needles_under_knobs(knob):
    env = dict(os.environ, **{knob: "1"})
    code = "from tests.test_gpu_attention_context import knob_checks; knob_checks()"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and "KNOB_OK" in r.stdout, knob + ": " + r.stdout[-3000:] + r.stderr[-3000:]


# ---- dense prefill (attention_prefill / attention_prefill_varlen) ------------------------------------------------------------
# (head_dim, q heads, kv heads, sequence lengths, causal): SigLIP 16 x 72 at 729 / 1024 rows per image, the CLIP tower's 64,
# Llama-3-8B 32 / 8 x 128 over the whole context
DENSE = [(72, 16, 16, [729, 729], False), (72, 16, 16, [1024], False), (64, 16, 16, [577, 577], False), (64, 4, 2, [4096], True),
         (128, 32, 8, [4096], True), (128, 32, 8, [1000, 1000], False), (72, 16, 16, [1024], True)]
VARLEN = [(128, 32, 8, [1000, 1, 1999, 1096], True), (72, 16, 16, [729, 1024, 729], False), (64, 4, 2, [300, 64, 65], True)]


def dense_qkv(rows, nh, nkv, hd, dtype):
    """The fused [S, (nh + 2 nkv) hd] buffer the models hand over, and its q / k / v column views."""
    d = torch.cat([rows[0], rows[1], rows[2]], 1).to(dtype).to(DEV).contiguous()
    return d, d[:, :nh * hd], d[:, nh * hd:(nh + nkv) * hd], d[:, (nh + nkv) * hd:]


def run_dense(ops, case, q, k, v, varlen):
    hd, nh, nkv, lens, causal = case
    if varlen:
        cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=DEV)
        return ops.attention_prefill_varlen(q, k, v, cu, max(lens), nh, nkv, hd, hd ** -0.5, causal)
    return ops.attention_prefill(q, k, v, len(lens), lens[0], nh, nkv, hd, hd ** -0.5, causal)


def dense_census(ops, case, dtype, varlen, seed=5):
    hd, nh, nkv, lens, causal = case
    rng, tg = np.random.default_rng(seed), torch.Generator().manual_seed(seed)
    ks, vs, cls = [], [], []
    for n in lens:
        c = C.random_classes(n, hd, rng)
        cls.append(c)
        ks.append(torch.randn(n, nkv * hd, generator=tg) * 0.5)
        vs.append(torch.from_numpy(C.census_values(c, nkv, hd)).view(n, nkv * hd))
    S = sum(lens)
    _, q, k, v = dense_qkv([torch.zeros(S, nh * hd), torch.cat(ks), torch.cat(vs)], nh, nkv, hd, dtype)
    out = run_dense(ops, case, q, k, v, varlen).view(S, nh, hd)
    kv_of, o = np.arange(nh) // (nh // nkv), 0
    for b, n in enumerate(lens):
        vis = [r + 1 for r in range(n)] if causal else [n] * n
        C.assert_within_ulp(out[o:o + n], expected_census(cls[b], vis, kv_of, dtype, hd), dtype, f"prefill census {case}, sequence {b}")
        o += n


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("case", DENSE + VARLEN, ids=[f"{'varlen' if i >= len(DENSE) else 'dense'}-hd{c[0]}-{c[1]}x{c[2]}-{'-'.join(map(str, c[3]))}-{'causal' if c[4] else 'full'}"
                                                     for i, c in enumerate(DENSE + VARLEN)])
def test_dense_prefill_row_census(ops, elem, case):
    with ops.elem_dtype(DTYPES[elem]):
        dense_census(ops, case, DTYPES[elem], varlen=case in VARLEN)


PREFILL_NEEDLES = [0, 1, 63, 64, 127, 128, 255, 256, 2047, 4094, 4095]


def causal_needles(L, nkv, nh, dtype, seed, run):
    """K = 0 except one needle row per kv head at P_h (score ~ 45 nats against every q row); V census plus the needle's row.
    Rows at positions >= P_h must return the needle's V bit for bit, rows before it the census of positions [0, pos]."""
    rng, tg = np.random.default_rng(seed), torch.Generator().manual_seed(seed)
    cls = C.random_classes(L, HD, rng)
    v = torch.from_numpy(C.census_values(cls, nkv, HD))
    qv = torch.randn(nkv, HD, generator=tg).to(dtype).double()
    nk = (qv * (45.0 / ((qv * qv).sum(-1, keepdim=True) * SCALE))).to(dtype)
    vn = torch.randint(1, 9, (nkv, HD), generator=tg).float()
    kv_of = np.arange(nh) // (nh // nkv)
    js = [j for j in PREFILL_NEEDLES if j < L]
    census = None
    for i in range(len(js)):
        where = [js[(i + h) % len(js)] for h in range(nkv)]
        k, vv = torch.zeros(L, nkv, HD), v.clone()
        for h in range(nkv):
            k[where[h], h] = nk[h].float()
            vv[where[h], h] = vn[h]
        out = run(qv.float().repeat_interleave(nh // nkv, 0), k, vv).cpu()  # -> [rows, nh, HD] at positions pos0 .. L - 1
        pos0 = L - out.shape[0]
        if census is None:
            census = expected_census(cls, list(range(pos0 + 1, L + 1)), kv_of, dtype)
        for hh in range(nh):
            P = where[kv_of[hh]]
            r = max(P - pos0, 0)
            if r < out.shape[0]:
                C.assert_bits(out[r:, hh], vn[kv_of[hh]].expand(out.shape[0] - r, HD), f"needle at {P}, head {hh}, rows from {pos0 + r}")
            if r > 0:
                C.assert_within_ulp(out[:r, hh], census[:r, hh], dtype, f"census before the needle at {P}, head {hh}")


@pytest.mark.parametrize("elem", list(DTYPES))
def test_dense_causal_prefill_needles(ops, elem):
    dtype, nh, nkv, L = DTYPES[elem], 32, 8, 4096

    def run(q, k, v):
        _, qq, kk, vv = dense_qkv([q.reshape(1, -1).expand(L, -1), k.reshape(L, -1), v.reshape(L, -1)], nh, nkv, HD, dtype)
        return ops.attention_prefill(qq, kk, vv, 1, L, nh, nkv, HD, SCALE, True).view(L, nh, HD)
    with ops.elem_dtype(dtype):
        causal_needles(L, nkv, nh, dtype, 6, run)


def assert_close_by_rows(out, ref, what, rows=64):
    """The prefill kernels' relative bounds (rel_rms 1e-2, rel_max 8e-2) per block of 64 query rows.  A causal row's output shrinks
    like 1 / sqrt(visible rows), so over a whole 4096-row tensor the reference RMS is set by the late rows, and one bf16 rounding of
    an early row (values of order 1) alone would exceed rel_max."""
    for r0 in range(0, out.shape[0], rows):
        assert_close(out[r0:r0 + rows], ref[r0:r0 + rows], rel_rms=1e-2, rel_max=8e-2, what=f"{what}, rows {r0}..{min(r0 + rows, out.shape[0]) - 1}")


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("case", DENSE + VARLEN, ids=[f"{'varlen' if i >= len(DENSE) else 'dense'}-hd{c[0]}-{c[1]}x{c[2]}-{'-'.join(map(str, c[3]))}-{'causal' if c[4] else 'full'}"
                                                     for i, c in enumerate(DENSE + VARLEN)])
def test_dense_prefill_random_against_fp64(ops, elem, case):
    dtype = DTYPES[elem]
    hd, nh, nkv, lens, causal = case
    S = sum(lens)
    tg = torch.Generator().manual_seed(7)
    with ops.elem_dtype(dtype):
        d, q, k, v = dense_qkv([torch.randn(S, nh * hd, generator=tg), torch.randn(S, nkv * hd, generator=tg), torch.randn(S, nkv * hd, generator=tg)],
                               nh, nkv, hd, dtype)
        out = run_dense(ops, case, q, k, v, varlen=case in VARLEN)
        o = 0
        for n in lens:
            kv = torch.stack([k[o:o + n].double().view(n, nkv, hd), v[o:o + n].double().view(n, nkv, hd)], 1)
            ref = ref_attention(q[o:o + n].double().view(n, nh, hd), kv, nh // nkv, causal_from=0 if causal else None)
            assert_close_by_rows(out[o:o + n], ref.reshape(n, nh * hd), f"prefill {case}, sequence at row {o}")
            o += n


# ---- paged chunked prefill (attention_prefill_paged) -------------------------------------------------------------------------
# (q heads, kv heads, chunks as (start_pos, rows)); several chunks = one packed call, one sequence each
PAGED = [(32, 8, [(0, 4096)]), (32, 8, [(1000, 257)]), (32, 8, [(3840, 256)]), (32, 8, [(4000, 96)]), (32, 8, [(2047, 1)]),
         (32, 8, [(4095, 1)]), (32, 8, [(255, 2)]), (4, 2, [(17, 300)]), (32, 8, [(3796, 300), (16, 129), (1000, 7), (4095, 1)]),
         (4, 2, [(3000, 1096), (0, 1)])]


def run_paged(ops, pages, pt, chunks, q, nh, nkv):
    cu = torch.tensor([0] + np.cumsum([n for _, n in chunks]).tolist(), dtype=torch.int32, device=DEV)
    sp = torch.tensor([s for s, _ in chunks], dtype=torch.int32, device=DEV)
    return ops.attention_prefill_paged(q, pages, pt, PAGE, sp, cu, max(n for _, n in chunks), nh, nkv, HD, SCALE)


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,chunks", PAGED, ids=[f"{a}x{b}-" + "-".join(f"{s}+{n}" for s, n in c) for a, b, c in PAGED])
def test_paged_prefill_row_census(ops, elem, nh, nkv, chunks):
    dtype = DTYPES[elem]
    rng, tg = np.random.default_rng(8), torch.Generator().manual_seed(8)
    rows, cls = [], []
    for s, n in chunks:
        L = s + n
        r, c = census_rows(L, nkv, rng, tg, pad_to=-(-L // PAGE) * PAGE)  # slots past L hold finite census rows of their own
        rows.append(r)
        cls.append(c)
    R = sum(n for _, n in chunks)
    with ops.elem_dtype(dtype):
        pages, pt, _ = build_pool(rows, dtype, 9, tail=0.0)
        buf, _ = q_rows(R, nh, nkv)
        out = run_paged(ops, pages, pt, chunks, buf.to(dtype)[:, :nh * HD], nh, nkv).view(R, nh, HD)
        o, kv_of = 0, np.arange(nh) // (nh // nkv)
        for b, (s, n) in enumerate(chunks):
            C.assert_within_ulp(out[o:o + n], expected_census(cls[b], list(range(s + 1, s + n + 1)), kv_of, dtype), dtype,
                                f"paged census, chunk {b} at {s} + {n}")
            o += n


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("start,rows", [(0, 4096), (3000, 1096)])
def test_paged_prefill_needles(ops, elem, start, rows):
    dtype, nh, nkv, L = DTYPES[elem], 32, 8, start + rows

    def run(q, k, v):
        pages, pt, _ = build_pool([torch.stack([k, v], 1)], dtype, 10, tail=0.0)
        qq = q.reshape(1, -1).expand(rows, -1).to(dtype).to(DEV).contiguous()
        return run_paged(ops, pages, pt, [(start, rows)], qq, nh, nkv).view(rows, nh, HD)
    with ops.elem_dtype(dtype):
        causal_needles(L, nkv, nh, dtype, 11, run)


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,chunks", [(32, 8, [(0, 4096)]), (32, 8, [(3000, 1096)]), (32, 8, [(3796, 300), (16, 129), (4095, 1)])])
def test_paged_prefill_random_against_fp64(ops, elem, nh, nkv, chunks):
    dtype = DTYPES[elem]
    tg = torch.Generator().manual_seed(12)
    with ops.elem_dtype(dtype):
        pages, pt, _ = build_pool([torch.randn(s + n, 2, nkv, HD, generator=tg) for s, n in chunks], dtype, 13, tail=0.0)
        R = sum(n for _, n in chunks)
        q = torch.randn(R, nh * HD, generator=tg).to(dtype).to(DEV)
        out = run_paged(ops, pages, pt, chunks, q, nh, nkv)
        o = 0
        for b, (s, n) in enumerate(chunks):
            ref = ref_attention(q[o:o + n].double().view(n, nh, HD), gather(pages, pt[b], s + n), nh // nkv, causal_from=s)
            assert_close_by_rows(out[o:o + n], ref.reshape(n, nh * HD), f"paged random chunk {b} at {s} + {n}")
            o += n


# ---- writes into the cache at long positions ---------------------------------------------------------------------------------
def rope_ref(x, cos, sin, dtype):
    """x [rows, heads, HD] rotated with the element type's rounding after every product and the sum (modeling_llama.py:186-191)."""
    c = torch.cat([cos, cos], -1)[:, None].to(dtype)
    s = torch.cat([sin, sin], -1)[:, None].to(dtype)
    rot = torch.cat([-x[..., HD // 2:], x[..., :HD // 2]], -1)
    return (x * c) + (rot * s)


def assert_cache_writes(before, after, writes, what):
    """writes: (page table, positions, k rows [n, nkv, HD], v rows).  Each row lands bit for bit at page_table[pos // 16], slot
    pos % 16, and every other byte of the page array is unchanged."""
    want = before.clone()
    for pt, positions, k_rows, v_rows in writes:
        for i, pos in enumerate(positions):
            pg, sl = int(pt[pos // PAGE]), pos % PAGE
            want[pg, 0, sl] = k_rows[i].to(DEV)
            want[pg, 1, sl] = v_rows[i].to(DEV)
    bad = after.view(torch.int16) != want.view(torch.int16)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} cache elements differ, first at {tuple(int(x) for x in bad.nonzero()[0])}"


@pytest.mark.parametrize("elem", list(DTYPES))
def test_rope_kv_append_at_the_end_of_the_context(ops, elem):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    dtype, nh, nkv = DTYPES[elem], 32, 8
    cos, sin = build_rope_tables(LlamaDims(head_dim=HD, rope_theta=500000.0), 4096, DEV, dtype)
    tg = torch.Generator().manual_seed(14)
    n_lp = 4096 // PAGE
    n_pages = 2 * n_lp + 4
    pt_all = torch.randperm(n_pages, generator=tg)[:2 * n_lp].to(torch.int32).view(2, n_lp)
    with ops.elem_dtype(dtype):
        # one sequence: rows at positions 4077 .. 4095; packed: two sequences at 4090 .. 4095 and 2999 .. 3035
        for starts, lens in (([4077], [19]), ([4090, 2999], [6, 37])):
            qkv = torch.randn(sum(lens), (nh + 2 * nkv) * HD, generator=tg).to(dtype)
            pages = torch.randn(n_pages, 2, PAGE, nkv, HD, generator=tg).to(dtype).to(DEV)
            before, d = pages.clone(), qkv.to(DEV)
            sp = torch.tensor(starts, dtype=torch.int32, device=DEV)
            pts = pt_all[:len(starts)].contiguous().to(DEV)
            if len(starts) == 1:
                ops.rope_kv_append(d, nh, nkv, HD, cos, sin, sp, pages, pts[0], PAGE)
            else:
                cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=DEV)
                ops.rope_kv_append_varlen(d, nh, nkv, HD, cos, sin, sp, pages, pts, PAGE, cu)
            writes, o = [], 0
            for b, (s, n) in enumerate(zip(starts, lens)):
                pos = list(range(s, s + n))
                blk = qkv[o:o + n]
                c, sn = cos[pos].cpu(), sin[pos].cpu()
                qr = rope_ref(blk[:, :nh * HD].view(n, nh, HD), c, sn, dtype)
                kr = rope_ref(blk[:, nh * HD:(nh + nkv) * HD].view(n, nkv, HD), c, sn, dtype)
                assert torch.equal(d[o:o + n, :nh * HD].cpu().view(n, nh, HD), qr), f"rotated q, sequence {b}"
                assert torch.equal(d[o:o + n, nh * HD:(nh + nkv) * HD].cpu().view(n, nkv, HD), kr), f"rotated k, sequence {b}"
                writes.append((pt_all[b], pos, kr, blk[:, (nh + nkv) * HD:].view(n, nkv, HD)))
                o += n
            assert_cache_writes(before, pages, writes, f"rope_kv_append at {starts}")


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("pos", [4080, 4094, 4095])
def test_gemv_qkv_rope_appends_at_the_end_of_the_context(ops, elem, pos):
    from oracle import srgpt_oracle as O
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    from tests.util import BF16_CHAIN
    dtype, nh, nkv, K = DTYPES[elem], 32, 8, 4096
    N = (nh + 2 * nkv) * HD
    tg = torch.Generator().manual_seed(pos)
    x = torch.randn(K, generator=tg).to(dtype)
    nw = (1 + 0.1 * torch.randn(K, generator=tg)).to(dtype)
    w = (torch.randn(N, K, generator=tg) * K ** -0.5).to(dtype)
    cos, sin = build_rope_tables(LlamaDims(head_dim=HD, rope_theta=500000.0), 4096, DEV, dtype)
    n_pages = 4096 // PAGE + 3
    pt = torch.randperm(n_pages, generator=tg)[:4096 // PAGE + 1].to(torch.int32)
    with ops.elem_dtype(dtype):
        pages = torch.randn(n_pages, 2, PAGE, nkv, HD, generator=tg).to(dtype).to(DEV)
        before = pages.clone()
        q = torch.empty(nh * HD, dtype=dtype, device=DEV)
        ops.gemv(x.to(DEV), w.to(DEV), q, norm_weight=nw.to(DEV), eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=HD,
                 cos_tab=cos, sin_tab=sin, pos=torch.tensor([pos], dtype=torch.int32, device=DEV), kv_pages=pages, page_table=pt.to(DEV),
                 page_size=PAGE)
    pg, sl = int(pt[pos // PAGE]), pos % PAGE
    full = w.float() @ O.rms_norm(x.float(), nw.float(), 1e-5)
    c, s = cos[pos].cpu().float().repeat(2), sin[pos].cpu().float().repeat(2)
    kr = full[nh * HD:(nh + nkv) * HD].view(nkv, HD)
    assert_close(pages[pg, 0, sl], kr * c + O.rotate_half(kr) * s, **BF16_CHAIN, what="k row")
    assert_close(pages[pg, 1, sl], full[(nh + nkv) * HD:].view(nkv, HD), **BF16_CHAIN, what="v row")
    assert_cache_writes(before, pages, [(pt, [pos], pages[pg, 0, sl][None], pages[pg, 1, sl][None])], f"gemv qkv append at {pos}")


# ---- one end-to-end run at long context --------------------------------------------------------------------------------------
def test_long_context_chunked_prefill_and_graph_decode_against_the_oracle():
    """tiny_masks_gqa (hd 128, GQA 4 / 2) with max_seq_len 4096: 4000 prompt rows through three prefill chunks, then 40 graph-decoded
    tokens (positions up to 4039), against the fp32 CPU oracle's greedy search."""
    from oracle import srgpt_oracle as O
    from tests.golden.make_golden import CASES
    from tests.test_gpu_pipeline import build_model
    kw = CASES["tiny_masks_gqa"][0]
    oc, sd, model = build_model(kw, 41, max_seq_len=4096)
    llm, S, n_new = model.llm, 4000, 40
    emb = (torch.randn(S, oc.hidden, generator=torch.Generator().manual_seed(42)) * 0.05).to(DEV, model.dtype)
    llm.generate_from_embeds(emb[:1500], 1)
    llm.generate_from_embeds(emb[:3100], 1, reuse_rows=1500)
    ids, lg = llm.generate_from_embeds(emb, n_new, return_logits=True, reuse_rows=3100, use_graph=True)
    assert llm.prefix_rows == S
    ref_ids, ref_lg = O.greedy_generate(oc, sd["llm"], emb.float().cpu(), n_new, return_logits=True)
    sigma = float(ref_lg.std())
    err = float((lg.float().cpu() - ref_lg).abs().max())
    assert err <= 0.06 * sigma, f"logit error {err:.4f} > 0.06 sigma ({sigma:.3f})"
    top2 = ref_lg.topk(2, -1).values
    safe = int(((top2[:, 0] - top2[:, 1]) > 0.12 * sigma).long().cumprod(0).sum())
    assert ids.tolist()[:safe] == ref_ids.tolist()[:safe], f"greedy ids differ within the first {safe} clear steps"
