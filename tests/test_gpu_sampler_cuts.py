"""The sampler's top-k and top-p cuts on the H100 against transformers' TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper,
on the row families of tests/test_sampler_cuts_cpu.py (confident rows past the resolution of a probability cut and past fp32 exp
underflow, blocks straddling k, near-ties and division ties at the k-th value, masked rows, 16-bit rows with many ties), through every
entry point (sample_top_p with and without scores, sample_rows over fp32 and element-type rows, the warped forms with the warpers off and
on) in both builds: the finite entries of the score row are HF's top-k set exactly and HF's top-p set within DESIGN.md §7, the warped
values are HF's x / T bit for bit, and every draw over 2^17 (row, seed) pairs lies in HF's set with a positive probability."""
import numpy as np
import pytest
import torch

from spatialrgpt_b200.llama_decoder import sequence_seeds
from tests import warpers_oracle as W
from tests.test_gpu_warpers import _near_cut, _splits_a_tie
from tests.test_sampler_cuts_cpu import (KS, PS, TS, VS, check_top_p, check_topk, confident, elem_ties, family_rows, hf_warp,
                                         masked)

pytestmark = pytest.mark.gpu
DEV = "cuda"
ELEMS = [torch.bfloat16, torch.float16]
WARPED = (0.2, 50, 1.0, 0.9, 3e-4, 2e-3)  # (T, top_k, top_p, typical_p, epsilon, eta): the warpers after top-k 50 at T = 0.2


def _params(T, k, p, *warp):
    return torch.tensor([T, p, k, *warp], dtype=torch.float32, device=DEV)


def _step(v=0):
    return torch.full((1,), v, dtype=torch.int32, device=DEV)


def _rows(x, params, seeds=None, step=0, scores=True):
    """sample_rows over rows [R, V] on the device -> (ids, warped rows [R, V] on the host, or None)."""
    from spatialrgpt_b200 import ops
    R, V = x.shape
    seeds = torch.arange(R, dtype=torch.int64, device=DEV) if seeds is None else seeds
    ids = torch.empty(R, dtype=torch.int64, device=DEV)
    if not scores:
        ops.sample_rows(x, params, seeds, _step(step), 0, ids)
        return ids.cpu(), None
    sc = torch.empty((1, R, V), dtype=torch.float32, device=DEV)
    ops.sample_rows(x, params, seeds, _step(step), 0, ids, scores=sc)
    return ids.cpu(), sc[0].cpu()


def _one(x, params, seed, scores):
    """sample_top_p over one fp32 row on the device -> (id, warped row or None)."""
    from spatialrgpt_b200 import ops
    out = torch.full((1,), -1, dtype=torch.int64, device=DEV)
    seed = torch.tensor([seed], dtype=torch.int64, device=DEV)
    if not scores:
        ops.sample_top_p(x, params, seed, _step(), 0, out)
        return int(out), None
    sc = torch.empty(x.numel(), dtype=torch.float32, device=DEV)
    ops.sample_top_p(x, params, seed, _step(), 0, out, scores=sc, step_stride=x.numel())
    return int(out), sc.cpu()


def _check_rows(x, ids, got, T, k, p, where):
    """Warped rows [R, V] of fp32 rows x against HF: values bit-equal to x / T where kept, the kept set HF's (top-k exactly, top-p
    within §7), and every draw in the kept set with a positive float64 probability (under HF's renormalised distribution where the
    sets are HF's exactly: top_p = 1)."""
    ref = hf_warp(x, T, k, p)
    fin = torch.isfinite(got)
    assert torch.equal(got[fin], (x / T)[fin]), where
    prob = torch.softmax((ref if p >= 1.0 else got).double(), -1)
    assert bool((prob.gather(1, ids[:, None]) > 0).all()), (where, ids.tolist())
    if p >= 1.0:
        check_topk(got, ref, x, T, where)
        if k == 1:
            assert torch.equal(fin, (x / T) == (x / T).max(-1, keepdim=True).values), where
    else:
        check_top_p(fin, x, T, k, p, where)


@pytest.mark.parametrize("V", VS)
@pytest.mark.parametrize("elem", ELEMS)
def test_fp32_rows_keep_hfs_sets(elem, V):
    from spatialrgpt_b200 import ops
    with ops.elem_dtype(elem):
        for T in TS:
            for k in KS:
                x = family_rows(V, T, k)
                xd = x.to(DEV)
                for p in PS:
                    ids, got = _rows(xd, _params(T, k, p))
                    _check_rows(x, ids, got, T, k, p, (V, T, k, p))


@pytest.mark.parametrize("elem", ELEMS)
def test_element_type_rows_with_ties_keep_hfs_sets_and_draw_as_fp32(elem):
    from spatialrgpt_b200 import ops
    with ops.elem_dtype(elem):
        for V, T, k in ((32000, 1.0, 50), (32002, 0.7, 2), (128256, 0.2, 50), (128259, 0.05, 1000), (1000, 0.7, 50)):
            x16 = torch.cat([torch.stack([elem_ties(V, k, elem, seed=s) for s in range(32)]), family_rows(V, T, k).to(elem)])  # R = 64
            x = x16.float()
            for p in (1.0, 0.95):
                ids, got = _rows(x16.to(DEV), _params(T, k, p))
                _check_rows(x, ids, got, T, k, p, (elem, V, T, k, p))
                ids32, got32 = _rows(x.to(DEV), _params(T, k, p))
                assert torch.equal(ids, ids32) and torch.equal(got, got32)


@pytest.mark.parametrize("elem", ELEMS)
def test_every_entry_point_draws_alike_and_keeps_hfs_sets(elem):
    from spatialrgpt_b200 import ops
    with ops.elem_dtype(elem):
        for V in (1000, 128259):
            for T, k, p in ((0.2, 50, 1.0), (0.2, 50, 0.95), (0.7, 1, 1.0), (1.0, 1000, 0.5), (0.05, 2, 1.0)):
                x = family_rows(V, T, k)
                p3, p6 = _params(T, k, p), _params(T, k, p, 1.0, 0.0, 0.0)
                for R in (1, 3, 32):
                    rows = x[:R].to(DEV)
                    seeds = torch.tensor(sequence_seeds(R + 3, R), dtype=torch.int64, device=DEV)
                    ids, got = _rows(rows, p3, seeds)
                    _check_rows(x[:R], ids, got, T, k, p, (V, T, k, p, R))
                    ids6, got6 = _rows(rows, p6, seeds)
                    assert torch.equal(ids, ids6) and torch.equal(got, got6)
                    if R == 3:
                        for r in range(R):
                            row = rows[r].contiguous()
                            for params in (p3, p6):
                                a, _ = _one(row, params, int(seeds[r]), False)
                                b, sc = _one(row, params, int(seeds[r]), True)
                                assert a == b == int(ids[r]) and torch.equal(sc, got[r]), (V, T, k, p, r)
            # the warpers on, after top-k 50 at T = 0.2: HF's chain within §7, one-row and rows forms alike
            x = family_rows(V, 0.2, 50)
            T, k, p, typ, eps, eta = WARPED
            pw = _params(T, k, p, typ, eps, eta)
            ids, got = _rows(x.to(DEV), pw)
            fin = torch.isfinite(got)
            assert torch.equal(got[fin], (x / T)[fin])
            for r in range(x.shape[0]):
                assert bool(fin[r, int(ids[r])]) and float(torch.softmax(got[r].double(), 0)[int(ids[r])]) > 0
                if torch.equal(fin[r], W.kept(x[r], *WARPED) & torch.isfinite(x[r])) or _splits_a_tie(x[r], WARPED):
                    continue
                lo, hi = _near_cut(x[r], WARPED)
                assert bool((lo <= fin[r]).all() and (fin[r] <= hi).all()), (V, r)
            for r in (0, 20, 29):
                a, sc = _one(x[r].to(DEV), pw, r, True)
                assert a == int(ids[r]) and torch.equal(sc, got[r])


def _draw_rows(V=128256):
    """The rows of the draw tests: N(0, 0.1) with the top token 18.5 nats above the 50th, a 25-nat confident row, a masked row and a
    masked row with fewer than 50 finite entries."""
    g = torch.Generator().manual_seed(5)
    a = torch.randn(V, generator=g) * 0.1
    a[int(torch.randint(V, (1,), generator=g))] = float(a.sort(descending=True).values[48]) + 18.5
    return torch.stack([a, confident(V, 1.0, 25, 1.0, seed=4), masked(V, seed=1), masked(V, finite=20, seed=2)])


def test_draws_over_2_17_row_seed_pairs_lie_in_hfs_top_k_set():
    from scipy.stats import chisquare
    x = _draw_rows()
    T, k = 1.0, 50
    ref = hf_warp(x, T, k, 1.0)
    keep = torch.isfinite(ref)
    assert keep.sum(-1).tolist() == [50, 50, 50, 20]
    prob = torch.softmax(ref.double(), -1)
    n_seeds, n_steps = 256, 128
    rows = x.repeat_interleave(n_seeds, 0).to(DEV)  # [4 * 256, V]
    seeds = torch.tensor(sequence_seeds(77, rows.shape[0]), dtype=torch.int64, device=DEV)
    params = _params(T, k, 1.0)
    counts = torch.zeros_like(prob)
    first = None
    for step in range(n_steps):
        ids, got = _rows(rows, params, seeds, step, scores=step == 0)
        if step == 0:
            first = (ids, got)
            assert torch.equal(torch.isfinite(got[::n_seeds]), keep)
        d = ids.view(4, n_seeds)
        assert bool(keep.gather(1, d).all()), f"step {step}: {int((~keep.gather(1, d)).sum())} draws outside HF's top-{k} set"
        assert bool((prob.gather(1, d) > 0).all())
        counts.scatter_add_(1, d, torch.ones_like(d, dtype=counts.dtype))
    again = _rows(rows, params, seeds, 0)
    assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])  # two launches are bit-identical
    n = n_seeds * n_steps
    for r in (0, 2):  # the confident and the masked row: the draws follow HF's renormalised distribution
        exp = prob[r].numpy() * n
        obs = counts[r].numpy()
        big = exp >= 5
        obs_b, exp_b = np.append(obs[big], obs[~big].sum()), np.append(exp[big], exp[~big].sum())
        if exp_b[-1] == 0:
            obs_b, exp_b = obs_b[:-1], exp_b[:-1]
        if len(exp_b) > 1:
            assert chisquare(obs_b, exp_b).pvalue > 1e-3, r


def test_rows_draws_equal_one_row_draws():
    from spatialrgpt_b200 import ops
    x = _draw_rows(128259)
    for T, k, p in ((1.0, 50, 1.0), (0.2, 50, 0.95)):
        params = _params(T, k, p)
        for r in range(x.shape[0]):
            R = 16
            seeds = torch.tensor(sequence_seeds(r + 40, R), dtype=torch.int64, device=DEV)
            row = x[r].to(DEV)
            ids = torch.empty(R, dtype=torch.int64, device=DEV)
            ops.sample_rows(row[None].expand(R, -1).contiguous(), params, seeds, _step(3), 0, ids)
            one = []
            for i in range(R):
                out = torch.full((4,), -1, dtype=torch.int64, device=DEV)
                ops.sample_top_p(row, params, seeds[i:i + 1], _step(3), 0, out)
                one.append(int(out[3]))
            assert ids.tolist() == one, (T, k, p, r)
