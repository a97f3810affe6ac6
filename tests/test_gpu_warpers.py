"""Typical, epsilon and eta sampling on the H100: the warped sampler's kept set against transformers 5.5 on every golden row in both
element types, the one-row and rows kernels' draws, the draw frequencies, and the decoder's sampled paths (batch 1, batched,
num_return_sequences, batch-invariant rows, guidance): epsilon_cutoff=0.99 against greedy, graph against eager, rows against batch 1,
warpers off bit-identical to today, and the ValueError before any device work."""
import numpy as np
import pytest
import torch

from spatialrgpt_b200.llama_decoder import sequence_seeds
from tests import warpers_oracle as W
from tests.test_warpers_cpu import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAU, DEV_SLACK = 1e-4, 1e-5  # DESIGN.md §7: a token may differ from HF only this close to a cut


def _params(st):
    """The sampler's float[6] {T, top_p, top_k, typical_p, epsilon, eta} of a golden setting (T, top_k, top_p, typical_p, epsilon, eta)."""
    T, k, p, typ, eps, eta = (float(v) for v in st)
    return torch.tensor([T, p, k, typ, eps, eta], dtype=torch.float32, device=DEV)


def _near_cut(x, st):
    """(smallest, largest) kept sets of the HF chain with top_p / typical_p / epsilon / eta moved by a relative TAU and typical's
    deviation threshold by DEV_SLACK (float64 oracle)."""
    T, k, p, typ, eps, eta = st
    out = []
    for sg in (-1, 1):
        base = W.base_keep(x, T, int(k), min(p * (1 + sg * TAU), 1.0) if p < 1 else p)
        out.append(W.cuts(x, base, T, typ * (1 + sg * TAU) if typ < 1 else typ, eps * (1 - sg * TAU), eta * (1 - sg * TAU),
                          dev_slack=sg * DEV_SLACK))
    return out


def _splits_a_tie(x, st):
    """Whether HF's top-p (its sort) splits tokens of equal score: the nucleus keeps every tie here (DESIGN.md §7), HF a sorted prefix."""
    T, k, p = st[:3]
    base = W.base_keep(x, T, int(k), p)
    if p >= 1:
        return False
    kept, dropped = set(x[base].tolist()), set(x[~base & torch.isfinite(x)].tolist())
    return bool(kept & dropped)


@pytest.mark.parametrize("elem", [torch.bfloat16, torch.float16])
def test_kept_set_equals_hf_on_every_golden_row(elem):
    from spatialrgpt_b200 import ops
    settings, sets, _ = golden()
    compared, exceptions, inputs = 0, 0, 2 if elem == torch.bfloat16 else 1
    with ops.elem_dtype(elem):
        for V, x, keep in sets:
            R = x.shape[0]
            for j, st in enumerate(settings):
                rows = [x.to(DEV)] + ([x.to(DEV, torch.bfloat16)] if elem == torch.bfloat16 else [])
                for lg in rows:
                    scores = torch.empty((1, R, V), dtype=torch.float32, device=DEV)
                    ids = torch.empty(R, dtype=torch.int64, device=DEV)
                    ops.sample_rows(lg, _params(st), torch.arange(R, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV),
                                    0, ids, scores=scores)
                    got = torch.isfinite(scores[0]).cpu()
                    for r in range(R):
                        assert bool(got[r, int(ids[r])]), "the draw lies outside the kept set"
                        if _splits_a_tie(x[r], st):
                            continue
                        compared += 1
                        bad = got[r] != keep[r, j]
                        if bool(bad.any()):
                            lo, hi = _near_cut(x[r], st)
                            assert bool((lo <= got[r]).all() and (got[r] <= hi).all()), (V, r, j, int(bad.sum()))
                            exceptions += int(bad.sum())
                    # the warped row: logits / T where kept
                    want = torch.where(got, x / float(st[0]), -torch.inf)
                    assert torch.equal(scores[0].cpu(), want)
    assert compared >= inputs * (2 * 4 * len(settings) - 12)  # the flat and tied rows under top-p < 1 are the skipped ones
    assert exceptions <= 8 * inputs, exceptions


def test_one_row_and_rows_kernels_draw_alike():
    from spatialrgpt_b200 import ops
    settings, sets, _ = golden()
    V, x, _ = sets[0]
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    for st in settings:
        for r in range(x.shape[0]):
            R = 16
            seeds = torch.tensor(sequence_seeds(r + 5, R), dtype=torch.int64, device=DEV)
            lg = x[r].to(DEV)[None].expand(R, V).contiguous()
            ids = torch.empty(R, dtype=torch.int64, device=DEV)
            ops.sample_rows(lg, _params(st), seeds, step, 0, ids)
            one = []
            for i in range(R):
                out = torch.full((1,), -1, dtype=torch.int64, device=DEV)
                ops.sample_top_p(x[r].to(DEV), _params(st), seeds[i:i + 1], step, 0, out)
                one.append(int(out))
            assert ids.tolist() == one


@pytest.mark.parametrize("st", [(1.0, 0, 1.0, 0.6, 0.0, 0.0), (0.8, 0, 1.0, 1.0, 0.02, 0.0), (1.0, 0, 1.0, 1.0, 0.0, 0.05),
                                (1.1, 40, 0.95, 0.8, 1e-3, 2e-3)])
def test_distribution_of_one_launch_over_many_seeds(st):
    from scipy.stats import chisquare

    from spatialrgpt_b200 import ops
    R, V = 8192, 64
    g = torch.Generator().manual_seed(3)
    row = (torch.randn(V, generator=g) * 1.5).to(torch.bfloat16).float()
    x = row.to(DEV)[None].expand(R, V).contiguous()
    seeds = torch.tensor(sequence_seeds(99, R), dtype=torch.int64, device=DEV)
    ids = torch.empty(R, dtype=torch.int64, device=DEV)
    scores = torch.empty((1, R, V), dtype=torch.float32, device=DEV)
    ops.sample_rows(x, _params(st), seeds, torch.zeros(1, dtype=torch.int32, device=DEV), 0, ids, scores=scores)
    keep = W.kept(row, *st[:1], int(st[1]), *st[2:])
    assert torch.equal(torch.isfinite(scores[0, 0]).cpu(), keep)
    assert 1 < int(keep.sum()) < V
    ref = torch.softmax(torch.where(keep, row.double() / st[0], -torch.inf), 0).numpy()
    draws = ids.cpu().numpy()
    assert np.all(ref[draws] > 0), "a draw outside the kept set"
    counts = np.bincount(draws, minlength=V).astype(np.float64)
    exp = ref * R
    big = exp >= 5
    obs_b, exp_b = np.append(counts[big], counts[~big].sum()), np.append(exp[big], exp[~big].sum())
    if exp_b[-1] == 0:
        obs_b, exp_b = obs_b[:-1], exp_b[:-1]
    assert chisquare(obs_b, exp_b).pvalue > 1e-3


# ---- the decoder -----------------------------------------------------------------------------------------------------------------
LENS = [12, 20, 7]
SMP = dict(temperature=0.9, top_p=0.95, seed=11)
ARMS = [dict(typical_p=0.7), dict(epsilon_cutoff=3e-4), dict(eta_cutoff=2e-3), dict(typical_p=0.9, epsilon_cutoff=1e-4, eta_cutoff=1e-3)]


def _dec(monkeypatch):
    from tests.test_gpu_packed_decode import _decoder
    return _decoder(monkeypatch, True, layers=4)


def _x(lens, H=4096, seed=9):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(sum(lens), H, generator=g) * 0.3).to(torch.bfloat16).to(DEV)


def _split(x, lens):
    return list(torch.split(x, lens))


def _agree(sampled, greedy, kept_counts) -> int:
    """epsilon_cutoff=0.99 keeps only the tokens tied at the row's top logit, so where one token is kept the draw is greedy's choice.
    Walks the steps while the histories agree: a step with one kept token must agree; the first disagreement must come at a step whose
    top is tied (there the draw may pick another of the tied tokens than greedy's lowest index).  Returns the forced steps checked."""
    n = 0
    for t, (a, b) in enumerate(zip(sampled, greedy)):
        if a != b:
            assert kept_counts[t] > 1, (t, a, b)
            break
        n += int(kept_counts[t]) == 1
    return n


def _kept(scores):
    return torch.isfinite(scores).sum(-1).tolist()


def test_epsilon_099_is_greedy_on_every_sampled_path(monkeypatch):
    dec = _dec(monkeypatch)
    x = _x(LENS)
    eps = dict(SMP, epsilon_cutoff=0.99)
    # batch 1
    e0 = _split(x, LENS)[0]
    forced = 0
    s, ex = dec.generate_from_embeds(e0, 12, sampling=eps, output_scores=True)
    forced += _agree(s.tolist(), dec.generate_from_embeds(e0, 12).tolist(), _kept(ex["scores"][:, 0]))
    # a batched sample and num_return_sequences
    g = [o.tolist() for o in dec.generate_batch(x, LENS, 12)]
    s, ex = dec.generate_batch(x, LENS, 12, sampling=eps, output_scores=True)
    for b in range(3):
        forced += _agree(s[b].tolist(), g[b], _kept(ex["scores"][:, b]))
    s, ex = dec.generate_batch(e0, LENS[:1], 12, sampling=eps, num_return_sequences=2, output_scores=True)
    g1 = dec.generate_batch(e0, LENS[:1], 12)[0].tolist()
    for r in range(2):
        forced += _agree(s[r].tolist(), g1, _kept(ex["scores"][:, r]))
    # the batch-invariant rows step: the raw logits tell where the top is unique
    embeds = _split(x, LENS)
    rows, lg = dec.generate_rows(embeds, 12, sampling=eps, seeds=[1, 2, 3], return_logits=True)
    gr = dec.generate_rows(embeds, 12)
    for b in range(3):
        forced += _agree(rows[b].tolist(), gr[b].tolist(), (lg[b] == lg[b].max(-1, keepdim=True).values).sum(-1).tolist())
    assert forced >= 20, forced
    # guidance: sampled with the cut equals guided greedy
    neg = [e[:4] for e in embeds[:2]]
    a = dec.generate_rows(embeds[:2], 10, sampling=eps, seeds=[5, 6], guidance_scale=1.8, negative_embeds=neg)
    b_ = dec.generate_rows(embeds[:2], 10, guidance_scale=1.8, negative_embeds=neg)
    assert [o.tolist()[:5] for o in a] == [o.tolist()[:5] for o in b_]


@pytest.mark.parametrize("arm", range(len(ARMS)))
def test_graph_equals_eager_and_rows_equal_batch_one(monkeypatch, arm):
    dec = _dec(monkeypatch)
    x = _x(LENS)
    smp = dict(SMP, **ARMS[arm])
    e0 = _split(x, LENS)[0]
    a = dec.generate_from_embeds(e0, 12, sampling=smp).tolist()
    assert dec.generate_from_embeds(e0, 12, sampling=smp, use_graph=False).tolist() == a
    assert any(k.warp for k in dec._graphs)
    bg = [o.tolist() for o in dec.generate_batch(x, LENS, 12, sampling=smp)]
    assert [o.tolist() for o in dec.generate_batch(x, LENS, 12, sampling=smp, use_graph=False)] == bg
    embeds = _split(x, LENS)
    seeds = [21, 22, 23]
    rows = [o.tolist() for o in dec.generate_rows(embeds, 12, sampling=smp, seeds=seeds)]
    assert [o.tolist() for o in dec.generate_rows(embeds, 12, sampling=smp, seeds=seeds, use_graph=False)] == rows
    for b in range(3):
        assert rows[b] == dec.generate_from_embeds(embeds[b], 12, sampling=dict(smp, seed=seeds[b])).tolist()
    # the warped row of output_scores marks the tokens a draw can pick, and the sampled ids lie in it
    s, ex = dec.generate_from_embeds(e0, 12, sampling=smp, output_scores=True)
    assert s.tolist() == a
    sc = ex["scores"][:, 0]
    assert all(bool(torch.isfinite(sc[t, s[t]])) for t in range(12))
    assert bool((torch.isfinite(sc).sum(-1) < dec.dims.vocab_size).all())


def test_warpers_off_or_neutral_are_todays_sampler(monkeypatch):
    from spatialrgpt_b200 import ops
    dec = _dec(monkeypatch)
    x = _x(LENS)
    e0 = _split(x, LENS)[0]
    neutral = dict(SMP, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)
    off_range = dict(SMP, typical_p=3.0, epsilon_cutoff=1.0, eta_cutoff=-2.0)

    def run(smp):
        l0 = ops.LAUNCHES
        one, ex = dec.generate_from_embeds(e0, 10, sampling=smp, output_scores=True)
        bt, exb = dec.generate_batch(x, LENS, 10, sampling=smp, output_scores=True)
        rows = dec.generate_rows(_split(x, LENS), 10, sampling=smp, seeds=[1, 2, 3])
        return (one.tolist(), ex["scores"].clone(), [o.tolist() for o in bt], exb["scores"].clone(), [o.tolist() for o in rows],
                ops.LAUNCHES - l0)

    run(SMP)  # captures the graphs (their warm-up launches count too); the score buffer settles at the batch's size
    run(SMP)
    base = run(SMP)
    for smp in (neutral, off_range):
        got = run(smp)
        assert got[0] == base[0] and got[2] == base[2] and got[4] == base[4] and got[5] == base[5]
        assert torch.equal(got[1], base[1]) and torch.equal(got[3], base[3])
    assert not any(k.warp for k in dec._graphs)


def test_typical_p_at_zero_raises_before_device_work(monkeypatch):
    from spatialrgpt_b200 import ops
    dec = _dec(monkeypatch)
    x = _x(LENS)
    for call in (lambda: dec.generate_from_embeds(_split(x, LENS)[0], 4, sampling=dict(SMP, typical_p=0.0)),
                 lambda: dec.generate_rows(_split(x, LENS), 4, sampling=dict(SMP, typical_p=-0.5), seeds=[1, 2, 3])):
        l0 = ops.LAUNCHES
        with pytest.raises(ValueError, match="typical_p"):
            call()
        assert ops.LAUNCHES == l0


def test_generate_epsilon_099_equals_greedy_text_only():
    from tests.test_gpu_guidance import _build, _text
    oc, _, model = _build(torch.bfloat16)
    ids = _text(oc, 2, 9, 4)
    greedy = model.generate(ids, max_new_tokens=8)
    out = model.generate(ids, max_new_tokens=8, do_sample=True, epsilon_cutoff=0.99, seed=3, return_dict_in_generate=True,
                         output_scores=True)
    sc = torch.stack(out.scores)  # [T, B, V]
    forced = sum(_agree(out.sequences[b].tolist()[-8:], greedy[b].tolist()[-8:], _kept(sc[:, b])) for b in range(2))
    assert forced >= 2, forced
