"""Per-step scores on the H100 (generate(return_dict_in_generate=True, output_scores=True)): ids with the flags are bit-identical to
ids without them on every path, graph and eager steps give bit-identical scores, greedy rows are the rows the arg max picked from (the
output_logits rows without processors), sampled rows are HF's temperature / top-k / top-p warpers over the processed rows, beam rows
sum to sequences_scores, and generate() reproduces HF's generate() / compute_transition_scores (tests/golden/output_scores_kats.npz,
made by ``make_output_scores_golden.py``).  Both element types."""
import os

import pytest
import torch

from tests.golden.make_golden import CASES
from tests.golden.make_output_scores_golden import SCORE_CASES
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
TOL = {torch.bfloat16: 0.08, torch.float16: 0.02}  # score tolerance against the fp32 golden
SMP = dict(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, seed=5)
_MODELS = {}


def _model(dtype):
    if dtype not in _MODELS:
        from tests.test_gpu_fp16 import build_model
        g = load_npz(os.path.join(os.path.dirname(__file__), "golden", "output_scores_kats.npz"))
        _MODELS[dtype] = (g, build_model(CASES["tiny_masks_gqa"][0], int(g["weight_seed"]), dtype=dtype)[2])
    return _MODELS[dtype]


def _gen(model, ids, **kw):
    return model.generate(input_ids=ids.to(DEV), eos_token_id=kw.pop("eos_token_id", None), **kw)


def _scores(model, ids, **kw):
    out = _gen(model, ids, return_dict_in_generate=True, output_scores=True, **kw)
    return out, torch.stack(out.scores)  # [steps, rows, V]


def _prompts(g, n):
    return torch.as_tensor(g["input_ids"][:n])


def _argmax_is_token(sc, seqs, lens=None):
    for t in range(sc.shape[0]):
        for r in range(sc.shape[1]):
            if lens is None or t < lens[r]:
                assert int(sc[t, r].argmax()) == int(seqs[r, t]), (t, r)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch1_greedy_rows_are_the_output_logits_rows(dtype):
    g, model = _model(dtype)
    ids = _prompts(g, 1)
    plain = _gen(model, ids, max_new_tokens=10)
    out, sc = _scores(model, ids, max_new_tokens=10)
    assert torch.equal(out.sequences, plain) and sc.dtype == torch.float32 and sc.shape[:2] == (10, 1)
    _argmax_is_token(sc, out.sequences)
    _, logits = _gen(model, ids, max_new_tokens=10, output_logits=True)
    assert torch.equal(sc[:, 0], logits[0])
    _, eager = _scores(model, ids, max_new_tokens=10, use_cuda_graph=False)
    assert torch.equal(sc, eager)
    both = _gen(model, ids, max_new_tokens=10, return_dict_in_generate=True, output_scores=True, output_logits=True)
    assert torch.equal(torch.stack(both.scores), sc) and torch.equal(both.logits[0], logits[0])


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch1_processors_prefix_cache_and_prompt_lookup(dtype):
    g, model = _model(dtype)
    ids = _prompts(g, 1)
    proc = dict(repetition_penalty=1.3, no_repeat_ngram_size=2)
    plain = _gen(model, ids, max_new_tokens=12, **proc)
    out, sc = _scores(model, ids, max_new_tokens=12, **proc)
    assert torch.equal(out.sequences, plain)
    _argmax_is_token(sc, out.sequences)
    _, raw = _gen(model, ids, max_new_tokens=12, output_logits=True, **proc)
    assert not torch.equal(sc[:, 0], raw[0])  # the processors acted on the rows
    _, eager = _scores(model, ids, max_new_tokens=12, use_cuda_graph=False, **proc)
    assert torch.equal(sc, eager)
    # prefix_cache: the second turn reuses the first's prompt rows
    _gen(model, ids, max_new_tokens=4, prefix_cache=True)
    longer = torch.cat([ids, ids[:, :5]], 1)
    plain = _gen(model, longer, max_new_tokens=8, prefix_cache=True)
    _gen(model, ids, max_new_tokens=4, prefix_cache=True)
    out, sc = _scores(model, longer, max_new_tokens=8, prefix_cache=True)
    assert torch.equal(out.sequences, plain) and model.last_prefix_reuse[0] > 0
    _argmax_is_token(sc, out.sequences)
    # prompt lookup: the scores are the verify passes' raw rows
    rep = torch.cat([ids, ids], 1)
    plain = _gen(model, rep, max_new_tokens=16, prompt_lookup_num_tokens=4)
    out, sc = _scores(model, rep, max_new_tokens=16, prompt_lookup_num_tokens=4)
    assert torch.equal(out.sequences, plain)
    _, logits = _gen(model, rep, max_new_tokens=16, output_logits=True)
    assert torch.equal(sc[:, 0], logits[0])


def hf_warp(rows: torch.Tensor, temperature: float, top_k: int, top_p: float):
    """transformers' TemperatureLogitsWarper, TopKLogitsWarper and TopPLogitsWarper on fp32 CPU rows [R, V], and per row whether the
    kept set may differ from the kernel's as DESIGN.md §7 allows: a cumulative mass within 1e-4 of top_p, or tokens of equal score that
    HF's sort splits at the nucleus cut (the kernel keeps every tied token).  The top-k set is exact: no exemption."""
    from transformers.generation import logits_process as lp
    x = rows.float().cpu()
    x = lp.TemperatureLogitsWarper(temperature)(None, x)
    x = lp.TopKLogitsWarper(top_k)(None, x)
    x = lp.TopPLogitsWarper(top_p)(None, x)
    t = rows.float().cpu() / temperature
    srt = t.sort(-1, descending=True).values
    p = torch.softmax(srt[:, :top_k], -1)
    cum = p.cumsum(-1)
    near_p = ((cum - top_p).abs() < 1e-4).any(-1)
    # a tie (equal scores, frequent in 16-bit rows) across the cut HF's sort made: the kernel keeps every tied token
    n = torch.isfinite(x).sum(-1).clamp(max=srt.shape[-1] - 1)
    split = srt.gather(-1, (n - 1)[:, None])[:, 0] == srt.gather(-1, n[:, None])[:, 0]
    return x, near_p | split


def _check_warped(sc, raw_rows, seqs, lens=None):
    """sc [steps, rows, V] against HF's warpers over raw_rows [steps, rows, V]; every drawn token has a finite score."""
    checked = total = 0
    for t in range(sc.shape[0]):
        ref, near = hf_warp(raw_rows[t], SMP["temperature"], SMP["top_k"], SMP["top_p"])
        got = sc[t].cpu()
        for r in range(sc.shape[1]):
            if lens is not None and t >= lens[r]:
                continue
            total += 1
            assert torch.isfinite(got[r, int(seqs[r, t])]), (t, r)
            if near[r]:
                continue
            checked += 1
            fin, gfin = torch.isfinite(ref[r]), torch.isfinite(got[r])
            assert torch.equal(fin, gfin), (t, r, (fin ^ gfin).nonzero().flatten().tolist(), int(fin.sum()), int(gfin.sum()))
            assert torch.equal(got[r][fin], ref[r][fin]), (t, r)
    assert checked >= total // 2, (checked, total)


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch1_sampled_rows_are_hf_warped_rows(dtype):
    g, model = _model(dtype)
    ids = _prompts(g, 1)
    plain = _gen(model, ids, max_new_tokens=12, **SMP)
    out, sc = _scores(model, ids, max_new_tokens=12, **SMP)
    assert torch.equal(out.sequences, plain)
    _, raw = _gen(model, ids, max_new_tokens=12, output_logits=True, **SMP)
    _check_warped(sc, raw[0][:, None], out.sequences)
    _, eager = _scores(model, ids, max_new_tokens=12, use_cuda_graph=False, **SMP)
    assert torch.equal(sc, eager)
    proc = dict(repetition_penalty=1.3)
    plain = _gen(model, ids, max_new_tokens=12, **proc, **SMP)
    out, sc = _scores(model, ids, max_new_tokens=12, **proc, **SMP)
    assert torch.equal(out.sequences, plain) and all(torch.isfinite(sc[t, 0, int(out.sequences[0, t])]) for t in range(12))


@pytest.mark.parametrize("dtype", DTYPES)
def test_batched_greedy_sampled_and_num_return_sequences(dtype):
    g, model = _model(dtype)
    ids = torch.cat([_prompts(g, 2), _prompts(g, 2).flip(1)], 0)  # 4 prompts of one length
    eos = int(_gen(model, ids[1:2], max_new_tokens=4)[0, 3])  # prompt 1 stops early
    plain = _gen(model, ids, max_new_tokens=10, eos_token_id=eos)
    out, sc = _scores(model, ids, max_new_tokens=10, eos_token_id=eos)
    assert torch.equal(out.sequences, plain) and sc.shape[:2] == (10, 4)
    lens = [row.tolist().index(eos) + 1 if eos in row.tolist() else 10 for row in out.sequences.cpu()]
    assert min(lens) < 10
    _argmax_is_token(sc, out.sequences, lens)
    _, eager = _scores(model, ids, max_new_tokens=10, eos_token_id=eos, use_cuda_graph=False)
    assert torch.equal(sc, eager)
    proc = dict(no_repeat_ngram_size=2)
    plain = _gen(model, ids, max_new_tokens=10, **proc)
    out, sc = _scores(model, ids, max_new_tokens=10, **proc)
    assert torch.equal(out.sequences, plain)
    _argmax_is_token(sc, out.sequences)
    # sampled: the batched rows are HF's warpers over the bf16 / fp16 lm_head rows widened
    plain = _gen(model, ids, max_new_tokens=10, **SMP)
    out, sc = _scores(model, ids, max_new_tokens=10, **SMP)
    assert torch.equal(out.sequences, plain)
    _, eager = _scores(model, ids, max_new_tokens=10, use_cuda_graph=False, **SMP)
    assert torch.equal(sc, eager)
    assert all(torch.isfinite(sc[t, r, int(out.sequences[r, t])]) for t in range(10) for r in range(4))
    kept = torch.isfinite(sc).sum(-1)
    assert int(kept.min()) >= 1 and int(kept.max()) <= SMP["top_k"]  # the top-k cut and the nucleus left -inf elsewhere
    plain = _gen(model, ids[:2], max_new_tokens=8, num_return_sequences=3, **SMP)
    out, sc = _scores(model, ids[:2], max_new_tokens=8, num_return_sequences=3, **SMP)
    assert torch.equal(out.sequences, plain) and sc.shape[:2] == (8, 6)
    assert all(torch.isfinite(sc[t, r, int(out.sequences[r, t])]) for t in range(8) for r in range(6))


@pytest.mark.parametrize("dtype", DTYPES)
def test_beam_scores_sum_to_sequences_scores(dtype):
    g, model = _model(dtype)
    for n, lp in ((1, 1.0), (2, 0.7)):
        ids = _prompts(g, n)
        plain = _gen(model, ids, max_new_tokens=8, num_beams=3, length_penalty=lp)
        out, sc = _scores(model, ids, max_new_tokens=8, num_beams=3, length_penalty=lp)
        assert torch.equal(out.sequences, plain) and sc.shape[1] == 3 * n
        assert torch.allclose(torch.logsumexp(sc, -1), torch.zeros(()), atol=1e-4)
        tr = model.compute_transition_scores(out.sequences, out.scores, out.beam_indices)
        L = (out.beam_indices >= 0).sum(-1)
        assert torch.allclose(tr.sum(-1) / L.float() ** lp, out.sequences_scores, rtol=1e-5, atol=1e-5)
        _, eager = _scores(model, ids, max_new_tokens=8, num_beams=3, length_penalty=lp, use_cuda_graph=False)
        assert torch.equal(sc, eager)


@pytest.mark.parametrize("dtype", DTYPES)
def test_against_hf_generate(dtype):
    g, model = _model(dtype)
    tol = TOL[dtype]
    for name, n, kw in SCORE_CASES:
        out = _gen(model, _prompts(g, n), return_dict_in_generate=True, output_scores=True, **kw)
        ref_ids, ref_sc, margin = g[f"{name}__ids"], g[f"{name}__scores"], g[f"{name}__margin"]
        sc = torch.stack(out.scores).cpu()
        # the first step reads the same prompt rows; later steps are compared up to the first one whose top-2 margin does not clear
        # the tolerance (from there on the two may follow different tokens)
        assert torch.allclose(sc[0], torch.as_tensor(ref_sc[0]), atol=tol, rtol=0), name
        clear = [bool((margin[t] > 2 * tol).all()) for t in range(margin.shape[0])]
        steps = clear.index(False) if False in clear else len(clear)
        print(f"{name} {dtype}: {steps} of {len(clear)} steps clear the tolerance")
        assert torch.allclose(sc[:steps], torch.as_tensor(ref_sc[:steps]), atol=tol, rtol=0), name
        if "num_beams" in kw:
            if steps == len(clear):
                assert out.sequences.cpu().tolist() == ref_ids.tolist(), name
                assert out.beam_indices.cpu().tolist() == g[f"{name}__beam_indices"].tolist(), name
                assert torch.allclose(out.sequences_scores.cpu(), torch.as_tensor(g[f"{name}__sequences_scores"]), atol=tol), name
                tr = model.compute_transition_scores(out.sequences, out.scores, out.beam_indices).cpu()
                assert torch.allclose(tr, torch.as_tensor(g[f"{name}__transition"]), atol=tol), name
        else:
            assert out.sequences.cpu()[:, :steps].tolist() == ref_ids[:, :steps].tolist(), name
        if "num_beams" not in kw and steps == len(clear):
            tr = model.compute_transition_scores(out.sequences, out.scores).cpu()
            assert torch.allclose(tr, torch.as_tensor(g[f"{name}__transition"]), atol=tol), name
