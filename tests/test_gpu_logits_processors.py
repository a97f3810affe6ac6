"""HF's logits processors on the H100: the processing kernel bit for bit against transformers' processors on the same CUDA fp32 rows,
the one-token decoder (eager, graph, sampling; packed and bf16 steps) and the batched greedy path against the rule "every token is the
arg max of the processed logits of its step", generate() against HF generate() (tests/golden/processor_kats.npz, made by
``make_processor_golden.py``), and neutral values leaving everything unchanged."""
import os

import numpy as np
import pytest
import torch

from spatialrgpt_b200 import logits_processors as LP
from tests.golden.make_golden import CASES
from tests.golden.make_processor_golden import PROCESSOR_CASES, PROCESSOR_NEW_TOKENS
from tests.test_gpu_packed_decode import _decoder
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"


def hf_process(rows: torch.Tensor, hist: torch.Tensor, spec: dict) -> torch.Tensor:
    """transformers' processors, in _get_logits_processor's order, on CUDA fp32 rows [R, V] with input_ids = hist [R, n]."""
    from transformers.generation import logits_process as lp
    x = rows.float().clone()
    ids = hist.to(DEV, torch.long)
    eos = spec.get("eos_token_ids") or []
    procs = []
    if "repetition_penalty" in spec:
        procs.append(lp.RepetitionPenaltyLogitsProcessor(float(spec["repetition_penalty"])))
    if "no_repeat_ngram_size" in spec:
        procs.append(lp.NoRepeatNGramLogitsProcessor(int(spec["no_repeat_ngram_size"])))
    if spec.get("bad_words_ids"):
        procs.append(lp.NoBadWordsLogitsProcessor(spec["bad_words_ids"], eos_token_id=eos or None))
    if spec.get("min_new_tokens", 0) > 0 and eos:
        procs.append(lp.MinLengthLogitsProcessor(spec["min_new_tokens"], eos, device=DEV))
        procs.append(lp.MinNewTokensLengthLogitsProcessor(0, spec["min_new_tokens"], eos, device=DEV))
    for p in procs:
        x = p(ids, x)
    return x


def _set(ops, spec):
    f, ints = LP.encode(spec)
    return torch.from_numpy(f).to(DEV), torch.from_numpy(ints).to(DEV)


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_cuda_division_by_a_scalar_is_a_reciprocal_multiply():
    """The rule the kernel implements for score / penalty: on a CUDA tensor ATen multiplies by fp32(1 / penalty), the reciprocal taken in
    double (1.1, 1.7 and 1.15 are penalties where it differs from the reciprocal of fp32(penalty))."""
    x = torch.linspace(0.01, 50, 200000, device=DEV)
    for p in (1.1, 1.3, 0.7, 1.7, 1.15):
        inv = float(LP.encode({"repetition_penalty": p})[0][1])
        assert torch.equal(x / p, x * torch.tensor(inv, device=DEV)), p
        assert not torch.equal((x.cpu() / p), x.cpu() * inv)  # CPU torch divides: the two rules differ on these values


def _case(R, V, n, seed):
    g = torch.Generator().manual_seed(seed)
    hist = torch.randint(0, 40, (R, n), generator=g)
    if n > 8:
        hist[:, -3:] = hist[:, 2:5]                              # a planted 3-gram repeat
        hist[:, n // 2] = V - 1 - torch.arange(R) % 7            # tokens in the last segment
        hist[:, n // 3] = torch.randint(0, V, (R,), generator=g)  # and anywhere
    rows = torch.randn(R, V, generator=g) * 3
    rows[:, 1:8:3] = 0.0
    rows[:, 2:9:3] = -0.0
    rows[:, 40] = rows[:, 41] = rows.max() + 1  # a planted arg max tie (lowest index wins)
    rows[:, V - 2] = rows[:, 40]                 # ... across segments
    return rows, hist


def _last(h, row, k):
    return int(h[row, -k]) if h.shape[1] >= k else 1


SPECS = {
    "all": lambda h, V: dict(repetition_penalty=1.3, no_repeat_ngram_size=3, eos_token_ids=[V - 1, 7], min_new_tokens=h.shape[1] + 1,
                             bad_words_ids=[[5], [_last(h, 0, 1), 9], [_last(h, 0, 2), _last(h, 0, 1), 11], [3, 4, 5, 6] * 2000, [V - 3]]),
    "penalty_below_1": lambda h, V: dict(repetition_penalty=0.7),
    "penalty_1_1": lambda h, V: dict(repetition_penalty=1.1),
    "ngram1_eos_off": lambda h, V: dict(no_repeat_ngram_size=1, eos_token_ids=[40], min_new_tokens=h.shape[1]),
    "ngram5_bad": lambda h, V: dict(no_repeat_ngram_size=5, bad_words_ids=[[40], [_last(h, -1, 1), 41]]),
}


@pytest.mark.parametrize("R,V", [(1, 128259), (3, 128259), (32, 128259), (3, 1003)])
@pytest.mark.parametrize("elem", ["f32", "bf16"])
@pytest.mark.parametrize("n", [0, 1, 40, 4096])
def test_kernel_matches_transformers_bit_for_bit(R, V, elem, n):
    from spatialrgpt_b200 import ops
    if n == 4096 and R == 32 and elem == "f32":
        pytest.skip("covered by the bf16 rows")
    rows, hist = _case(R, V, n, R * 7 + n)
    x = rows.to(DEV, torch.float32 if elem == "f32" else torch.bfloat16)
    if elem == "bf16":  # the batched lm_head's rows: 16-byte aligned row stride
        buf = torch.zeros(R, (V + 7) // 8 * 8, dtype=torch.bfloat16, device=DEV)
        buf[:, :V].copy_(x)
        x = buf[:, :V]
    hist_dev = hist.t().contiguous().view(-1).to(DEV)  # the batched step's [t, b] table
    step = torch.tensor([n], dtype=torch.int32, device=DEV)
    for name, mk in SPECS.items():
        spec = mk(hist, V)
        f, ints = _set(ops, spec)
        out = torch.empty(R, V, dtype=torch.float32, device=DEV)
        ids = torch.empty(R, dtype=torch.int64, device=DEV)
        ops.logits_process(x, hist_dev if n else None, 1, R, step, 0, f, ints, out=out, ids=ids)
        ref = hf_process(x, hist, spec)
        assert torch.equal(_bits(out), _bits(ref)), (name, (out != ref).nonzero()[:5].tolist())
        assert torch.equal(ids, torch.argmax(ref, -1)), name
        ids2 = torch.empty(R, dtype=torch.int64, device=DEV)
        ops.logits_process(x, hist_dev if n else None, 1, R, step, 0, f, ints, ids=ids2)  # without the rows
        assert torch.equal(ids2, ids)
    if R == 1 and n:  # the one-token layout: stride 1 over out_ids, count = *step - 1
        spec = SPECS["all"](hist, V)
        f, ints = _set(ops, spec)
        out_ids = torch.zeros(n + 5, dtype=torch.int64, device=DEV)
        out_ids[:n] = hist[0].to(DEV)
        out = torch.empty(1, V, dtype=torch.float32, device=DEV)
        ops.logits_process(x, out_ids, 0, 1, step + 1, -1, f, ints, out=out)
        assert torch.equal(_bits(out), _bits(hf_process(x, hist, spec)))


def test_pick_token_writes_the_choice_and_its_embedding():
    from spatialrgpt_b200 import ops
    emb = torch.randn(50, 64, device=DEV).to(torch.bfloat16)
    out_ids = torch.zeros(8, dtype=torch.int64, device=DEV)
    step = torch.tensor([3], dtype=torch.int32, device=DEV)
    nx = torch.zeros(64, dtype=torch.bfloat16, device=DEV)
    ops.logits_pick_token(torch.tensor([17], device=DEV), step, -1, out_ids, emb, nx)
    assert out_ids.tolist() == [0, 0, 17, 0, 0, 0, 0, 0] and torch.equal(nx, emb[17])


# ---- the decoder -----------------------------------------------------------------------------------------------------------------
SPEC = dict(repetition_penalty=1.15, no_repeat_ngram_size=2, min_new_tokens=6, eos_token_ids=[128009])


def _check_rule(ids, logits, spec):
    """every token = arg max of HF's processors over the raw logits of its step and the tokens before it."""
    ids = ids.tolist()
    for k in range(len(ids)):
        ref = hf_process(logits[k:k + 1], torch.tensor([ids[:k]], dtype=torch.long), spec)
        assert int(torch.argmax(ref, -1)) == ids[k], k


@pytest.mark.parametrize("pack", [True, False])
def test_one_token_decoder(monkeypatch, pack):
    from spatialrgpt_b200 import ops
    dec = _decoder(monkeypatch, pack)
    x = (torch.randn(20, 4096, generator=torch.Generator().manual_seed(5)) * 0.3).to(torch.bfloat16).to(DEV)
    plain, raw0 = dec.generate_from_embeds(x, 40, use_graph=False, return_logits=True)
    spec = dict(SPEC, bad_words_ids=[[int(plain[3])], [int(plain[0]), int(plain[1])]])
    ids, raw = dec.generate_from_embeds(x, 40, use_graph=False, return_logits=True, processors=spec)
    assert not torch.equal(ids, plain)
    assert torch.equal(raw[0], raw0[0])  # output_logits stays raw
    _check_rule(ids, raw, spec)
    g = dec.generate_from_embeds(x, 40, processors=spec)  # captures the graph
    assert torch.equal(g, ids)
    assert torch.equal(dec.generate_from_embeds(x, 40), plain)  # captures the plain graph, which stays as it was
    l0 = ops.LAUNCHES
    dec.generate_from_embeds(x, 40)
    l1 = ops.LAUNCHES
    assert torch.equal(dec.generate_from_embeds(x, 40, processors=spec), ids)
    assert ops.LAUNCHES - l1 == l1 - l0 + 40 * 3  # processing, key unpack and pick per token (the first one eager)
    # sampling: reproducible, graph == eager, top-k support of the processed logits, banned tokens never drawn
    smp = dict(temperature=0.9, top_k=5, seed=11)
    s1 = dec.generate_from_embeds(x, 30, sampling=smp, processors=spec)
    s2 = dec.generate_from_embeds(x, 30, sampling=smp, processors=spec)
    se, sraw = dec.generate_from_embeds(x, 30, sampling=smp, processors=spec, use_graph=False, return_logits=True)
    assert torch.equal(s1, s2) and torch.equal(s1, se)
    toks = se.tolist()
    for k in range(len(toks)):
        ref = hf_process(sraw[k:k + 1], torch.tensor([toks[:k]], dtype=torch.long), spec)[0]
        assert float(ref[toks[k]]) >= float(ref.topk(5).values[-1]), k
        assert torch.isfinite(ref[toks[k]]), k


def test_batched_greedy_path(monkeypatch):
    from spatialrgpt_b200 import ops
    dec = _decoder(monkeypatch, True)
    g = torch.Generator().manual_seed(9)
    lens = [12, 20, 7]
    x = (torch.randn(sum(lens), 4096, generator=g) * 0.3).to(torch.bfloat16).to(DEV)
    plain = dec.generate_batch(x, lens, 24)
    spec = dict(SPEC, bad_words_ids=[[int(plain[0][2])], [int(plain[1][0]), int(plain[1][1])], [7, 9]])
    calls = []
    real = ops.logits_process

    def spy(logits, hist, rs, ts, step, off, *a, **k):
        n = (int(step) if step is not None else 0) + off
        h = None if hist is None else hist[: n * ts].view(n, ts).t().clone() if n else torch.zeros(logits.shape[0], 0, dtype=torch.long)
        real(logits, hist, rs, ts, step, off, *a, **k)
        calls.append((logits.float().clone(), h, k["ids"].clone()))

    monkeypatch.setattr(ops, "logits_process", spy)
    eager = dec.generate_batch(x, lens, 24, use_graph=False, processors=spec)
    monkeypatch.setattr(ops, "logits_process", real)
    assert len(calls) == 24  # the first tokens, then every step
    for lg, h, ids in calls:
        hh = torch.zeros(lg.shape[0], 0, dtype=torch.long) if h is None else h
        assert torch.equal(ids, torch.argmax(hf_process(lg, hh, spec), -1))
    graph = dec.generate_batch(x, lens, 24, processors=spec)
    assert all(torch.equal(a, b) for a, b in zip(eager, graph))
    one = dec.generate_batch(x, lens, 1, processors=spec)
    assert [o.tolist() for o in one] == [e[:1].tolist() for e in eager]
    assert any(not torch.equal(a, b) for a, b in zip(plain, graph))
    # the sequential path (output_logits): every token of every sequence obeys the rule against its own logits and history
    seq, lgs = dec.generate_batch(x, lens, 10, return_logits=True, processors=spec)
    for ids, lg in zip(seq, lgs):
        _check_rule(ids, lg, spec)
    smp = dict(temperature=0.8, top_k=4, seed=3)
    a = dec.generate_batch(x, lens, 10, sampling=smp, processors=spec)
    b = dec.generate_batch(x, lens, 10, sampling=smp, processors=spec, use_graph=False)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


# ---- generate() ------------------------------------------------------------------------------------------------------------------
def _model(dtype):
    from tests.test_gpu_fp16 import build_model
    g = load_npz(os.path.join(os.path.dirname(__file__), "golden", "processor_kats.npz"))
    oc, sd, model = build_model(CASES["tiny_masks_gqa"][0], int(g["weight_seed"]), dtype=dtype)
    return g, oc, sd, model


def _kwargs(g, name, kw):
    kw = dict(kw)
    kw.pop("eos", None)
    eos = int(g[f"{name}__eos"])
    if kw.get("bad_words_ids") == "plain":
        b = g[f"{name}__bad"].tolist()
        n, toks = b[:3], b[3:]
        kw["bad_words_ids"] = [toks[sum(n[:i]):sum(n[:i + 1])] for i in range(3)]
    return dict(kw, eos_token_id=None if eos < 0 else eos)


@pytest.mark.parametrize("dtype,tol,need", [(torch.float16, 0.02, 40), (torch.bfloat16, 0.08, 30)])
def test_generate_reproduces_hf_generate(dtype, tol, need):
    g, oc, sd, model = _model(dtype)
    ids = g["input_ids"][None].to(DEV)
    checked = 0
    for name, kw in PROCESSOR_CASES:
        kwargs = _kwargs(g, name, kw)
        ref, margin = g[f"{name}__ids"].tolist(), g[f"{name}__margin"].tolist()
        out = model.generate(ids, do_sample=False, max_new_tokens=PROCESSOR_NEW_TOKENS, **kwargs)[0].tolist()
        eager = model.generate(ids, do_sample=False, max_new_tokens=PROCESSOR_NEW_TOKENS, use_cuda_graph=False, **kwargs)[0].tolist()
        assert out == eager, name
        safe = next((k for k, m in enumerate(margin) if m < tol), len(margin))  # tokens after a near tie may follow either branch
        assert out[:safe] == ref[:safe], (name, out, ref, safe)
        checked += safe
    assert checked >= need, checked
    # min_length maps through the prompt length exactly as min_new_tokens
    a = model.generate(ids, max_new_tokens=8, min_length=27, eos_token_id=int(g["all__eos"]))[0].tolist()
    b = model.generate(ids, max_new_tokens=8, min_new_tokens=7, eos_token_id=int(g["all__eos"]))[0].tolist()
    assert a == b


def test_neutral_values_change_nothing():
    from spatialrgpt_b200 import ops
    g, oc, sd, model = _model(torch.bfloat16)
    ids = g["input_ids"][None].to(DEV)
    neutral = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)
    for graph in (True, False):
        model.generate(ids, max_new_tokens=12, use_cuda_graph=graph)  # warm-up (graph capture)
        l0 = ops.LAUNCHES
        a, la = model.generate(ids, max_new_tokens=12, use_cuda_graph=graph, output_logits=True)
        l1 = ops.LAUNCHES
        b, lb = model.generate(ids, max_new_tokens=12, use_cuda_graph=graph, output_logits=True, **neutral)
        l2 = ops.LAUNCHES
        assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(la, lb)) and l1 - l0 == l2 - l1
        c = model.generate(ids, max_new_tokens=12, use_cuda_graph=graph)
        l3 = ops.LAUNCHES
        d = model.generate(ids, max_new_tokens=12, use_cuda_graph=graph, **neutral)
        assert torch.equal(c, d) and ops.LAUNCHES - l3 == l3 - l2


def test_multimodal_prefix_cache_and_stopping_with_processors(golden_dir):
    from oracle import srgpt_oracle as O
    from tests.test_gpu_fp16 import build_model
    name = "tiny_masks_gqa"
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    gz = load_npz(os.path.join(golden_dir, name + ".npz"))
    oc, sd, model = build_model(kw, int(gz["weight_seed"]), dtype=torch.bfloat16)
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    args = dict(images=images.to(DEV, torch.bfloat16), depths=depths.to(DEV, torch.bfloat16), masks=[m.to(DEV, torch.bfloat16) for m in masks])
    spec = dict(repetition_penalty=1.4, no_repeat_ngram_size=2)
    ids, lg = model.generate(input_ids.to(DEV), max_new_tokens=12, output_logits=True, eos_token_id=None, **args, **spec)
    _check_rule(ids[0], lg[0], spec)
    assert torch.equal(model.generate(input_ids.to(DEV), max_new_tokens=12, eos_token_id=None, **args, **spec), ids)
    # a prefix-cached follow-up: the processors act at decode time only
    model.generate(input_ids.to(DEV), max_new_tokens=4, eos_token_id=None, prefix_cache=True, **args)
    follow = torch.cat([input_ids, input_ids[:, -5:]], 1).to(DEV)
    f_ids, f_lg = model.generate(follow, max_new_tokens=10, output_logits=True, eos_token_id=None, prefix_cache=True, **args, **spec)
    assert model.last_prefix_reuse[0] > 0
    _check_rule(f_ids[0], f_lg[0], spec)
    # EOS below the minimum length is never chosen; the first EOS after it ends the answer; a stopping criterion cuts as usual
    plain = model.generate(input_ids.to(DEV), max_new_tokens=12, eos_token_id=None, **args)[0].tolist()
    eos = plain[2]
    cut = model.generate(input_ids.to(DEV), max_new_tokens=12, eos_token_id=eos, min_new_tokens=5, **args)[0].tolist()
    assert eos not in cut[:5] and (eos not in cut or cut.index(eos) == len(cut) - 1)

    class StopAfter4:
        def __call__(self, output_ids, scores=None, **k):
            return output_ids.shape[1] >= 4

    short = model.generate(input_ids.to(DEV), max_new_tokens=12, eos_token_id=None, stopping_criteria=[StopAfter4()], **args, **spec)[0]
    assert short.tolist() == ids[0, :4].tolist()
