"""Diverse beam search on the CPU: the restatement of transformers 4.37.2's group_beam_search (tests/group_beam_oracle.py) reduced to
plain beam search (pinned to HF by beam_kats.npz / beam_batch_kats.npz), two hand-worked cases, the exports and argument checks of the
new kernels, and generate()'s argument handling with the decoder unreached."""
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import srgpt_oracle as O
from tests.group_beam_oracle import group_beam_generate, group_beam_search
from tests.util import load_npz

L = math.log


def _model(golden_dir, name):
    from tests.golden.make_golden import CASES
    g = load_npz(os.path.join(golden_dir, name))
    oc = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    return g, oc, O.make_weights(oc, seed=int(g["weight_seed"]))


# ---- reductions ---------------------------------------------------------------------------------------------------------------------
def test_one_group_is_plain_beam_search(golden_dir):
    """G = 1 (and any lambda: no earlier group) gives the oracle's beam search, which the beam fixtures pin to HF's generate()."""
    from tests.golden.make_beam_batch_golden import BEAM_BATCH_CASES
    from tests.golden.make_golden import BEAM_CASES
    g, oc, sd = _model(golden_dir, "beam_kats.npz")
    for nb, eos, n_new, lp, es in BEAM_CASES:
        want = O.beam_search_generate(oc, sd["llm"], g["inputs_embeds"], nb, n_new, eos_token_id=eos, length_penalty=lp, early_stopping=es)
        got = group_beam_generate(oc, sd["llm"], g["inputs_embeds"], nb, 1, 0.7, n_new, eos, lp, es)["ids"]
        assert got == want.tolist(), (nb, eos, got, want.tolist())
    g, oc, sd = _model(golden_dir, "beam_batch_kats.npz")
    lens = [int(n) for n in g["seq_lens"]]
    off = np.cumsum([0] + lens)
    for nb, eos, n_new, lp, es in BEAM_BATCH_CASES[1:4]:
        for b in (1, 3):
            emb = g["packed_embeds"][off[b]:off[b + 1]]
            want = O.beam_search_generate(oc, sd["llm"], emb, nb, n_new, eos_token_id=eos, length_penalty=lp, early_stopping=es)
            assert group_beam_generate(oc, sd["llm"], emb, nb, 1, 0.7, n_new, eos, lp, es)["ids"] == want.tolist()


@pytest.mark.parametrize("k,G,eos", [(4, 2, None), (4, 2, [460]), (3, 3, [460]), (6, 3, None)])
def test_a_vanishing_penalty_gives_every_group_plain_beams(golden_dir, k, G, eos):
    """lambda = 1e-30 is below half an ulp of every log-prob, so each group follows beam search with num_beams = k / G: the same beams
    in every step, and the same answer."""
    g, oc, sd = _model(golden_dir, "beam_kats.npz")
    gs, n_new = k // G, 8
    want, trace, _ = O.beam_search_generate(oc, sd["llm"], g["inputs_embeds"], max(gs, 1), n_new, eos_token_id=eos, return_trace=True)
    res = group_beam_generate(oc, sd["llm"], g["inputs_embeds"], k, G, 1e-30, n_new, eos)
    assert res["ids"] == want.tolist()
    for step, nxt in enumerate(trace[:len(res["steps"])]):
        chosen = res["steps"][step]["chosen"]
        for grp in range(G):
            assert [(p - grp * gs, t) for p, t in chosen[grp * gs:(grp + 1) * gs]] == [(b, t) for _, b, t in nxt], (step, grp)


# ---- hand-worked cases ----------------------------------------------------------------------------------------------------------------
P0 = [0.05, 0.1, 0.1, 0.05, 0.2, 0.5]
QB = [0.3, 0.1, 0.2, 0.3, 0.05, 0.05]


def _advance_by_token(rows):
    """The next logits of a beam depend on its last token only: rows[token] (log-probabilities)."""
    return lambda parents, tokens: torch.stack([torch.tensor([L(p) for p in rows[t]]) for t in tokens])


def _check(steps, want):
    for step, (ranked, chosen) in enumerate(want):
        for grp, exp in enumerate(ranked):
            got = steps[step]["ranked"][grp]
            if exp is None:
                assert got is None, (step, grp)
                continue
            assert [(b, t) for _, b, t in got] == [(b, t) for _, b, t in exp], (step, grp, got)
            assert all(abs(s - e) < 1e-5 for (s, _, _), (e, _, _) in zip(got, exp)), (step, grp, got)
        assert steps[step]["chosen"] == chosen, (step, steps[step]["chosen"])


def test_hand_worked_step_tables():
    """V = 6, k = 4, G = 2, lambda = 2: group 1 sees the tokens group 0 chose penalised by lambda per occurrence."""
    p = [0.4, 0.3, 0.1, 0.1, 0.05, 0.05]
    nxt = [0.1, 0.5, 0.2, 0.1, 0.05, 0.05]
    res = group_beam_search(torch.tensor([L(x) for x in p]), _advance_by_token([nxt] * 6), 4, 2, 2.0, 2)
    want = [
        # step 0: group 0 takes tokens 0 and 1 from beam 0; for group 1 they cost 2 each, so 2 and 3 lead
        ([[(L(.4), 0, 0), (L(.3), 0, 1), (L(.1), 0, 2), (L(.1), 0, 3)],
          [(L(.1), 0, 2), (L(.1), 0, 3), (L(.4) - 2, 0, 0), (L(.05), 0, 4)]],
         [(0, 0), (0, 1), (2, 2), (2, 3)]),
        # step 1: group 0 takes token 1 twice, so token 1 costs 4 in group 1
        ([[(L(.4) + L(.5), 0, 1), (L(.3) + L(.5), 1, 1), (L(.4) + L(.2), 0, 2), (L(.3) + L(.2), 1, 2)],
          [(L(.1) + L(.2), 0, 2), (L(.1) + L(.2), 1, 2), (L(.1) + L(.1), 0, 0), (L(.1) + L(.1), 0, 3)]],
         [(0, 1), (1, 1), (2, 2), (3, 2)]),
    ]
    _check(res["steps"], want)
    assert res["ids"] == [0, 1]


def test_a_done_groups_pad_token_penalises_later_groups():
    """Group 0 closes two hypotheses by step 1 and is done; at step 2 it emits pad_token_id 3 for both beams, which costs 2 * lambda in
    group 1, so token 3 (tied with token 0 at the top) drops out.  The answer is the tie of the two groups' EOS-only hypotheses, which
    goes to the later group."""
    rows = [QB, P0, QB, QB, P0, QB]  # tokens 1 and 4 (group 0's) lead to P0, the others to QB
    res = group_beam_search(torch.tensor([L(x) for x in P0]), _advance_by_token(rows), 4, 2, 2.0, 3, eos_token_id=5, pad_token_id=3)
    want = [
        ([[(L(.5), 0, 5), (L(.2), 0, 4), (L(.1), 0, 1), (L(.1), 0, 2)],
          [(L(.5), 0, 5), (L(.1), 0, 2), (L(.05), 0, 0), (L(.05), 0, 3)]],
         [(0, 4), (0, 1), (2, 2), (2, 0)]),
        ([[(L(.2) + L(.5), 0, 5), (L(.1) + L(.5), 1, 5), (L(.2) + L(.2), 0, 4), (L(.2) + L(.1), 0, 1)],
          [(L(.1) + L(.3), 0, 0), (L(.1) + L(.3), 0, 3), (L(.1) + L(.2), 0, 2), (L(.05) + L(.3), 1, 0)]],
         [(0, 4), (0, 1), (2, 0), (2, 3)]),
        ([None,
          [(L(.03) + L(.3), 0, 0), (L(.03) + L(.3), 1, 0), (L(.03) + L(.2), 0, 2), (L(.03) + L(.2), 1, 2)]],
         [(0, 3), (0, 3), (2, 0), (3, 0)]),
    ]
    _check(res["steps"], want)
    assert res["ids"] == [5]


# ---- the kernels' exports and argument checks -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_libraries_export_and_check_arguments(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    x = 16  # a 16-byte aligned non-NULL address: every call below fails its argument check before any launch
    ok = [x, 1000, 1000, 4, 8, x, x, x, x, None]
    for i, v in ((0, None), (4, None), (6, None), (7, None), (8, None), (2, 0), (5, 0), (5, 1001)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_beam_candidates_scored_bf16(*args) == -1, i
    #     logits ldx  V   stats beam cand L  P  k  G  n_cand eos n_eos pad lam done outs...                 stream
    ok = [x, 1000, 1000, x, x, x, 10, 2, 8, 2, 8, x, 1, 0, 1.0, x, x, x, x, x, x, None]
    for i, v in ((0, None), (3, None), (4, None), (5, None), (15, None), (16, None), (20, None), (2, 0), (1, 999), (7, 0), (9, 3),
                 (9, 9), (8, 65), (10, 0), (10, 513), (6, 0), (6, 1001), (11, None), (12, -1), (13, 1000), (13, -1)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_beam_group_select(*args) == -1, i
    args = list(ok)
    args[3] = 12  # stats must be 8-byte aligned (float2)
    assert lib.srgpt_beam_group_select(*args) == -1
    args = list(ok)
    args[8], args[9], args[6] = 64, 2, 4000  # gs * (L + k - gs) = 32 * 4032 > 4096
    args[1] = args[2] = 5000
    assert lib.srgpt_beam_group_select(*args) == -1
    assert "invalid argument" in _lib.last_error()


# ---- generate()'s argument handling --------------------------------------------------------------------------------------------------
def _gen():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2, vocab_size=1000, pad_token_id=0))
    return gen, m


class NoDevice:  # any device work fails the test
    supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_output_scores = True
    supports_batch_invariant = supports_generate_outputs = True

    def generate_beam_batch(self, *a, **k):
        raise AssertionError("reached the decoder")

    def __getattr__(self, name):
        raise AssertionError(f"reached the decoder ({name})")


def test_invalid_group_arguments_raise_value_error_before_device_work():
    gen, m = _gen()
    m.llm = NoDevice()
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    for kw, msg in ((dict(num_beams=4, num_beam_groups=3, diversity_penalty=0.5), "divisible"),
                    (dict(num_beams=2, num_beam_groups=4, diversity_penalty=0.5), "divisible"),
                    (dict(num_beams=1, num_beam_groups=2, diversity_penalty=0.5), "divisible"),
                    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, do_sample=True), "do_sample"),
                    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, do_sample=True, temperature=0.0), "do_sample"),
                    (dict(num_beams=4, num_beam_groups=2), "diversity_penalty > 0"),
                    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.0), "diversity_penalty > 0"),
                    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=-1.0), "diversity_penalty > 0"),
                    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=float("nan")), "diversity_penalty > 0"),
                    (dict(num_beams=4, diversity_penalty=0.5), "num_beam_groups > 1"),
                    (dict(num_beams=4, num_beam_groups=1, diversity_penalty=0.5), "num_beam_groups > 1"),
                    (dict(diversity_penalty=0.5), "num_beam_groups > 1")):
        for b in (1, 2):
            with pytest.raises(ValueError, match=msg):
                gen(m, ids[:b], **kw)


def test_unsupported_options_raise_not_implemented_before_device_work():
    gen, m = _gen()
    m.llm = NoDevice()
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    grp = dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5)
    for kw in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2), dict(output_logits=True),
               dict(return_dict_in_generate=True, output_scores=True), dict(return_dict_in_generate=True, output_hidden_states=True),
               dict(return_dict_in_generate=True, output_attentions=True), dict(prefix_cache=True), dict(prompt_lookup_num_tokens=3),
               dict(guidance_scale=2.0, negative_prompt_ids=ids[:1]), dict(batch_invariant=True), dict(num_return_sequences=2)):
        for b in (1, 2):
            with pytest.raises(NotImplementedError):
                gen(m, ids[:b], **grp, **kw)
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    m.llm = TPLlamaDecoder.__new__(TPLlamaDecoder)
    for b in (1, 2):
        with pytest.raises(NotImplementedError, match="tensor-parallel"):
            gen(m, ids[:b], **grp)


class Recorder:
    """A decoder that records which beam entry point generate() reaches and with what."""
    supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_output_scores = True

    def __init__(self):
        self.calls = []

    def embed_tokens(self, ids):
        return torch.zeros(ids.numel(), 4)

    def generate_beam(self, emb, k, n, **kw):
        self.calls.append(("generate_beam", tuple(emb.shape), k, n, kw))
        return torch.tensor([7, 8])

    def generate_beam_batch(self, packed, lens, k, n, **kw):
        self.calls.append(("generate_beam_batch", tuple(packed.shape), tuple(lens), k, n, kw))
        return [torch.tensor([7, 8]) for _ in lens]


def test_calls_without_the_new_keywords_reach_the_same_entry_points():
    gen, m = _gen()
    m.weights = types.SimpleNamespace(llama=types.SimpleNamespace(embed=torch.zeros(1)))  # the result's device
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    plain_keys = {"eos_token_ids", "stopping_fn", "length_penalty", "early_stopping", "use_graph"}
    runs = {}
    for name, extra in (("plain", {}), ("neutral", dict(num_beam_groups=1, diversity_penalty=0.0)), ("none", dict(num_beam_groups=None)),
                        ("group", dict(num_beam_groups=2, diversity_penalty=0.5, pad_token_id=9))):
        m.llm = Recorder()
        for b in (1, 2):
            gen(m, ids[:b], num_beams=4, max_new_tokens=5, length_penalty=0.5, **extra)
        runs[name] = m.llm.calls
    assert [c[0] for c in runs["plain"]] == ["generate_beam", "generate_beam_batch"]
    assert set(runs["plain"][0][-1]) == plain_keys and set(runs["plain"][1][-1]) == plain_keys
    assert runs["plain"][0][1:-1] == ((3, 4), 4, 5) and runs["plain"][1][1:-1] == ((6, 4), (3, 3), 4, 5)
    for name in ("neutral", "none"):
        assert [c[:-1] for c in runs[name]] == [c[:-1] for c in runs["plain"]]
        assert [{k: v for k, v in c[-1].items() if k != "stopping_fn"} for c in runs[name]] == \
               [{k: v for k, v in c[-1].items() if k != "stopping_fn"} for c in runs["plain"]]
    # group mode: batch 1 runs the batched step too, with the group keywords
    assert [c[0] for c in runs["group"]] == ["generate_beam_batch", "generate_beam_batch"]
    assert runs["group"][0][1:-1] == ((3, 4), (3,), 4, 5)
    for c in runs["group"]:
        assert set(c[-1]) == plain_keys | {"num_beam_groups", "diversity_penalty", "pad_token_id"}
        assert (c[-1]["num_beam_groups"], c[-1]["diversity_penalty"], c[-1]["pad_token_id"]) == (2, 0.5, 9)
