"""Contrastive search on the CPU: the oracle's restatement (tests/contrastive_oracle.py) pinned to the 4.37.2 loop over HF's stock
LlamaForCausalLM (tests/golden/contrastive_kats.npz), generate()'s mode rule and refusals against host-only stand-in decoders, the host
argument checks of the C entry points and the kernels' resource usage."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests.test_batch_invariant_cpu import TWO, HostDecoder, _model

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "contrastive_kats.npz")


def fixture_cases(k):
    return sorted({n.split("__")[0] for n in k.files if "__" in n})


# ---- the oracle against HF ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hf_model():
    from oracle import srgpt_oracle as O
    from tests.golden.make_cfg_golden import BEAM_WEIGHT_SEED
    from tests.golden.make_golden import CASES as MODEL_CASES
    k = np.load(GOLDEN)
    cfg = O.OracleConfig(**MODEL_CASES["tiny_masks_gqa"][0])
    return cfg, O.make_weights(cfg, seed=BEAM_WEIGHT_SEED), k


def test_fixture_covers_the_cases():
    k = np.load(GOLDEN)
    names = fixture_cases(k)
    assert len(names) == 12
    assert {(int(k[f"{n}__k"]), float(k[f"{n}__alpha"])) for n in names} == {(2, 0.3), (4, 0.6), (6, 0.9)}
    assert any(k[f"{n}__input_ids"].shape[0] == 2 for n in names) and any(k[f"{n}__input_ids"].shape[1] > 64 for n in names)
    eos = [n for n in names if int(k[f"{n}__eos"]) >= 0]
    assert eos and all(int(k[f"{n}__ids0"][-1]) == int(k[f"{n}__eos"]) and len(k[f"{n}__ids0"]) < int(k["max_new"]) for n in eos)


@pytest.mark.parametrize("name", fixture_cases(np.load(GOLDEN)))
def test_oracle_equals_hf_contrastive_search(hf_model, name):
    """Ids exact; the top-k probabilities, penalties and scores of every step within fp32 noise of HF's."""
    from tests.contrastive_oracle import contrastive_generate
    cfg, sd, k = hf_model
    ids = torch.from_numpy(k[f"{name}__input_ids"])
    eos = int(k[f"{name}__eos"])
    emb = sd["llm"]["model.embed_tokens.weight"].float()
    for b in range(ids.shape[0]):
        out, rec = contrastive_generate(cfg, sd["llm"], emb[ids[b]], int(k[f"{name}__k"]), float(k[f"{name}__alpha"]), int(k["max_new"]),
                                        None if eos < 0 else eos)
        assert out.tolist() == k[f"{name}__ids{b}"].tolist()
        assert torch.equal(rec["topk_ids"], torch.from_numpy(k[f"{name}__topk_ids{b}"]))
        for key in ("topk_probs", "pen", "score"):
            ref = torch.from_numpy(k[f"{name}__{key}{b}"])
            assert torch.allclose(rec[key], ref, rtol=1e-5, atol=1e-6), (key, (rec[key] - ref).abs().max())


def test_ranking_rules():
    from tests.contrastive_oracle import first_max, penalty
    ctx = torch.tensor([[1.0, 0.0], [0.0, 2.0]])
    nxt = torch.tensor([[3.0, 0.0], [1.0, 1.0], [0.0, -1.0]])
    assert torch.allclose(penalty(nxt, ctx), torch.tensor([1.0, 2 ** -0.5, 0.0]))
    assert first_max(torch.tensor([0.1, 0.3, 0.3])) == 1


# ---- generate()'s surface -----------------------------------------------------------------------------------------------------------
class ContrastiveDecoder(HostDecoder):
    """HostDecoder with the contrastive and beam entry points: each records its call and returns row b's first prompt row's value."""
    supports_contrastive = True

    def generate_contrastive(self, packed, lens, top_k, alpha, n, **kw):
        self.calls.append(("contrastive", lens, n, dict(kw, top_k=top_k, alpha=alpha)))
        outs, off = [], 0
        for L in lens:
            outs.append(torch.full((n,), int(packed[off, 0]), dtype=torch.int64))
            off += L
        return (outs, {"scores": torch.zeros(n, len(lens), 11)}) if kw.get("output_scores") else outs

    def generate_beam(self, emb, nb, n, **kw):
        self.calls.append(("beam", int(emb.shape[0]), n, kw))
        return torch.zeros(n, dtype=torch.int64)

    def generate_beam_batch(self, packed, lens, nb, n, **kw):
        self.calls.append(("beam", lens, n, kw))
        return [torch.zeros(n, dtype=torch.int64) for _ in lens]


@pytest.mark.parametrize("kw,what", [(dict(repetition_penalty=1.3), "processors"), (dict(prompt_lookup_num_tokens=3), "prompt_lookup"),
                                     (dict(prefix_cache=True), "prefix_cache"), (dict(output_logits=True), "output_logits"),
                                     (dict(guidance_scale=2.0, negative_prompt_ids=torch.tensor([[4, 4], [9, 8]])), "guidance_scale"),
                                     (dict(batch_invariant=True), "batch_invariant"), (dict(top_k=65), "top_k")])
@pytest.mark.parametrize("batch", [1, 2])
def test_refusals_before_any_decoder_call(kw, what, batch):
    gen, m = _model(ContrastiveDecoder())
    if "guidance_scale" in kw:
        kw = dict(kw, negative_prompt_ids=kw["negative_prompt_ids"][:batch])
    with pytest.raises(NotImplementedError, match=what):
        gen(m, TWO[:batch], max_new_tokens=4, penalty_alpha=0.6, **kw)
    assert m.llm.calls == []


def test_tensor_parallel_and_return_sequences_refused():
    """A decoder without contrastive search (the tensor-parallel one) is refused; num_return_sequences > 1 keeps greedy's ValueError."""
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert TPLlamaDecoder.supports_contrastive is False
    gen, m = _model(HostDecoder())
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, TWO, max_new_tokens=4, penalty_alpha=0.6, top_k=4)
    gen, m = _model(ContrastiveDecoder())
    with pytest.raises(ValueError, match="num_return_sequences"):
        gen(m, TWO, max_new_tokens=4, penalty_alpha=0.6, top_k=4, num_return_sequences=2)
    assert m.llm.calls == []


def test_refused_before_any_device_work_on_a_decoder_that_fails_every_call():
    """The NoDevice stub of test_beam_batch_cpu.py: any attribute the refusals would not need fails the test."""
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    import types
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")

    class NoDevice:  # any device work fails the test
        supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_contrastive = True
        fp8 = False

        def __getattr__(self, name):
            raise AssertionError(f"reached the decoder ({name})")

    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2, vocab_size=1000))
    m.llm = NoDevice()
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    for kw, msg in ((dict(repetition_penalty=1.2), "processors"), (dict(prefix_cache=True), "prefix_cache"),
                    (dict(prompt_lookup_num_tokens=3), "prompt_lookup"), (dict(output_logits=True), "output_logits"),
                    (dict(batch_invariant=True), "batch_invariant")):
        for b in (1, 2):
            with pytest.raises(NotImplementedError, match=msg):
                gen(m, ids[:b], penalty_alpha=0.5, top_k=3, **kw)


@pytest.mark.parametrize("alpha", [-0.1, 1.5, float("nan"), float("inf"), "x", None])
def test_penalty_alpha_outside_the_unit_interval_is_a_value_error(alpha):
    gen, m = _model(ContrastiveDecoder())
    if alpha is None:  # the default: no contrastive search
        gen(m, TWO, max_new_tokens=2, penalty_alpha=alpha, top_k=4)
        assert m.llm.calls[0][0] == "batch"
        return
    with pytest.raises(ValueError, match="penalty_alpha"):
        gen(m, TWO, max_new_tokens=2, penalty_alpha=alpha, top_k=4)
    assert m.llm.calls == []


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("kw", [dict(penalty_alpha=0.6, top_k=1), dict(penalty_alpha=0.0, top_k=4), dict(penalty_alpha=0, top_k=50),
                                dict(penalty_alpha=0.6, top_k=4, do_sample=True, temperature=0.7, seed=3),
                                dict(penalty_alpha=0.6, top_k=4, num_beams=3)])
def test_mode_rule_other_modes_run_what_they_run_today(kw, batch):
    """top_k = 1, penalty_alpha = 0, do_sample and beams: the decoder is called exactly as without penalty_alpha (HF ignores it)."""
    ids = TWO[:batch]
    base = {key: v for key, v in kw.items() if key != "penalty_alpha"}
    gen, m = _model(ContrastiveDecoder())
    plain = gen(m, ids, max_new_tokens=3, **base)
    calls = list(m.llm.calls)
    m.llm.calls.clear()
    out = gen(m, ids, max_new_tokens=3, **kw)
    assert m.llm.calls == calls and torch.equal(out, plain)
    assert all(c[0] != "contrastive" for c in calls)


def test_contrastive_calls_with_every_prompt_packed():
    gen, m = _model(ContrastiveDecoder())
    am = torch.tensor([[0, 1, 1], [1, 1, 1]])  # left padding
    stop = [lambda ids, scores: False]
    r = gen(m, TWO, attention_mask=am, max_length=7, penalty_alpha=0.25, eos_token_id=[5, 9], stopping_criteria=stop, pad_token_id=3,
            return_dict_in_generate=True, output_scores=True)
    (kind, lens, n, kw), = m.llm.calls
    assert kind == "contrastive" and lens == [2, 3] and n == 4  # max_length - the longest prompt
    assert kw["top_k"] == 50 and kw["alpha"] == 0.25 and kw["eos_token_ids"] == [5, 9] and kw["output_scores"]
    assert kw["stopping_fn"] is not None and kw["use_graph"]
    assert r.sequences[:, 0].tolist() == [6, 1] and len(r.scores) == 4
    m.llm.calls.clear()
    out = gen(m, TWO[1:], max_new_tokens=2, penalty_alpha=1, top_k=3)
    (kind, lens, n, kw), = m.llm.calls
    assert kind == "contrastive" and lens == [3] and kw["top_k"] == 3 and kw["alpha"] == 1.0 and out.tolist() == [[1, 1]]


# ---- the C entry points -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_host_argument_checks(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    f = 0x1000  # never dereferenced: every call below is refused on the host
    assert lib.srgpt_contrastive_partial_floats(2, 4, 100) == 2 * 4 * 4
    assert lib.srgpt_contrastive_partial_floats(0, 4, 100) == -1 and lib.srgpt_contrastive_partial_floats(1, 4, 0) == -1
    pen = lambda **kw: lib.srgpt_contrastive_penalty_bf16(*[kw.get(n, d) for n, d in (  # noqa: E731
        ("cand", f), ("ldc", 64), ("ctx", f), ("L_cap", 100), ("H", 64), ("pos", f), ("B", 2), ("k", 4), ("partial", f), ("stream", None))])
    for bad in (dict(k=0), dict(k=65), dict(H=60), dict(ldc=32), dict(cand=None), dict(ctx=f + 8), dict(B=0), dict(H=16384, ldc=16384),
                dict(L_cap=0)):
        assert pen(**bad) == -1, bad
    sel_args = [f, f, f, f, f, 64, 64, f, 1008, 1003, f, 100, f, 1008, f, 2, 4, f, f, f, f, f, f, None]
    for i, v in ((16, 0), (16, 65), (2, None), (8, 1000), (4, f + 4), (5, 60), (15, 0)):
        a = list(sel_args)
        a[i] = v
        assert lib.srgpt_contrastive_select_bf16(*a) == -1, (i, v)
    kv = [f, 2, 10, 16, 256, f, 5, f, -1, f, 2, 4, None]
    for i, v in ((0, None), (4, 100), (10, 0), (11, 0), (6, 0), (0, f + 4)):
        a = list(kv)
        a[i] = v
        assert lib.srgpt_kv_broadcast_rows(*a) == -1, (i, v)


def test_signatures_match_the_header_argument_counts():
    from spatialrgpt_b200 import _lib
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "srgpt_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for name in ("srgpt_contrastive_partial_floats", "srgpt_contrastive_penalty_bf16", "srgpt_contrastive_select_bf16", "srgpt_kv_broadcast_rows"):
        decl = re.search(name + r"\s*\(([^;]*)\);", src).group(1)
        assert len(decl.split(",")) == len(_lib.SIGNATURES[name][1]), name


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_contrastive_kernels_are_sm90a_sass_with_no_local_memory(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path(elem)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    lines = r.stdout.splitlines()
    found = {m.group(1): lines[i + 1] for i, line in enumerate(lines)
             for m in [re.search(r"Function (\S*(penalty_kernel|contrastive13select_kernel|kv_broadcast_kernel)\S*):", line)] if m}
    assert len(found) == 3, found
    for fn, usage in found.items():
        assert "LOCAL:0" in usage and "STACK:0" in usage, (fn, usage)
    sass = subprocess.run(["cuobjdump", "-sass", "-arch", "sm_90a", _lib.lib_path(elem)], capture_output=True, text=True).stdout
    for fn in found:
        assert fn in sass, fn
