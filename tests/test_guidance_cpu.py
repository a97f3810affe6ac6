"""Classifier-free guidance on the CPU: the oracle's guidance (tests/guidance_oracle.py) pinned to HF's own generate(guidance_scale=,
negative_prompt_ids=) (tests/golden/cfg_kats.npz), generate()'s refusals and argument checks against a host-only stand-in decoder, what
that decoder is handed, the host argument checks of the C entry points and the kernel's resource usage."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from tests.test_batch_invariant_cpu import TWO, V, HostDecoder, _model

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cfg_kats.npz")
CASES = ["g0.5_b1", "g1.5_b1_long", "g3.0_b1", "g1.5_b2", "g3.0_b2"]


# ---- the oracle against HF ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hf_model():
    from oracle import srgpt_oracle as O
    from tests.golden.make_golden import CASES as MODEL_CASES
    k = np.load(GOLDEN)
    cfg = O.OracleConfig(**MODEL_CASES["tiny_masks_gqa"][0])
    sd = O.make_weights(cfg, seed=int(k["weight_seed"]))
    return cfg, sd, k


@pytest.mark.parametrize("name", CASES)
def test_oracle_guidance_equals_hf_generate(hf_model, name):
    """Ids exact; guided rows and raw logits within fp32 noise of HF's (its batched forward rounds in another order)."""
    from tests.guidance_oracle import guided_generate
    cfg, sd, k = hf_model
    ids, neg, g = torch.from_numpy(k[f"{name}__input_ids"]), torch.from_numpy(k[f"{name}__negative_ids"]), float(k[f"{name}__scale"])
    emb = sd["llm"]["model.embed_tokens.weight"].float()
    for b in range(ids.shape[0]):
        out, raw, rows = guided_generate(cfg, sd["llm"], emb[ids[b]], neg[b], g, int(k["max_new"]))
        assert out.tolist() == k[f"{name}__ids"][b].tolist()
        hf_rows = torch.from_numpy(k[f"{name}__scores"][:, b])
        hf_raw = torch.from_numpy(k[f"{name}__logits"][:, b])
        assert torch.allclose(rows, hf_rows, rtol=1e-5, atol=1e-4), (rows - hf_rows).abs().max()
        assert torch.allclose(raw, hf_raw, rtol=1e-5, atol=1e-4), (raw - hf_raw).abs().max()


def test_guided_row_rules():
    from tests.guidance_oracle import argmax_rule, combine, guided_row
    c = torch.tensor([1.0, 3.0, 3.0, float("-inf")])
    u = torch.tensor([0.0, 1.0, 2.0, 0.0])
    row = guided_row(c, u, 2.0)
    s, q = torch.log_softmax(c, -1), torch.log_softmax(u, -1)
    assert torch.equal(row, combine(s, q, 2.0)) and argmax_rule(row) == 1
    assert argmax_rule(torch.tensor([1.0, 5.0, float("nan"), 5.0])) == 1  # lowest index on ties, NaN never wins
    assert argmax_rule(torch.full((3,), float("nan"))) == 0
    assert argmax_rule(torch.tensor([float("-inf")] * 3)) == 0


# ---- generate()'s surface -----------------------------------------------------------------------------------------------------------
NEG = torch.tensor([[4, 4], [9, 8]])


@pytest.mark.parametrize("kw,what", [(dict(num_beams=2), "beam"), (dict(repetition_penalty=1.3), "processors"),
                                     (dict(prompt_lookup_num_tokens=3), "prompt_lookup"), (dict(prefix_cache=True), "prefix_cache"),
                                     (dict(do_sample=True, temperature=1.0, num_return_sequences=2), "num_return_sequences"),
                                     (dict(return_dict_in_generate=True, output_scores=True), "output_scores")])
def test_refusals_before_any_decoder_call(kw, what):
    gen, m = _model()
    with pytest.raises(NotImplementedError, match=what):
        gen(m, TWO, max_new_tokens=4, guidance_scale=1.5, negative_prompt_ids=NEG, **kw)
    assert m.llm.calls == []


def test_fp8_and_tensor_parallel_refused():
    dec = HostDecoder()
    dec.fp8 = True
    gen, m = _model(dec)
    with pytest.raises(NotImplementedError, match="fp8"):
        gen(m, TWO, max_new_tokens=4, guidance_scale=2.0, negative_prompt_ids=NEG)
    dec = HostDecoder()
    dec.supports_batch_invariant = False
    gen, m = _model(dec)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, TWO, max_new_tokens=4, guidance_scale=2.0, negative_prompt_ids=NEG)
    assert dec.calls == []


@pytest.mark.parametrize("neg,mask,what", [
    (None, None, "needs negative_prompt_ids"),
    (torch.tensor([[4, 4]]), None, r"\[2, T >= 1\]"),  # one row for two prompts
    (torch.tensor([4, 4]), None, r"\[2, T >= 1\]"),
    (torch.tensor([[4, V], [1, 2]]), None, "outside the vocabulary"),
    (torch.tensor([[4, -200], [1, 2]]), None, "IMAGE_TOKEN_INDEX"),
    (NEG, torch.tensor([[1, 1]]), "does not match"),
    (NEG, torch.tensor([[1, 0], [0, 0]]), "one non-empty run"),
    (torch.tensor([[4, 5, 6], [1, 2, 3]]), torch.tensor([[1, 0, 1], [1, 1, 1]]), "one non-empty run"),
])
def test_value_errors_before_any_decoder_call(neg, mask, what):
    gen, m = _model()
    with pytest.raises(ValueError, match=what):
        gen(m, TWO, max_new_tokens=4, guidance_scale=0.5, negative_prompt_ids=neg, negative_prompt_attention_mask=mask)
    assert m.llm.calls == []


@pytest.mark.parametrize("scale", [None, 1, 1.0])
@pytest.mark.parametrize("batch", [1, 2])
def test_scale_one_or_none_is_plain_generate(scale, batch):
    """guidance_scale None or 1: the decoder is called exactly as without the kwargs, and the negative prompt is ignored (as HF does)."""
    ids = TWO[:batch]
    gen, m = _model()
    plain = gen(m, ids, max_new_tokens=3)
    calls = list(m.llm.calls)
    m.llm.calls.clear()
    out = gen(m, ids, max_new_tokens=3, guidance_scale=scale, negative_prompt_ids=NEG[:batch])
    assert m.llm.calls == calls and torch.equal(out, plain)


def test_guided_calls_their_rows_in_groups_of_four():
    """Six prompts: groups of 4 and 2, each prompt with its own unpadded negative prompt embeddings, budget and seed."""
    from spatialrgpt_b200.llama_decoder import sequence_seeds
    gen, m = _model()
    ids = torch.arange(6 * 3).view(6, 3) + 1
    neg = torch.tensor([[0, 7, 7]] * 3 + [[7, 6, 0]] * 3)
    am = torch.tensor([[0, 1, 1]] * 3 + [[1, 1, 0]] * 3)
    out, lg = gen(m, ids, max_new_tokens=3, guidance_scale=3.0, negative_prompt_ids=neg, negative_prompt_attention_mask=am, do_sample=True,
                  temperature=0.7, seed=5, output_logits=True)
    rows = [c for c in m.llm.calls if c[0] == "rows"]
    assert [len(c[1]) for c in rows] == [4, 2] and len(m.llm.calls) == 2
    assert [s for c in rows for s in c[3]["seeds"]] == sequence_seeds(5, 6)
    for c in rows:
        assert c[3]["guidance_scale"] == 3.0 and c[3]["return_logits"] and c[3]["sampling"]["temperature"] == 0.7
    negs = [e[:, 0].tolist() for c in rows for e in c[3]["negative_embeds"]]
    assert negs == [[7.0, 7.0]] * 3 + [[7.0, 6.0]] * 3
    assert out[:, 0].tolist() == ids[:, 0].tolist() and len(lg) == 6


def test_batch1_guided_uses_its_own_seed_and_max_length():
    gen, m = _model()
    gen(m, TWO[:1], max_length=7, guidance_scale=2.0, negative_prompt_ids=NEG[:1], do_sample=True, temperature=1.0, seed=11)
    (kind, lens, budgets, kw), = m.llm.calls
    assert kind == "rows" and lens == [3] and budgets == [4] and kw["seeds"] == [11]
    m.llm.calls.clear()
    gen(m, TWO, max_new_tokens=2, guidance_scale=2.0, negative_prompt_ids=NEG, do_sample=True, temperature=1.0, seed=[3, 4])
    assert m.llm.calls[0][3]["seeds"] == [3, 4]
    m.llm.calls.clear()
    r = gen(m, TWO, max_new_tokens=2, guidance_scale=2.0, negative_prompt_ids=NEG, batch_invariant=True, return_dict_in_generate=True)
    assert m.llm.calls[0][0] == "rows" and r.scores is None and r.sequences.shape == (2, 2)


def test_negative_prompt_rows_strip_padding_on_either_side():
    from spatialrgpt_b200.llava_llama import negative_prompt_rows
    ids = torch.tensor([[0, 0, 5, 6], [7, 8, 0, 0], [1, 2, 3, 4]])
    am = torch.tensor([[0, 0, 1, 1], [1, 1, 0, 0], [1, 1, 1, 1]])
    assert [r.tolist() for r in negative_prompt_rows(ids, am, 3, V)] == [[5, 6], [7, 8], [1, 2, 3, 4]]
    assert [r.tolist() for r in negative_prompt_rows(ids, None, 3, V)] == ids.tolist()


# ---- the C entry points -------------------------------------------------------------------------------------------------------------
def test_host_argument_checks():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    fake, far = 0x1000, 0x10000000  # never dereferenced: every call below is refused on the host
    for P in (0, -1, 5):
        assert lib.srgpt_guidance_rows(fake, 100, P, fake, far, None, None, None) == -1
        assert lib.srgpt_guidance_pair_ids(fake, P, None) == -1
    assert lib.srgpt_guidance_rows(None, 100, 2, fake, far, None, None, None) == -1
    assert lib.srgpt_guidance_rows(fake, 100, 2, None, far, None, None, None) == -1
    assert lib.srgpt_guidance_rows(fake, 100, 2, fake, fake + 4 * 100, None, None, None) == -1  # guided rows overlap the logits
    assert lib.srgpt_guidance_rows(fake + 2, 100, 2, fake, far, None, None, None) == -1  # misaligned fp32 rows


def test_signatures_match_the_header_argument_counts():
    from spatialrgpt_b200 import _lib
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "srgpt_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for name in ("srgpt_guidance_rows", "srgpt_guidance_pair_ids", "srgpt_llama_decode_rows_guided_bf16"):
        decl = re.search(name + r"\s*\(([^;]*)\);", src).group(1)
        assert len(decl.split(",")) == len(_lib.SIGNATURES[name][1]), name


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_guidance_kernels_use_no_local_memory(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path(elem)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    lines = r.stdout.splitlines()
    found = {m.group(1): lines[i + 1] for i, line in enumerate(lines)
             for m in [re.search(r"Function (\S*(guidance_rows_kernel|pair_ids_kernel)\S*):", line)] if m}
    assert len(found) == 2, found
    for fn, usage in found.items():
        assert "LOCAL:0" in usage and "STACK:0" in usage, (fn, usage)
