"""Typical, epsilon and eta sampling without a GPU: the set rules of csrc/sampling.cu (tests/warpers_oracle.py) against transformers 5.5's
warper chain (tests/golden/warpers_kats.npz), generate()'s argument rules, the C ABI and the kernels' resource usage."""
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import warpers_oracle as W

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "warpers_kats.npz")


def golden():
    z = np.load(GOLDEN)
    out = []
    for V in (1000, 128256):
        x = torch.from_numpy(z[f"x_{V}"]).view(torch.bfloat16).float()
        keep = torch.from_numpy(np.unpackbits(z[f"keep_{V}"], axis=-1, count=V).astype(bool))
        out.append((V, x, keep))
    return z["settings"], out, z["warped_1000"]


def test_the_set_rules_match_hf_on_every_golden_row():
    settings, sets, _ = golden()
    n = 0
    for V, x, keep in sets:
        for r in range(x.shape[0]):
            for j, (T, k, p, typ, eps, eta) in enumerate(settings):
                got = W.kept(x[r], T, int(k), p, typ, eps, eta)
                assert torch.equal(got, keep[r, j]), (V, r, j, int((got != keep[r, j]).sum()))
                n += 1
    assert n == 2 * 4 * len(settings)


def test_golden_warped_rows_are_logits_over_t_on_the_kept_set():
    settings, sets, warped = golden()
    _, x, keep = sets[0]
    for r in range(x.shape[0]):
        for j, st in enumerate(settings):
            want = torch.where(keep[r, j], x[r] / torch.tensor(st[0], dtype=torch.float32), -torch.inf)
            assert torch.equal(torch.from_numpy(warped[r, j]), want)


def test_the_golden_covers_ties_flat_rows_and_every_warper():
    settings, sets, _ = golden()
    _, x, keep = sets[1]
    assert bool((x[2] == 0).all()) and bool(keep[2].all(-1).any())  # a flat row: typical keeps everything
    sizes = keep.sum(-1)
    assert int(sizes.min()) >= 1 and bool((sizes < x.shape[1]).any())
    on = [(t < 1, 0 < e < 1, 0 < h < 1) for _, _, _, t, e, h in settings]
    assert any(a and not b and not c for a, b, c in on) and any(b and not a for a, b, c in on) and any(c and not a for a, b, c in on)


@pytest.mark.parametrize("kw,want", [
    (dict(typical_p=0.9), (0.9, 0.0, 0.0)), (dict(typical_p=1.0), (1.0, 0.0, 0.0)), (dict(typical_p=1.5), (1.0, 0.0, 0.0)),
    (dict(epsilon_cutoff=3e-4), (1.0, 3e-4, 0.0)), (dict(epsilon_cutoff=0.0), (1.0, 0.0, 0.0)), (dict(epsilon_cutoff=1.0), (1.0, 0.0, 0.0)),
    (dict(epsilon_cutoff=-0.5), (1.0, 0.0, 0.0)), (dict(eta_cutoff=2.0), (1.0, 0.0, 0.0)), (dict(eta_cutoff=float("nan")), (1.0, 0.0, 0.0)),
    (dict(eta_cutoff=1e-3, typical_p=None), (1.0, 0.0, 1e-3)), (dict(typical_p=float("nan")), (1.0, 0.0, 0.0)),
])
def test_the_warpers_hf_turns_on(kw, want):
    from spatialrgpt_b200.llama_decoder import sampling_warpers
    assert sampling_warpers(kw) == want


@pytest.mark.parametrize("typ", [0.0, -0.2])
def test_typical_p_at_or_below_zero_raises_as_hf(typ):
    from transformers.generation.logits_process import TypicalLogitsWarper

    from spatialrgpt_b200.llama_decoder import sampling_warpers
    with pytest.raises(ValueError):
        TypicalLogitsWarper(typ)
    with pytest.raises(ValueError, match="typical_p"):
        sampling_warpers(dict(typical_p=typ))


def test_the_warped_entry_points_are_declared_and_bound():
    from spatialrgpt_b200 import _lib
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "srgpt_b200.h")).read()
    for name in ("srgpt_sample_warped_f32", "srgpt_sample_warped_scores_f32", "srgpt_sample_rows_warped", "srgpt_sample_rows_warped_scores",
                 "srgpt_llama_decode_rows_warped_bf16"):
        assert f"int {name}(" in header and name in _lib.SIGNATURES
    for elem in ("bf16", "f16"):
        lib = _lib.load(elem=elem)
        assert all(hasattr(lib, n) for n in ("srgpt_sample_warped_f32", "srgpt_sample_rows_warped", "srgpt_llama_decode_rows_warped_bf16"))


def test_warped_kernels_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    for elem in ("bf16", "f16"):
        _lib.load(elem=elem)
        r = subprocess.run(["cuobjdump", "-sass", _lib.lib_path(elem)], capture_output=True, text=True)
        if r.returncode != 0:
            pytest.skip("cuobjdump unavailable")
        funcs, cur = {}, None
        for line in r.stdout.splitlines():
            if "Function : " in line:
                cur = line.split("Function : ")[1].strip()
                funcs[cur] = []
            elif cur is not None:
                funcs[cur].append(line)
        new = [f for f in funcs if "warped_kernel" in f]
        assert len(new) == 3, new  # the one-row kernel, fp32 rows and element-type rows
        for f in new:
            body = "\n".join(funcs[f])
            assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"


@pytest.mark.parametrize("typ", [0.0, -1.0])
def test_generate_raises_for_typical_p_at_or_below_zero_before_any_decoder_call(typ):
    from tests.test_guidance_cpu import TWO, _model
    gen, m = _model()
    with pytest.raises(ValueError, match="typical_p"):
        gen(m, TWO, max_new_tokens=4, do_sample=True, typical_p=typ)
    assert m.llm.calls == []


def test_greedy_and_temperature_zero_ignore_the_warpers_and_sampling_passes_them():
    """HF builds the warpers only when sampling, and temperature 0 stays greedy here: no ValueError and no sampling reaches the decoder.
    Sampled, the three values reach it in the sampling dict."""
    from tests.test_guidance_cpu import TWO, _model
    for kw in (dict(typical_p=0.0, epsilon_cutoff=5.0), dict(do_sample=True, temperature=0, typical_p=-1.0)):
        gen, m = _model()
        gen(m, TWO, max_new_tokens=2, **kw)
        assert m.llm.calls and all(c[3].get("sampling") is None for c in m.llm.calls)
    gen, m = _model()
    gen(m, TWO, max_new_tokens=2, do_sample=True, typical_p=0.5, epsilon_cutoff=3e-4, eta_cutoff=2.0)
    smp = m.llm.calls[0][3]["sampling"]
    assert (smp["typical_p"], smp["epsilon_cutoff"], smp["eta_cutoff"]) == (0.5, 3e-4, 2.0)
