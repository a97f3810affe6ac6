"""generate(output_hidden_states=, output_attentions=) on the CPU: the oracle's restatement (tests/generate_outputs_oracle.py) pinned to
HF's generate() (tests/golden/generate_outputs_kats.npz), the column mapping, the refusals and the memory guard generate() raises before
any device work, the flags ignored without return_dict_in_generate, and the new C entry points' exports and SASS."""
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "generate_outputs_kats.npz")
NEW = ("srgpt_attention_probs_decode_bf16", "srgpt_store_step_rows_bf16", "srgpt_llama_decode_step_probe_bf16")


# ---- the oracle against HF ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fixture():
    from oracle import srgpt_oracle as O
    from tests.golden.make_golden import CASES
    k = np.load(GOLDEN)
    cfg = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    return cfg, O.make_weights(cfg, seed=int(k["weight_seed"])), k


def _close(a, b, what):
    b = torch.as_tensor(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.allclose(a.float(), b, rtol=1e-4, atol=1e-5), (what, float((a.float() - b).abs().max()))


def _check_row(cfg, sd, k, prefix, b, emb, off, T):
    from tests.generate_outputs_oracle import generate_outputs
    N = int(k["n_new"])
    ids, hs, att = generate_outputs(cfg, sd["llm"], emb, N, off=off, T=T)
    assert ids.tolist() == k[prefix + "ids"][b].tolist()
    n = emb.shape[0]
    rows = slice(off, off + n)
    for l in range(cfg.layers + 1):
        _close(hs[0][l], k[prefix + "hidden0"][l, b, rows], f"prompt hidden {l}")
    for l in range(cfg.layers):
        _close(att[0][l], k[prefix + "attn0"][l, b, :, rows, rows], f"prompt attn {l}")
    assert len(hs) == len(att) == N
    for t in range(1, N):
        for l in range(cfg.layers + 1):
            _close(hs[t][l], k[prefix + "hidden_steps"][t - 1, l, b], f"step {t} hidden {l}")
        for l in range(cfg.layers):
            ref = k[prefix + "attn_steps"][t - 1, l, b]
            assert not ref[..., T + t:].any()  # HF's entry t is T + t wide
            _close(att[t][l], ref[..., :T + t], f"step {t} attn {l}")
            assert torch.allclose(att[t][l].sum(-1), torch.ones(cfg.heads, 1), atol=1e-5)


def test_one_prompt_against_hf(fixture):
    cfg, sd, k = fixture
    emb = torch.from_numpy(k["single_embeds"])
    _check_row(cfg, sd, k, "single_", 0, emb, 0, emb.shape[0])


def test_left_padded_batch_against_hf(fixture):
    cfg, sd, k = fixture
    emb, mask = torch.from_numpy(k["batch_embeds"]), torch.from_numpy(k["batch_mask"]).bool()
    T = emb.shape[1]
    for b, n in enumerate(k["batch_lens"].tolist()):
        assert bool(mask[b, T - n:].all()) and not bool(mask[b, :T - n].any())
        _check_row(cfg, sd, k, "batch_", b, emb[b, T - n:], T - n, T)


def test_column_mapping():
    from tests.generate_outputs_oracle import decode_columns
    assert decode_columns(3, 2, 5, 1).tolist() == [2, 3, 4, 5]  # left padding: the prompt ends at T, then the generated keys
    assert decode_columns(3, 0, 5, 2).tolist() == [0, 1, 2, 5, 6]  # right padding: columns 3, 4 are the pad
    assert decode_columns(5, 0, 5, 3).tolist() == list(range(8))


# ---- generate()'s refusals, the flags without the dict, the memory guard ------------------------------------------------------------
class NoDevice:
    """A decoder stand-in: any attribute the refusals would not need fails the test."""
    dims = types.SimpleNamespace(num_hidden_layers=32, num_attention_heads=32, hidden_size=4096, vocab_size=1000)
    supports_logits_processors = True
    supports_prompt_lookup = True
    supports_prefix_reuse = True
    supports_output_scores = True
    supports_batch_invariant = True
    supports_contrastive = True
    supports_batch_sampling = True
    fp8 = False

    def __init__(self, supports: bool = True):
        self.supports_generate_outputs = supports

    def generate_beam(self, *a, **kw):
        raise AssertionError("reached the decoder (generate_beam)")

    def __getattr__(self, name):
        raise AssertionError(f"reached the decoder ({name})")


def _model(llm):
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.weights = types.SimpleNamespace(dtype=torch.bfloat16, llama=types.SimpleNamespace(embed=torch.zeros(1)))
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(vocab_size=1000, eos_token_id=None, pad_token_id=0))
    m.llm = llm
    return m


FLAGS = dict(return_dict_in_generate=True, output_attentions=True, output_hidden_states=True)


@pytest.mark.parametrize("kw,what", [
    (dict(num_beams=2), "beam search"),
    (dict(penalty_alpha=0.5, top_k=4), "penalty_alpha"),
    (dict(guidance_scale=1.5, negative_prompt_ids=torch.tensor([[5, 6]])), "guidance_scale"),
    (dict(batch_invariant=True), "batch_invariant"),
    (dict(prompt_lookup_num_tokens=3), "prompt_lookup_num_tokens"),
    (dict(prefix_cache=True), "prefix_cache"),
    (dict(num_return_sequences=2, do_sample=True, temperature=0.7), "num_return_sequences"),
])
def test_refusals_before_device_work(kw, what):
    with pytest.raises(NotImplementedError, match=what):
        _model(NoDevice()).generate(input_ids=torch.tensor([[1, 2, 3]]), max_new_tokens=4, **FLAGS, **kw)


def test_output_logits_over_a_batch_and_tensor_parallel_refused():
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    with pytest.raises(NotImplementedError, match="output_logits over a batch"):
        _model(NoDevice()).generate(input_ids=ids, max_new_tokens=4, output_logits=True, **FLAGS)
    with pytest.raises(NotImplementedError, match="tensor-parallel decoder: no rank holds every attention head"):
        _model(NoDevice(False)).generate(input_ids=ids[:1], max_new_tokens=4, **FLAGS)
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert TPLlamaDecoder.supports_generate_outputs is False and LlamaDecoder.supports_generate_outputs is True


def test_flags_are_ignored_without_the_dict():
    """Without return_dict_in_generate the flags are dropped before the refusals: a combination refused with the dict goes on to the
    decoder (here the stand-in's beam search), as with no flags at all."""
    for flags in ({}, dict(output_attentions=True, output_hidden_states=True)):
        with pytest.raises(AssertionError, match="reached the decoder"):
            _model(NoDevice()).generate(input_ids=torch.tensor([[1, 2, 3]]), max_new_tokens=4, num_beams=2, **flags)


@pytest.mark.parametrize("h,a", [(True, False), (False, True), (True, True)])
def test_memory_guard_names_the_bytes(monkeypatch, h, a):
    from spatialrgpt_b200.llava_llama import generate_outputs_bytes
    B, T, N, L, H, nh = 2, 300, 128, 32, 4096, 32
    need = (2 * ((L + 1) * B * T * H * h + L * B * nh * T * T * a) + (N - 1) * (L + 1) * B * H * 2 * h
            + (N - 1) * L * B * nh * (T + N - 1) * 2 * a)
    assert generate_outputs_bytes(L, H, nh, B, T, N, h, a) == need
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need - 1, 80 << 30))
    ids = torch.ones(B, T, dtype=torch.int64)
    with pytest.raises(RuntimeError, match=f"needs {need} bytes"):
        _model(NoDevice()).generate(input_ids=ids, max_new_tokens=N, return_dict_in_generate=True, output_hidden_states=h, output_attentions=a)
    # max_length sets the budget as generate() does: max_length less the longest prompt
    need_ml = generate_outputs_bytes(L, H, nh, B, T, 10, h, a)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need_ml - 1, 80 << 30))
    with pytest.raises(RuntimeError, match=f"needs {need_ml} bytes"):
        _model(NoDevice()).generate(input_ids=ids, max_length=T + 10, return_dict_in_generate=True, output_hidden_states=h, output_attentions=a)


# ---- the C entry points -------------------------------------------------------------------------------------------------------------
def test_new_symbols_declared_typed_and_exported():
    from spatialrgpt_b200 import _lib
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "srgpt_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for elem in ("bf16", "f16"):
        out = subprocess.run(["nm", "-D", "--defined-only", _lib.lib_path(elem)], capture_output=True, text=True, check=True).stdout
        for name in NEW:
            assert re.search(r"\sT\s+" + name + r"\b", out), (elem, name)
    for name in NEW:
        decl = re.search(name + r"\s*\(([^;]*)\);", src).group(1)
        assert len(decl.split(",")) == len(_lib.SIGNATURES[name][1]), name
    fields = re.search(r"typedef struct \{([^}]*)\} srgpt_decode_probe;", src).group(1)
    n_fields = sum(len(decl.split(",")) for decl in fields.split(";") if decl.strip())
    assert n_fields == len(_lib.DecodeProbe._fields_)
    assert _lib.load().srgpt_abi_version() == 1


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_host_argument_checks(elem):
    import ctypes as C

    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    f = 0x1000  # never dereferenced: every call below is refused on the host
    good = dict(q=f, q_ld=4096, kv=f, pt=f, pt_stride=64, page_size=16, pos=f, rows=2, nh=32, nkv=8, hd=128, scale=0.088, off=f, n_prompt=f,
                T=100, n_cols=120, step=f, step_offset=-1, out=f, step_stride=2 * 32 * 120, row_stride=32 * 120, head_stride=120, ws=f, stream=None)
    probs = lambda **kw: lib.srgpt_attention_probs_decode_bf16(*dict(good, **kw).values())  # noqa: E731
    for bad in (dict(q=None), dict(out=None), dict(ws=None), dict(step=None), dict(nkv=3), dict(nkv=2), dict(q_ld=4090), dict(kv=f + 8),
                dict(n_cols=99), dict(head_stride=119), dict(row_stride=32 * 120 - 1), dict(pt_stride=0), dict(rows=0)):
        assert probs(**bad) == -1, bad
    assert probs(hd=64, q_ld=2048) == -3 and b"head_dim" in lib.srgpt_last_error()
    assert lib.srgpt_store_step_rows_bf16(f, 1, 4096, None, -1, f, 4096, 4096, None) == -1  # no step
    assert lib.srgpt_store_step_rows_bf16(f, 1, 4096, f, -1, f, 4100, 4096, None) == -1  # step stride not a multiple of 8
    args = [f, f, None, None, None, 2, f, f, f, 512, 4, 2, 128, 1024, 1e-5, f, f, f, f, 16, f, f, None, 1000, f, f, None, f, f]
    assert lib.srgpt_llama_decode_step_probe_bf16(*args, None, None) == -1  # no probe
    probe = _lib.DecodeProbe()  # records nothing
    assert lib.srgpt_llama_decode_step_probe_bf16(*args, C.byref(probe), None) == -1
    probe.hidden = f
    both = list(args)
    both[2], both[3] = f, f  # packed and nf4 together
    assert lib.srgpt_llama_decode_step_probe_bf16(*both, C.byref(probe), None) == -1
    assert b"invalid argument" in lib.srgpt_last_error()


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_new_kernels_in_the_sass_without_local_memory(elem):
    from spatialrgpt_b200 import _lib
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
    new = [fn for fn in funcs if "decode_stats_kernel" in fn or "decode_probs_kernel" in fn or "store_rows_kernel" in fn]
    assert len(new) == 3, new
    for fn in new:
        body = "\n".join(funcs[fn])
        assert "LDL" not in body and "STL" not in body, f"{fn} uses local memory"
