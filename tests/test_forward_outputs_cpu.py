"""forward(output_hidden_states=, output_attentions=) on the CPU: the oracle's restatement (tests/forward_outputs_oracle.py) pinned to HF's
eager LlamaForCausalLM (tests/golden/forward_outputs_kats.npz), the new C entry points' exports and host argument checks, their kernels'
SASS, and the refusals forward() raises before any device work."""
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "forward_outputs_kats.npz")
NEW = ("srgpt_attention_probs_bf16", "srgpt_llama_prefill_layers_probe_bf16")


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


def test_one_prompt_conventions_and_values(fixture):
    from oracle import srgpt_oracle as O
    from tests.forward_outputs_oracle import llama_forward_outputs
    cfg, sd, k = fixture
    emb = torch.from_numpy(k["single_embeds"])
    logits, hs, att = llama_forward_outputs(cfg, sd["llm"], emb)
    assert len(hs) == cfg.layers + 1 and len(att) == cfg.layers
    assert torch.equal(hs[0], emb)  # [0] is inputs_embeds
    assert cfg.heads != cfg.kv_heads  # the GQA head mapping is exercised
    for l in range(cfg.layers + 1):
        _close(hs[l], k["single_hidden"][l], f"hidden {l}")
    for l in range(cfg.layers):
        _close(att[l], k["single_attn"][l], f"attn {l}")
        assert torch.allclose(att[l].sum(-1), torch.ones(cfg.heads, emb.shape[0]), atol=1e-5)  # fp32 softmax rows
        assert bool((att[l].triu(1) == 0).all())
    _close(logits, k["single_logits"], "logits")
    # [L] is the final norm of the last layer's residual stream: the rows lm_head reads
    assert torch.equal(logits, torch.nn.functional.linear(hs[-1], sd["llm"]["lm_head.weight"].float()).float())
    assert torch.equal(logits, O.llama_forward(cfg, sd["llm"], emb, None)[0])  # the oracle's default result is untouched


def test_left_padded_batch_on_its_valid_blocks(fixture):
    from tests.forward_outputs_oracle import llama_forward_outputs
    cfg, sd, k = fixture
    emb, mask = torch.from_numpy(k["batch_embeds"]), torch.from_numpy(k["batch_mask"]).bool()
    T = emb.shape[1]
    for b, n in enumerate(k["batch_lens"].tolist()):
        rows = slice(T - n, T)
        assert bool(mask[b, rows].all()) and not bool(mask[b, :T - n].any())
        _, hs, att = llama_forward_outputs(cfg, sd["llm"], emb[b, rows])
        for l in range(cfg.layers + 1):
            _close(hs[l], k["batch_hidden"][l, b, rows], f"hidden {l} prompt {b}")
        for l in range(cfg.layers):
            _close(att[l], k["batch_attn"][l, b, :, rows, rows], f"attn {l} prompt {b}")


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
    assert _lib.load().srgpt_abi_version() == 1


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_host_argument_checks(elem):
    import ctypes as C

    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    f = 0x1000  # never dereferenced: every call below is refused on the host
    R = 100
    good = dict(q=f, q_ld=1536, k=f, k_ld=1536, n_seqs=1, cu=None, max_seqlen=90, nh=8, nkv=2, hd=128, scale=0.088, out=f,
                seq_stride=8 * R * R, head_stride=R * R, ld=R, out_rows=R, row_off=None, stream=None)
    probs = lambda **kw: lib.srgpt_attention_probs_bf16(*dict(good, **kw).values())  # noqa: E731
    for bad in (dict(q=None), dict(out=None), dict(nkv=3), dict(q_ld=1530), dict(k=f + 8), dict(n_seqs=2), dict(max_seqlen=R + 1),
                dict(ld=R - 1), dict(head_stride=R * R - 1), dict(seq_stride=R * R), dict(n_seqs=0)):
        assert probs(**bad) == -1, bad
    assert probs(hd=64) == -3 and b"head_dim" in lib.srgpt_last_error()
    probe = _lib.PrefillProbe()
    probe.out_rows = 8  # shorter than the prompt
    args = [f, f, None, None, 1, f, f, f, f, None, None, 20, 512, 4, 2, 128, 1024, 1e-5, f, f, f, f, 16, 1, None, 0, 0]
    assert lib.srgpt_llama_prefill_layers_probe_bf16(*args, None, None) == -1  # no probe
    assert lib.srgpt_llama_prefill_layers_probe_bf16(*args, C.byref(probe), None) == -1
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
    new = [fn for fn in funcs if "attn_probs_kernel" in fn or "store_rows_kernel" in fn]
    assert len(new) == 2, new
    for fn in new:
        body = "\n".join(funcs[fn])
        assert "LDL" not in body and "STL" not in body, f"{fn} uses local memory"
    assert "HMMA" in "\n".join(funcs[[fn for fn in new if "attn_probs_kernel" in fn][0]])  # Q K^T on the tensor cores


# ---- forward()'s refusals -----------------------------------------------------------------------------------------------------------
class NoDevice:
    """A decoder stand-in: any attribute the refusals would not need fails the test."""
    dims = types.SimpleNamespace(num_hidden_layers=32, num_attention_heads=32, hidden_size=4096)

    def __init__(self, supports: bool):
        self.supports_forward_outputs = supports

    def __getattr__(self, name):
        raise AssertionError(f"reached the decoder ({name})")


def _model(llm):
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.weights = types.SimpleNamespace(dtype=torch.bfloat16, llama=types.SimpleNamespace(embed=torch.zeros(1)))
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(vocab_size=1000))
    m.llm = llm
    return m


@pytest.mark.parametrize("kw", [dict(output_attentions=True), dict(output_hidden_states=True)])
def test_tensor_parallel_decoder_refuses_before_device_work(kw):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert TPLlamaDecoder.supports_forward_outputs is False and LlamaDecoder.supports_forward_outputs is True
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        _model(NoDevice(False)).forward(input_ids=torch.tensor([[1, 2, 3]]), **kw)


@pytest.mark.parametrize("kw,need", [(dict(output_attentions=True), 32 * 2 * 32 * 4096 * 4096 * 2),
                                     (dict(output_hidden_states=True), 33 * 2 * 4096 * 4096 * 2),
                                     (dict(output_attentions=True, output_hidden_states=True), 32 * 2 * 32 * 4096 * 4096 * 2 + 33 * 2 * 4096 * 4096 * 2)])
def test_memory_guard_names_the_bytes_before_device_work(monkeypatch, kw, need):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (need - 1, 80 << 30))
    ids = torch.ones(2, 4096, dtype=torch.int64)
    with pytest.raises(RuntimeError, match=f"needs {need} bytes"):
        _model(NoDevice(True)).forward(input_ids=ids, **kw)
    emb = torch.zeros(2, 4096, 8)
    with pytest.raises(RuntimeError, match=f"needs {need} bytes"):
        _model(NoDevice(True)).forward(inputs_embeds=emb, **kw)
