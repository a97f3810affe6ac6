"""Sampled batches on the CPU: the exports and argument checks of the multi-row sampler, its SASS, the per-sequence seeds, the page
copies that give each of a prompt's rows its prompt, and the num_return_sequences combinations that raise before any GPU work."""
import subprocess
import types

import pytest
import torch

from spatialrgpt_b200.llama_decoder import PAGE_SIZE, SEED_MASK, prompt_page_pairs, sequence_seeds

BAD = -1


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_libraries_export_and_check_arguments(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    assert hasattr(lib, "srgpt_sample_rows")
    x = 16  # a non-NULL address: every call below fails its argument check before any launch
    ok = [x, 1, 128, 3, 100, x, x, x, 0, x, None]
    for i, v in ((0, None), (5, None), (6, None), (7, None), (9, None), (3, 0), (3, -1), (3, 65536), (4, 0), (4, -5), (2, 99), (1, 2)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_sample_rows(*args) == BAD, (i, v)
        assert "invalid argument" in _lib.last_error()


def test_ops_wrapper_rejects_bad_arguments_without_a_gpu():
    from spatialrgpt_b200 import ops
    from spatialrgpt_b200._lib import SrgptError
    f = torch.zeros(3, 100)
    p, s, st, ids = torch.ones(3), torch.zeros(3, dtype=torch.int64), torch.zeros(1, dtype=torch.int32), torch.zeros(3, dtype=torch.int64)
    with pytest.raises(SrgptError, match="CUDA"):
        ops.sample_rows(f, p, s, st, 0, ids)  # CPU tensors never reach the library


def _sass_functions(path):
    r = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    funcs, cur = {}, None
    for line in r.stdout.splitlines():
        if "Function : " in line:
            cur = line.split("Function : ")[1].strip()
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    return funcs


def test_new_kernel_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    for elem in ("bf16", "f16"):
        _lib.load(elem=elem)
        funcs = _sass_functions(_lib.lib_path(elem))
        new = [f for f in funcs if "sample_rows_kernel" in f]
        assert len(new) == 2, new  # fp32 rows and element-type rows
        for f in new:
            body = "\n".join(funcs[f])
            assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"
        assert any("sample_top_p_kernel" in f for f in funcs)


# ---- seeds -------------------------------------------------------------------------------------------------------------------------
def sequential_recurrence(seed: int, B: int):
    """What generate_batch did for B sampled sequences before the batched path: before sequence b,
    sample_seed = (sample_seed + 0x9E3779B97F4A7C15 * (b + 1)) & (2^63 - 1)."""
    s, out = seed & 0x7FFFFFFFFFFFFFFF, []
    for b in range(B):
        s = (s + 0x9E3779B97F4A7C15 * (b + 1)) & 0x7FFFFFFFFFFFFFFF
        out.append(s)
    return out


@pytest.mark.parametrize("seed", [0, 1, 11, 2 ** 62 + 12345, 2 ** 63 - 1, 2 ** 64 - 1])
def test_sequence_seeds_follow_the_sequential_recurrence(seed):
    for B in (1, 2, 3, 32, 256):
        got = sequence_seeds(seed, B)
        assert got == sequential_recurrence(seed, B)
        assert got == [(seed + 0x9E3779B97F4A7C15 * (b + 1) * (b + 2) // 2) % 2 ** 63 for b in range(B)]
        assert all(0 <= s <= SEED_MASK for s in got)
    seeds = sequence_seeds(seed, 256)
    assert len(set(seeds)) == 256
    assert any(b < a for a, b in zip(seeds, seeds[1:]))  # the 63-bit wrap happens within 256 sequences


# ---- the prompt pages of a prompt's rows -------------------------------------------------------------------------------------------
def beam_batch_inline_pairs(tables, seq_lens, k):
    """The pairs generate_beam_batch built inline at its prefill before prompt_page_pairs existed."""
    B = len(seq_lens)
    return [(tables[g * k][j], tables[g * k + i][j], 0, min(PAGE_SIZE, seq_lens[g] - j * PAGE_SIZE))
            for g in range(B) for i in range(1, k) for j in range((seq_lens[g] + PAGE_SIZE - 1) // PAGE_SIZE)]


@pytest.mark.parametrize("seq_lens,n", [([21, 16, 1, 40], 3), ([259], 4), ([7, 33], 2), ([16, 17, 15], 5), ([5, 9], 1)])
def test_prompt_page_pairs_cover_every_prompt_row_once(seq_lens, n):
    import numpy as np
    rs = np.random.RandomState(len(seq_lens) * 10 + n)
    R = len(seq_lens) * n
    per = (max(seq_lens) + PAGE_SIZE - 1) // PAGE_SIZE + 1
    perm = rs.permutation(R * per).tolist()
    tables = [perm[per * r:per * r + per] for r in range(R)]
    pairs = prompt_page_pairs(tables, seq_lens, n)
    assert pairs == beam_batch_inline_pairs(tables, seq_lens, n)
    sources = {s for s, _, _, _ in pairs}
    assert not sources & {d for _, d, _, _ in pairs}  # nothing needs staging
    for g, L in enumerate(seq_lens):
        for i in range(1, n):
            r = g * n + i
            covered = [(d, lo + t) for s, d, lo, cnt in pairs for t in range(cnt) if d in tables[r]]
            want = [(tables[r][p // PAGE_SIZE], p % PAGE_SIZE) for p in range(L)]
            assert sorted(covered) == sorted(want) and len(covered) == len(set(covered)) == L, (g, i)
            srcs = [(s, lo + t) for s, d, lo, cnt in pairs for t in range(cnt) if d in tables[r]]
            assert sorted(srcs) == sorted((tables[g * n][p // PAGE_SIZE], p % PAGE_SIZE) for p in range(L))
    if n == 1:
        assert pairs == []


# ---- what raises before any GPU work -----------------------------------------------------------------------------------------------
class NoDevice:  # any device work fails the test
    supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_batch_sampling = True

    def __getattr__(self, name):
        raise AssertionError(f"reached the decoder ({name})")


def _generate():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2, vocab_size=1000))
    m.llm = NoDevice()
    return gen, m


def test_num_return_sequences_combinations_raise_before_gpu_work():
    gen, m = _generate()
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    smp = dict(do_sample=True, temperature=0.7)
    cases = [
        (dict(num_return_sequences=0, **smp), ValueError, ">= 1"),
        (dict(num_return_sequences=-2), ValueError, ">= 1"),
        (dict(num_return_sequences=2), ValueError, "do_sample"),
        (dict(num_return_sequences=3, do_sample=False), ValueError, "do_sample"),
        (dict(num_return_sequences=2, do_sample=True, temperature=0), ValueError, "do_sample"),
        (dict(num_return_sequences=2, do_sample=True, temperature=0.0), ValueError, "do_sample"),
        (dict(num_return_sequences=2, num_beams=3), NotImplementedError, "beam search"),
        (dict(num_return_sequences=2, num_beams=3, **smp), NotImplementedError, "beam search"),
        (dict(num_return_sequences=2, prefix_cache=True, **smp), NotImplementedError, "prefix_cache"),
        (dict(num_return_sequences=2, prompt_lookup_num_tokens=3, **smp), NotImplementedError, "prompt_lookup_num_tokens"),
        (dict(num_return_sequences=2, output_logits=True, **smp), NotImplementedError, "output_logits"),
    ]
    for kw, exc, msg in cases:
        for b in (1, 2):
            with pytest.raises(exc, match=msg):
                gen(m, ids[:b], **kw)
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    m.llm = TPLlamaDecoder.__new__(TPLlamaDecoder)
    for b in (1, 2):
        with pytest.raises(NotImplementedError, match="tensor-parallel"):
            gen(m, ids[:b], num_return_sequences=2, **smp)


def test_decoder_validates_num_return_sequences_before_gpu_work():
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    fn = getattr(LlamaDecoder.generate_batch, "__wrapped__", LlamaDecoder.generate_batch)
    fn = getattr(fn, "__wrapped__", fn)
    dec = NoDevice()
    x = torch.zeros(6, 8)
    smp = dict(temperature=0.7, seed=1)
    with pytest.raises(ValueError, match=">= 1"):
        fn(dec, x, [3, 3], 4, num_return_sequences=0, sampling=smp)
    with pytest.raises(ValueError, match="sampling"):
        fn(dec, x, [3, 3], 4, num_return_sequences=2)
    with pytest.raises(NotImplementedError, match="output_logits"):
        fn(dec, x, [3, 3], 4, num_return_sequences=2, sampling=smp, return_logits=True)
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        fn(TPLlamaDecoder.__new__(TPLlamaDecoder), x, [3, 3], 4, num_return_sequences=2, sampling=smp)
