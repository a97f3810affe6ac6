"""HF's logits processors without a GPU: the numpy restatement of the device kernel (logits_processors.process_np) pinned to
transformers' processor classes on CPU tensors, the min_length / min_new_tokens mapping against _prepare_generated_length, the kwarg
validation of generate(), the RegionChat forwarding, the C-ABI argument checks and the new kernels' SASS."""
import subprocess
import types

import numpy as np
import pytest
import torch

from spatialrgpt_b200 import logits_processors as LP

V = 64


def _hf(scores, hist, spec):
    """transformers' processors, in _get_logits_processor's order, on a CPU fp32 row with the generated ids as input_ids."""
    lp = pytest.importorskip("transformers.generation.logits_process")
    ids = torch.tensor([list(hist)], dtype=torch.long).reshape(1, len(hist))
    x = torch.tensor(scores, dtype=torch.float32)[None]
    eos = spec.get("eos_token_ids") or []
    procs = []
    if "repetition_penalty" in spec:
        procs.append(lp.RepetitionPenaltyLogitsProcessor(float(spec["repetition_penalty"])))
    if "no_repeat_ngram_size" in spec:
        procs.append(lp.NoRepeatNGramLogitsProcessor(int(spec["no_repeat_ngram_size"])))
    if spec.get("bad_words_ids_raw"):
        procs.append(lp.NoBadWordsLogitsProcessor(spec["bad_words_ids_raw"], eos_token_id=eos or None))
    if spec.get("min_new_tokens", 0) > 0 and eos:
        procs.append(lp.MinLengthLogitsProcessor(spec["min_new_tokens"], eos))
        procs.append(lp.MinNewTokensLengthLogitsProcessor(0, spec["min_new_tokens"], eos))
    for p in procs:
        x = p(ids, x)
    return x[0].numpy()


def _spec(**kw):
    """A spec as generate() builds it, plus the raw bad-word list for transformers."""
    s = LP.resolve_min_length(LP.parse(**kw, vocab_size=V), 0) or {}
    if kw.get("bad_words_ids"):
        s["bad_words_ids_raw"] = kw["bad_words_ids"]
    return s


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _scores(seed):
    rs = np.random.RandomState(seed)
    x = (rs.randn(V) * 3).astype(np.float32)
    x[[3, 9]] = 0.0
    x[[4, 10]] = -0.0
    x[[5, 11]] = -2.5
    return x


HISTORIES = [[], [7], [3, 4, 5, 3, 3, 9, 4], [1, 2, 1, 2, 1], [5, 6, 7, 5, 6, 7, 5, 6], [9, 9, 9, 9, 9], [1, 2, 3, 4, 1, 2, 3],
             list(np.random.RandomState(1).randint(0, 8, 40)), list(np.random.RandomState(2).randint(0, V, 25))]


@pytest.mark.parametrize("penalty", [1.3, 0.7, 2.0, 1.1])
def test_repetition_penalty_matches_transformers(penalty):
    for i, h in enumerate(HISTORIES):
        s = _spec(repetition_penalty=penalty)
        x = _scores(i)
        assert _same(LP.process_np(x, h, s, true_division=True), _hf(x, h, s)), (penalty, h)


@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_no_repeat_ngram_matches_transformers(n):
    rs = np.random.RandomState(n)
    hs = HISTORIES + [[int(t) for t in rs.randint(0, 4, 30)] for _ in range(6)]
    hs += [[1, 2, 3, 4, 5, 9, 1, 2, 3, 4], [8, 8, 8, 8, 8, 8, 8]]  # planted repeats of every n up to 5
    for i, h in enumerate(hs):
        s = _spec(no_repeat_ngram_size=n)
        x = _scores(i)
        assert _same(LP.process_np(x, h, s), _hf(x, h, s)), (n, h)


def test_bad_words_match_transformers():
    bad = [[5], [1, 2], [2, 9], [3, 4, 5], [7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7], [63], [2]]
    for eos in (None, 2, [2, 5]):
        for i, h in enumerate(HISTORIES + [[7, 7, 3, 4], [3, 4], [1]]):
            s = _spec(bad_words_ids=bad, eos_token_id=eos)
            x = _scores(i)
            assert _same(LP.process_np(x, h, s), _hf(x, h, s)), (eos, h)
    assert LP.parse(bad_words_ids=[[2]], eos_token_id=2) is None  # the only bad word is [eos]: dropped, as HF does


def test_eos_lists_and_minimum_length_match_transformers():
    for eos in (3, [3, 4], [60, 3, 10]):
        for m in (1, 4, 9):
            for h in ([], [1, 2, 3], list(range(12))):
                s = _spec(min_new_tokens=m, eos_token_id=eos)
                x = _scores(len(h) + m)
                assert _same(LP.process_np(x, h, s), _hf(x, h, s)), (eos, m, h)
    assert LP.parse(min_new_tokens=5) is None  # no EOS id: a no-op, as in HF


def test_all_processors_together_match_transformers():
    rs = np.random.RandomState(7)
    for t in range(30):
        h = [int(v) for v in rs.randint(0, 10, rs.randint(0, 30))]
        s = _spec(repetition_penalty=float(rs.choice([0.5, 1.2, 1.7])), no_repeat_ngram_size=int(rs.randint(1, 5)),
                  bad_words_ids=[[int(rs.randint(0, 10))], [int(v) for v in rs.randint(0, 10, 2)], [int(v) for v in rs.randint(0, 10, 3)]],
                  min_new_tokens=int(rs.randint(0, 20)), eos_token_id=[int(rs.randint(0, 10))])
        x = _scores(t)
        assert _same(LP.process_np(x, h, s, true_division=True), _hf(x, h, s)), (t, h, s)


def test_penalty_rule_reciprocal_vs_division():
    """The device multiplies a positive score by fp32(1 / penalty) (the reciprocal taken in double), as ATen's CUDA division by a Python
    scalar does; CPU torch divides.  The two differ by one ulp on some scores (the GPU test pins the device rule to transformers on a
    CUDA tensor)."""
    x = np.linspace(0.01, 50, 20000, dtype=np.float32)
    inv = np.float32(1.0 / 1.1)
    assert inv != np.float32(1) / np.float32(1.1)  # ... and not the reciprocal of the fp32 penalty
    assert (x * inv != x / np.float32(1.1)).any()
    s = {"repetition_penalty": 1.1}
    assert _same(LP.process_np(x[:V], list(range(V)), s), x[:V] * inv)


def test_min_length_mapping_matches_prepare_generated_length():
    U = pytest.importorskip("transformers.generation.utils")
    from transformers import GenerationConfig
    S = 20
    for min_length, min_new in ((0, None), (5, None), (20, None), (27, None), (27, 3), (None, 4), (40, 0)):
        gc = GenerationConfig(min_length=min_length if min_length is not None else 0, min_new_tokens=min_new, max_new_tokens=8)
        host = types.SimpleNamespace(config=types.SimpleNamespace(is_encoder_decoder=False))
        gc = U.GenerationMixin._prepare_generated_length(host, gc, True, min_length is None, "inputs_embeds", 0, torch.zeros(1, S, 8))
        ours = LP.resolve_min_length(LP.parse(min_length=min_length, min_new_tokens=min_new, eos_token_id=2), S)
        m = 0 if ours is None else ours.get("min_new_tokens", 0)
        assert m == gc.min_length, (min_length, min_new, m, gc.min_length)


def test_encoding_layout():
    s = LP.parse(repetition_penalty=1.25, no_repeat_ngram_size=3, bad_words_ids=[[4], [5, 6, 7]], min_new_tokens=2, eos_token_id=[9, 8])
    f, ints = LP.encode(s)
    assert f.tolist() == [1.25, np.float32(1.0 / 1.25)]
    assert ints.tolist() == [15, 3, 2, 2, 2, 9, 8, 0, 1, 4, 4, 5, 6, 7]
    assert LP.parse(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, min_length=0, eos_token_id=2) is None


def test_validation():
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=1.5),
               dict(bad_words_ids=[]), dict(bad_words_ids=[1, 2]), dict(bad_words_ids=[[1], []]), dict(bad_words_ids=[[1, -2]]),
               dict(bad_words_ids=[[V]]), dict(bad_words_ids=[["a"]])):
        with pytest.raises(ValueError):
            LP.parse(**kw, vocab_size=V)


# ---- generate() kwargs -------------------------------------------------------------------------------------------------------------
def _unwrapped():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = LlavaLlamaModel.generate.__wrapped__.__wrapped__ if hasattr(LlavaLlamaModel.generate, "__wrapped__") else None
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2, vocab_size=V))
    m.llm = types.SimpleNamespace(supports_prompt_lookup=True, supports_logits_processors=True)
    return gen, m


def test_generate_kwargs_validation_and_unsupported_combinations():
    gen, m = _unwrapped()
    ids = torch.tensor([[1, 2, 3]])
    with pytest.raises(ValueError):
        gen(m, ids, repetition_penalty=0.0)
    with pytest.raises(ValueError):
        gen(m, ids, no_repeat_ngram_size=-2)
    with pytest.raises(ValueError):
        gen(m, ids, bad_words_ids=[[V + 3]])
    with pytest.raises(ValueError):
        gen(m, ids, bad_words_ids=[[1], 2])
    with pytest.raises(NotImplementedError, match="beam"):
        gen(m, ids, repetition_penalty=1.2, num_beams=2)
    with pytest.raises(NotImplementedError, match="prompt_lookup"):
        gen(m, ids, no_repeat_ngram_size=3, prompt_lookup_num_tokens=3)
    with pytest.raises(NotImplementedError, match="prompt_lookup"):
        gen(m, ids, min_new_tokens=3, prompt_lookup_num_tokens=3)
    m.llm = types.SimpleNamespace(supports_prompt_lookup=False, supports_logits_processors=False)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, ids, bad_words_ids=[[4]])
    with pytest.raises(TypeError):
        gen(m, ids, repetition_penalty=1.2, encoder_repetition_penalty=1.1)
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    assert LlamaDecoder.supports_logits_processors and not TPLlamaDecoder.supports_logits_processors


class _StubModel:
    device = torch.device("cpu")
    dtype = torch.bfloat16

    def __init__(self):
        self.calls = []
        self.config = types.SimpleNamespace(image_aspect_ratio="resize", mm_use_im_start_end=False)

    def generate(self, input_ids, **kw):
        self.calls.append(kw)
        return torch.tensor([[5, 6]])


def test_region_chat_forwards_only_non_neutral_values(monkeypatch):
    from spatialrgpt_b200 import chat as Ch
    monkeypatch.setattr(Ch, "process_images", lambda imgs, proc, cfg: torch.zeros(1, 3, 4, 4))
    monkeypatch.setattr(Ch, "tokenizer_image_token", lambda *a, **k: torch.tensor([1, 2, 3]))
    monkeypatch.setattr(Ch, "KeywordsStoppingCriteria", lambda *a, **k: None)
    tok = types.SimpleNamespace(batch_decode=lambda ids, skip_special_tokens=True: ["a b"])
    m = _StubModel()
    Ch.RegionChat(m, tok, None).ask("what is <region0>?", None, [])
    assert "repetition_penalty" not in m.calls[-1] and "no_repeat_ngram_size" not in m.calls[-1]
    Ch.RegionChat(m, tok, None, repetition_penalty=1.2, no_repeat_ngram_size=3).ask("what is <region0>?", None, [])
    assert m.calls[-1]["repetition_penalty"] == 1.2 and m.calls[-1]["no_repeat_ngram_size"] == 3


# ---- C-ABI and SASS --------------------------------------------------------------------------------------------------------------
def test_c_abi_argument_checks():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    x = 16
    bad = -1
    ok = (x, 1, 8, 1, 8, x, 0, 1, 4, x, -1, x, x, 16, x, 8, x, None)
    for i, v in ((0, None), (11, None), (12, None), (3, 0), (4, 0), (2, 4), (1, 2), (13, 4), (15, 4)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_logits_process(*args) == bad, i
    args = list(ok)
    args[14], args[16] = None, None  # neither processed rows nor ids
    assert lib.srgpt_logits_process(*args) == bad
    args = list(ok)
    args[5] = None  # a history length without the history
    assert lib.srgpt_logits_process(*args) == bad
    assert "invalid argument" in _lib.last_error()
    assert lib.srgpt_logits_pick_token(None, x, -1, x, None, None, 0, None) == bad
    assert lib.srgpt_logits_pick_token(x, x, -1, x, x, None, 8, None) == bad  # embedding table without next_x
    assert lib.srgpt_logits_pick_token(x, x, -1, x, x, x, 12, None) == bad    # K not a multiple of 8
    assert _lib.load(elem="f16").srgpt_logits_process(None, *ok[1:]) == bad


def test_new_kernels_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    _lib.load()
    for elem in ("bf16", "f16"):
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
        new = [f for f in funcs if "logits_process_kernel" in f or "logits_pick_kernel" in f]
        assert len(new) == 3, new  # fp32 rows, element-type rows, the pick
        for f in new:
            body = "\n".join(funcs[f])
            assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"
        assert any("ATOMS.OR" in ln for f in new for ln in funcs[f]), "the segment bitmaps live in shared memory"
