"""Prompt-lookup speculative decoding without a GPU: a numpy restatement of the lookup rule pinned to transformers'
PromptLookupCandidateGenerator, the acceptance rule, the C-ABI argument checks, the new kernels' SASS, and the generate() kwarg
plumbing through the eval driver and the region chat."""
import os
import subprocess
import types

import numpy as np
import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
T_MAX = 8


def lookup_draft(hist, ngram, k):
    """The drafts for the next verify pass: n-gram sizes from ngram down to 1, the earliest window equal to the last n ids whose
    continuation is non-empty, at most k tokens of it, cut at the first negative id (a prompt row that is not text)."""
    hist = [int(v) for v in hist]
    L = len(hist)
    for n in range(min(ngram, L - 1), 0, -1):
        tail = hist[L - n:]
        if min(tail) < 0:
            continue
        for i in range(0, L - n):
            if hist[i:i + n] == tail:
                out = []
                for v in hist[i + n:i + n + k]:
                    if v < 0:
                        break
                    out.append(v)
                return out
    return []


def accept(drafts, choices):
    """a = the number of leading drafts equal to the model's greedy choices; the pass emits choices[:a + 1]."""
    a = 0
    while a < len(drafts) and drafts[a] == choices[a]:
        a += 1
    return a


def simulate(prompt, greedy, k, ngram, max_new):
    """(verify passes, drafted, accepted) of a request whose greedy continuation is `greedy` (long enough to cover the last pass)."""
    T = min(k, T_MAX - 1) + 1
    out, passes, drafted, accepted = [int(greedy[0])], 0, 0, 0
    while len(out) < max_new:
        d = lookup_draft(list(prompt) + out, ngram, T - 1)
        s = len(out)
        a = accept(d, [int(v) for v in greedy[s:s + T]])
        out += [int(v) for v in greedy[s:s + a + 1]]
        passes, drafted, accepted = passes + 1, drafted + len(d), accepted + a
    return passes, drafted, accepted


def _hf_candidates(hist, ngram, k):
    tr = pytest.importorskip("transformers")
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    g = PromptLookupCandidateGenerator(eos_token_id=torch.tensor([-7]), num_output_tokens=k, max_matching_ngram_size=ngram, max_length=10 ** 6)
    # a sentinel row gets a unique negative id: it never matches anything, as in the kernel
    ids = torch.tensor([[v if v >= 0 else -1000 - i for i, v in enumerate(hist)]], dtype=torch.long)
    del tr
    cand, _ = g.get_candidates(ids)
    new = cand[0, ids.shape[1]:].tolist()
    out = []
    for v in new:
        if v < 0:
            break
        out.append(v)
    return out


def _histories():
    rs = np.random.RandomState(0)
    hs = [list(rs.randint(0, 6, n)) for n in (2, 3, 5, 9, 17, 40, 120) for _ in range(6)]
    hs += [[1, 2, 3, 1, 2, 3, 1, 2], [5, 5, 5, 5], [7, 1, 2, 9, 9, 1, 2], [4, 8], [3], [1, 2, 3, 4, 5, 6, 1]]
    hs += [[1, -1, 2, 1], [-1, 1, 2, -1, 1], [2, 3, -1, -1, 2, 3], [1, 2, -1, 5, 1, 2], [9, -1, 9]]  # sentinels
    hs += [list(np.where(rs.rand(60) < 0.2, -1, rs.randint(0, 4, 60))) for _ in range(8)]
    hs += [[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 8]]  # the only match of the last id is near the tail
    return hs


@pytest.mark.parametrize("ngram", [1, 2, 3, 5])
@pytest.mark.parametrize("k", [1, 3, 7])
def test_lookup_rule_matches_transformers(ngram, k):
    for h in _histories():
        assert lookup_draft(h, ngram, k) == _hf_candidates(h, ngram, k), (h, ngram, k)


def test_lookup_rule_cases():
    assert lookup_draft([1, 2, 3, 1, 2], 2, 3) == [3, 1, 2]     # earliest match of the bigram (1, 2)
    assert lookup_draft([1, 2, 3, 9, 2], 2, 3) == [3, 9, 2]     # no bigram match: the unigram 2
    assert lookup_draft([4, 5, 6], 2, 3) == []                  # nothing to match
    assert lookup_draft([1, -1, 1], 2, 3) == []                 # the continuation starts at a non-text row
    assert lookup_draft([1, 7, -1, 8, 1], 2, 3) == [7]          # ... or is cut by one
    assert lookup_draft([3, 3], 9, 4) == [3]                    # n larger than the history
    assert lookup_draft([-1, -1], 2, 2) == []                   # sentinels never match each other


def test_acceptance_rule():
    assert accept([], [5]) == 0
    assert accept([5, 6, 7], [5, 6, 7, 8]) == 3
    assert accept([5, 9, 7], [5, 6, 7, 8]) == 1
    assert accept([4, 6], [5, 6, 7]) == 0
    g = list(range(100, 140))
    # perfect drafts (the continuation planted in the prompt): every pass takes k drafts + 1
    assert simulate(g, g, 3, 2, 21) == (5, 15, 15)
    # drafts that never match: one token per pass
    assert simulate([], [1, 2, 3, 4, 5, 6], 3, 2, 6)[2] == 0


def test_c_abi_argument_checks():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    assert _lib.SPEC_T_MAX == T_MAX
    bad = -1
    assert lib.srgpt_gemv_multi_bf16(None, 8, None, 8, None, 8, 1, 2, 8, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == bad
    x = 16
    assert lib.srgpt_gemv_multi_bf16(x, 8, x, 8, 32, 8, T_MAX + 1, 2, 8, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == bad
    assert lib.srgpt_gemv_multi_packed_bf16(x, 8, None, 32, 8, 1, 2, 8, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == bad
    assert lib.srgpt_lm_head_multi_bf16(x, 8, x, 8, 0, 5, 8, None, 0.0, None, x, None) == bad
    assert lib.srgpt_lm_head_multi_packed_bf16(x, 8, None, 1, 5, 8, None, 0.0, None, x, None) == bad
    assert lib.srgpt_attention_decode_multi_bf16(x, 128, x, 128, x, x, 16, x, 0, 1, 1, 128, 1.0, None) == bad
    assert lib.srgpt_spec_draft(x, None, x, x, x, x, 2, 2, x, x, 8, x, x, None) == bad  # history without its length
    assert lib.srgpt_spec_draft(None, None, x, x, x, x, 2, 0, x, x, 8, x, x, None) == bad  # n-gram size 0
    assert lib.srgpt_spec_accept(x, 5, T_MAX + 1, x, x, 4, x, x, x, None, None, None) == bad
    assert lib.srgpt_spec_accept(x, 5, 2, x, x, 4, x, x, x, None, x, None) == bad  # logits copy without the pass's rows
    for name in ("srgpt_llama_verify_step_bf16", "srgpt_llama_verify_step_packed_bf16"):  # every pointer NULL, every size 0
        zeros = [None if t is _lib.vp else (0.0 if t is _lib.cf else 0) for t in _lib.SIGNATURES[name][1]]
        assert getattr(lib, name)(*zeros) == bad
    assert "invalid argument" in _lib.last_error()
    lib16 = _lib.load(elem="f16")  # the packing is bf16 only; the plain multi-token path serves fp16 decoders
    from spatialrgpt_b200 import ops  # noqa: F401
    d = _lib.Packed12(sm=16, ex=16, base=16, row_ptr=16, exc=16)
    import ctypes as C
    assert lib16.srgpt_gemv_multi_packed_bf16(x, 1024, C.byref(d), 32, 8, 1, 2, 1024, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0,
                                              None) == -3
    assert lib16.srgpt_lm_head_multi_packed_bf16(x, 1024, C.byref(d), 1, 5, 1024, None, 0.0, None, x, None) == -3


def test_new_kernels_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    _lib.load()
    r = subprocess.run(["cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    funcs, cur = {}, None
    for line in r.stdout.splitlines():
        if "Function : " in line:
            cur = line.split("Function : ")[1].strip()
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    multi = [f for f in funcs if "decode_gemv_multi_kernel" in f]
    assert len(multi) == 8, multi  # plain / SwiGLU / QKV + RoPE / lm_head, plain and packed weights
    spec = [f for f in funcs if "spec_draft_kernel" in f or "spec_accept_kernel" in f or "spec_copy_logits_kernel" in f]
    assert len(spec) == 3
    for f in multi + spec:
        body = "\n".join(funcs[f])
        assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"
    assert any("FFMA" in ln for f in multi for ln in funcs[f])


# ---- kwarg plumbing with stub models ------------------------------------------------------------------------------------------
class _StubModel:
    device = torch.device("cpu")
    dtype = torch.bfloat16

    def __init__(self):
        self.calls = []
        self.config = types.SimpleNamespace(image_aspect_ratio="resize", mm_use_im_start_end=False)

    def generate(self, input_ids, **kw):
        self.calls.append(kw)
        return torch.tensor([[5, 6]])


def test_eval_driver_threads_the_option(monkeypatch):
    from spatialrgpt_b200 import eval_spatial as E
    monkeypatch.setattr(E, "process_images", lambda imgs, proc, cfg: torch.zeros(1, 3, 4, 4))
    monkeypatch.setattr(E, "tokenizer_image_token", lambda *a, **k: torch.tensor([1, 2, 3]))
    tok = types.SimpleNamespace(batch_decode=lambda ids, skip_special_tokens=True: ["a b"])
    line = {"id": 1, "text_q": "q", "qa_info": {}, "conversations": [{"from": "human", "value": "<image>\nq"}, {"from": "gpt", "value": "g"}]}
    m = _StubModel()
    E.answer_questions(line, m, tok, None, None, None, None, "llava_v1", "x", "a.jpg")
    assert "prompt_lookup_num_tokens" not in m.calls[-1]
    E.answer_questions(line, m, tok, None, None, None, None, "llava_v1", "x", "a.jpg", prompt_lookup_num_tokens=5)
    assert m.calls[-1]["prompt_lookup_num_tokens"] == 5
    args = E.build_arg_parser().parse_args(["--model-path", "m", "--prompt-lookup-num-tokens", "4"])
    assert args.prompt_lookup_num_tokens == 4
    assert E.build_arg_parser().parse_args(["--model-path", "m"]).prompt_lookup_num_tokens == 0


def test_region_chat_threads_the_option(monkeypatch):
    from spatialrgpt_b200 import chat as Ch
    monkeypatch.setattr(Ch, "process_images", lambda imgs, proc, cfg: torch.zeros(1, 3, 4, 4))
    monkeypatch.setattr(Ch, "tokenizer_image_token", lambda *a, **k: torch.tensor([1, 2, 3]))
    monkeypatch.setattr(Ch, "KeywordsStoppingCriteria", lambda *a, **k: None)
    tok = types.SimpleNamespace(batch_decode=lambda ids, skip_special_tokens=True: ["a b"])
    for k in (0, 3):
        m = _StubModel()
        c = Ch.RegionChat(m, tok, None, prompt_lookup_num_tokens=k)
        c.ask("what is <region0>?", None, [])
        assert m.calls[-1].get("prompt_lookup_num_tokens", 0) == k


def test_unsupported_combinations_raise_before_any_gpu_work():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2))
    m.llm = types.SimpleNamespace(supports_prompt_lookup=True)
    ids = torch.tensor([[1, 2, 3]])
    gen = LlavaLlamaModel.generate.__wrapped__.__wrapped__ if hasattr(LlavaLlamaModel.generate, "__wrapped__") else None
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")
    with pytest.raises(NotImplementedError, match="do_sample"):
        gen(m, ids, prompt_lookup_num_tokens=3, do_sample=True, temperature=0.7)
    with pytest.raises(NotImplementedError, match="beam"):
        gen(m, ids, prompt_lookup_num_tokens=3, num_beams=2)
    m.llm = types.SimpleNamespace(supports_prompt_lookup=False)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, ids, prompt_lookup_num_tokens=3)
    with pytest.raises(TypeError):
        gen(m, ids, assistant_model=object())
