"""Likelihood scoring on the CPU: the argument checks of srgpt_token_logprobs, its SASS, the shared-page bookkeeping of the paged KV
cache, the pass planner of LlamaDecoder.score_candidates, the candidate checks, and eval_region_cls --score-categories with a stub
model and tokenizer."""
import ctypes as C
import json
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from spatialrgpt_b200.llama_decoder import PAGE_SIZE, PagedKVCache, candidate_pages, check_candidates, plan_score_passes

BAD = -1


def _host(vals, ctype):
    return (ctype * len(vals))(*vals)


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_token_logprobs_rejects_bad_arguments_without_a_gpu(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    x = 16  # a non-NULL, 16-byte aligned address: every call below fails its argument check before anything is read or launched
    rows, tg = _host([0, 1], C.c_int), _host([5, -100], C.c_longlong)
    ok = [x, 104, 3, 100, rows, tg, 2, x, 16, x, x, x, None]
    for i, v in ((0, None), (10, None), (2, 0), (3, 0), (1, 99), (6, -1), (4, None), (5, None), (7, None), (9, None), (8, 15), (7, 20)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_token_logprobs(*args) == BAD, (i, v)
        assert b"invalid argument" in lib.srgpt_last_error()
    for r, t in (([0, 3], [5, 7]), ([-1, 0], [5, 7]), ([0, 1], [100, 7]), ([0, 1], [5, -1]), ([0, 1], [5, -101]), ([0, 1], [2 ** 40, 1])):
        args = list(ok)
        args[4], args[5] = _host(r, C.c_int), _host(t, C.c_longlong)
        assert lib.srgpt_token_logprobs(*args) == BAD, (r, t)
        assert b"outside 3 rows x 100 columns" in lib.srgpt_last_error()


def test_ops_wrapper_rejects_bad_arguments_without_a_gpu():
    from spatialrgpt_b200 import ops
    from spatialrgpt_b200._lib import SrgptError
    with pytest.raises(SrgptError, match="CUDA"):
        ops.token_logprobs(torch.zeros(3, 100, dtype=torch.bfloat16), [0], [1])  # CPU tensors never reach the library


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


def test_new_kernels_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    for elem in ("bf16", "f16"):
        _lib.load(elem=elem)
        funcs = _sass_functions(_lib.lib_path(elem))
        new = [f for f in funcs if "row_lse_kernel" in f or "pair_logprob_kernel" in f]
        assert len(new) == 2, new
        for f in new:
            body = "\n".join(funcs[f])
            assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"


# ---- shared KV pages -----------------------------------------------------------------------------------------------------------
def _cache(n_pages=40, max_seqs=2):
    from spatialrgpt_b200.config import LlamaDims
    d = LlamaDims(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1, head_dim=32,
                  vocab_size=100)
    return PagedKVCache(d, n_pages, max_seqs, 16, "cpu")


def test_forks_share_prompt_pages_and_release_only_their_own():
    c = _cache()
    c.reserve_many([35, 16])  # 3 pages (35 = 2 full + 3 rows), 1 page
    p0, p1 = c.table(0), c.table(1)
    assert len(p0) == 3 and len(p1) == 1
    forks = [c.fork(0, 2, 35 + n) for n in (1, 3, 13, 14, 30)]
    tables = [c.table(f) for f in forks]
    for t, n in zip(tables, (1, 3, 13, 14, 30)):
        assert t[:2] == p0[:2]  # the full pages are the prompt's
        assert not set(t[2:]) & (set(p0) | set(p1))  # everything a fork writes is its own
        assert len(t) == (35 + n + PAGE_SIZE - 1) // PAGE_SIZE
    owned = [p for t in tables for p in t[2:]]
    assert len(owned) == len(set(owned))
    f1 = c.fork(1, 1, 16 + 4)  # a prompt of exactly one page: everything after it is new
    assert c.table(f1)[0] == p1[0] and len(c.table(f1)) == 2
    with pytest.raises(RuntimeError, match="lends"):
        c.release(0)  # the forks still read its pages
    for f in forks + [f1]:
        c.release(f)
    assert sorted(c.free + c.table(0) + c.table(1)) == list(range(40))
    c.release(0)
    c.release(1)
    assert sorted(c.free) == list(range(40)) and len(c.free) == 40  # every page free, none twice
    assert not c.forks and not any(c.lent.values())


def test_fork_limits():
    c = _cache(n_pages=5)
    c.reserve_many([33])
    with pytest.raises(RuntimeError, match="cannot share"):
        c.fork(0, 4, 40)
    with pytest.raises(RuntimeError, match="exhausted"):
        c.fork(0, 2, 33 + 16 * 3)
    with pytest.raises(RuntimeError, match="capacity"):
        c.fork(0, 2, 16 * 17)
    assert len(c.free) == 2 and not c.forks


# ---- pass planner --------------------------------------------------------------------------------------------------------------
def _check_plan(seq_lens, cand_lens, budget, free, passes, max_chunks=65535):
    seen = []
    for p in passes:
        assert sum(n for _, _, _, n, _ in p) <= budget
        assert sum(own for *_, own in p) <= free
        assert len(p) <= max_chunks
        r = 0
        for b, c, r0, n, own in p:
            S = seq_lens[b]
            assert r0 == r and n == cand_lens[c] - 1 >= 1
            # exact page need: the pages of positions [S - S % 16, S + n) counted from the prompt's last full page
            assert own == len(range((S // PAGE_SIZE) * PAGE_SIZE, S + n, PAGE_SIZE)) == candidate_pages(S, n)[1]
            r += n
            seen.append((b, c))
    assert seen == [(b, c) for b in range(len(seq_lens)) for c in range(len(cand_lens)) if cand_lens[c] > 1]


@pytest.mark.parametrize("seq_lens", [[32], [259], [16, 47], [15, 1, 64]])
def test_planner_budgets_and_exact_page_need(seq_lens):
    rng = np.random.RandomState(len(seq_lens))
    cand_lens = [1, 2, 5, 17, 1, 3, 33] + rng.randint(1, 6, size=40).tolist()
    for budget, free in ((10 ** 6, 10 ** 6), (40, 10 ** 6), (10 ** 6, 5), (33, 3), (32, 3)):
        if budget < 32 or free < 3:
            continue
        passes = plan_score_passes(seq_lens, cand_lens, budget, free)
        _check_plan(seq_lens, cand_lens, budget, free, passes)
        if budget >= 10 ** 6 and free >= 10 ** 6:
            assert len(passes) == 1
    passes = plan_score_passes(seq_lens, cand_lens, 10 ** 6, 10 ** 6, max_chunks=7)
    _check_plan(seq_lens, cand_lens, 10 ** 6, 10 ** 6, passes, max_chunks=7)


def test_planner_page_need_at_page_boundaries():
    # S % 16 == 0: a candidate's rows start a fresh page; S % 16 != 0: the partial page is its own copy
    assert candidate_pages(32, 1) == (2, 1) and candidate_pages(32, 16) == (2, 1) and candidate_pages(32, 17) == (2, 2)
    assert candidate_pages(35, 1) == (2, 1) and candidate_pages(35, 13) == (2, 1) and candidate_pages(35, 14) == (2, 2)
    assert candidate_pages(5, 3) == (0, 1)  # a prompt shorter than a page shares nothing


def test_planner_one_token_candidates_get_no_rows_and_oversized_ones_raise():
    assert plan_score_passes([259, 40], [1, 1, 1], 8, 1) == []
    p = plan_score_passes([259], [1, 4, 1, 2], 100, 100)
    assert [(b, c, n) for b, c, _, n, _ in p[0]] == [(0, 1, 3), (0, 3, 1)]
    with pytest.raises(RuntimeError, match="needs 5 rows"):
        plan_score_passes([10], [6], 4, 100)
    with pytest.raises(RuntimeError, match="2 KV pages"):
        plan_score_passes([15], [3], 100, 1)


def test_candidate_checks():
    assert check_candidates([[1, 2], torch.tensor([3])], 10) == [[1, 2], [3]]
    for bad, msg in (([], "non-empty"), (None, "non-empty"), ([[1], []], "candidate 1 is empty"), ([[1, 10]], "outside"), ([[-1]], "outside")):
        with pytest.raises(ValueError, match=msg):
            check_candidates(bad, 10)


# ---- eval_region_cls --score-categories ------------------------------------------------------------------------------------------
def _annotations(tmp_path):
    from PIL import Image
    os.makedirs(tmp_path / "coco" / "val2017")
    Image.fromarray(np.random.RandomState(2).randint(0, 255, (60, 90, 3), dtype=np.uint8)).save(tmp_path / "coco" / "val2017" / "img1.jpg")
    coco = {"images": [{"id": 5, "height": 60, "width": 90, "coco_url": "http://x/val2017/img1.jpg"}],
            "categories": [{"id": 1, "name": "Dog"}, {"id": 2, "name": "hot dog"}, {"id": 3, "name": "cat"}],
            "annotations": [{"id": 1, "image_id": 5, "category_id": 1, "iscrowd": 0, "bbox": [10, 5, 30, 40], "segmentation": [[12, 8, 38, 8, 38, 40, 12, 40]]},
                            {"id": 2, "image_id": 5, "category_id": 3, "iscrowd": 0, "bbox": [50, 20, 20, 20], "segmentation": [[50, 20, 70, 20, 70, 40]]}]}
    (tmp_path / "ann.json").write_text(json.dumps(coco))
    return str(tmp_path / "ann.json")


def test_score_categories_writes_the_argmax(tmp_path):
    from transformers import SiglipImageProcessor

    from spatialrgpt_b200 import eval_region_cls as R
    from tests.golden.make_host_golden import ToyTokenizer
    ann = _annotations(tmp_path)
    tok = ToyTokenizer()
    seen = []
    pick = iter([2, 1])  # the candidate index the stub scores highest, per sample

    class Stub:
        device = torch.device("cpu")
        dtype = torch.float16
        config = SimpleNamespace(image_aspect_ratio="resize", mm_use_im_start_end=False)

        def score(self, input_ids, images=None, masks=None, candidates=None, **kw):
            assert images.dtype == torch.float16 and masks[0].dtype == torch.float16 and not kw
            seen.append((input_ids.clone(), candidates))
            s = torch.zeros(1, len(candidates))
            s[0, next(pick)] = 1.0
            return SimpleNamespace(sequence_logprobs=s)

        def generate(self, *a, **k):
            raise AssertionError("--score-categories does not generate")

    args = SimpleNamespace(model_path="m/tiny-cls", model_base=None, image_folder=str(tmp_path), annotation_file=ann,
                           answers_file=str(tmp_path / "ans.jsonl"), conv_mode="llava_v1", num_chunks=1, chunk_idx=0, temperature=0.0, top_p=None,
                           num_beams=1, dataset="lvis", prompt_type="seg", score_categories=True)
    assert R.eval_model(args, loader=lambda p, name, base: (tok, Stub(), SiglipImageProcessor(size={"height": 28, "width": 28}), 2048), seed=0) == 2
    rec = [json.loads(l) for l in open(args.answers_file)]
    assert [r["text"] for r in rec] == ["cat", "hot dog"] and [r["gt_name"] for r in rec] == ["dog", "cat"]
    ids, cands = seen[0]
    # each candidate is the tail of the prompt answered with the name: the name's words, the last one joined to the template's "</s>"
    # (the whitespace tokenizer keeps "dog</s>" as one token)
    assert cands == [[tok._id("dog</s>")], [tok._id("hot"), tok._id("dog</s>")], [tok._id("cat</s>")]]
    assert R.build_arg_parser().parse_args(["--model-path", "m", "--score-categories"]).score_categories


def test_candidate_ids_raise_when_the_prompt_is_not_a_prefix():
    from spatialrgpt_b200 import eval_region_cls as R
    from spatialrgpt_b200.conversation import conv_templates
    from tests.golden.make_host_golden import ToyTokenizer

    class Merging(ToyTokenizer):
        """Tokenises "ASSISTANT:" followed by text as one merged token, so the answered prompt does not start with the prompt's ids."""

        def __call__(self, text):
            return SimpleNamespace(input_ids=[self.bos_token_id] + [self._id(w) for w in text.replace("ASSISTANT: ", "ASSISTANT:").split()])

    conv = conv_templates["llava_v1"].copy()
    conv.append_message(conv.roles[0], "<image>\nwhat is <mask>?")
    conv.append_message(conv.roles[1], None)
    tok = ToyTokenizer()
    prompt = R.tokenizer_image_token(conv.get_prompt(), tok, R.IMAGE_TOKEN_INDEX, return_tensors="pt")
    assert R.candidate_ids(conv, ["dog", "hot dog"], tok, prompt) == [[tok._id("dog</s>")], [tok._id("hot"), tok._id("dog</s>")]]
    tok = Merging()
    prompt = R.tokenizer_image_token(conv.get_prompt(), tok, R.IMAGE_TOKEN_INDEX, return_tensors="pt")
    with pytest.raises(ValueError, match="not a prefix"):
        R.candidate_ids(conv, ["dog"], tok, prompt)


def test_tensor_parallel_decoder_does_not_score():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert not TPLlamaDecoder.supports_scoring
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        TPLlamaDecoder.score_candidates(object.__new__(TPLlamaDecoder), None, [1], [[1]], 8)
    m = object.__new__(LlavaLlamaModel)
    m.weights, m.llm = SimpleNamespace(dtype=torch.bfloat16), object.__new__(TPLlamaDecoder)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        m.score(torch.zeros(1, 4, dtype=torch.long), candidates=[[1]])
