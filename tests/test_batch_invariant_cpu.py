"""generate(batch_invariant=True) on the CPU: the refusals, the seed list check, the grouping of large batches, the per-row prompts, budgets
and seeds handed to a host-only stand-in decoder, the host argument checks of the rows entry points, and their kernels' resource usage."""
import re
import subprocess
import types

import pytest
import torch

from spatialrgpt_b200.llama_decoder import sequence_seeds

V = 11


class HostDecoder:
    """A stand-in decoder on the host: generate_rows returns row b's first prompt id repeated, and records what it was called with."""
    supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_batch_sampling = True
    supports_output_scores = supports_batch_invariant = True
    fp8 = False
    dims = types.SimpleNamespace(vocab_size=V)

    def __init__(self):
        self.calls = []

    def embed_tokens(self, ids):
        return ids.reshape(-1, 1).float().repeat(1, 4)

    def generate_from_embeds(self, emb, n, **kw):
        self.calls.append(("one", int(emb.shape[0]), n, kw))
        return torch.full((n,), int(emb[0, 0]), dtype=torch.int64)

    def generate_batch(self, packed, lens, n, **kw):
        self.calls.append(("batch", lens, n, kw))
        return [torch.zeros(n, dtype=torch.int64) for _ in lens]

    def generate_rows(self, embeds, budgets, **kw):
        self.calls.append(("rows", [int(e.shape[0]) for e in embeds], list(budgets), kw))
        outs = [torch.full((n,), int(e[0, 0]), dtype=torch.int64) for e, n in zip(embeds, budgets)]
        return (outs, [torch.zeros(o.numel(), V) for o in outs]) if kw.get("return_logits") else outs


def _model(dec=None):
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")

    class M(LlavaLlamaModel):
        device = torch.device("cpu")

    m = M.__new__(M)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=None, vocab_size=V, pad_token_id=0, tokenizer_padding_side="left"))
    m.llm = HostDecoder() if dec is None else dec
    return gen, m


TWO = torch.tensor([[5, 6, 7], [1, 2, 3]])


@pytest.mark.parametrize("kw,what", [(dict(num_beams=2), "beam"), (dict(repetition_penalty=1.3), "processors"),
                                     (dict(prompt_lookup_num_tokens=3), "prompt_lookup"), (dict(prefix_cache=True), "prefix_cache"),
                                     (dict(do_sample=True, temperature=1.0, num_return_sequences=2), "num_return_sequences"),
                                     (dict(return_dict_in_generate=True, output_scores=True), "output_scores")])
def test_refusals_before_any_decoder_call(kw, what):
    gen, m = _model()
    with pytest.raises(NotImplementedError, match=what):
        gen(m, TWO, max_new_tokens=4, batch_invariant=True, **kw)
    assert m.llm.calls == []


def test_fp8_and_tensor_parallel_refused():
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert TPLlamaDecoder.supports_batch_invariant is False
    dec = HostDecoder()
    dec.fp8 = True
    gen, m = _model(dec)
    with pytest.raises(NotImplementedError, match="fp8"):
        gen(m, TWO, max_new_tokens=4, batch_invariant=True)
    dec = HostDecoder()
    dec.supports_batch_invariant = False
    gen, m = _model(dec)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, TWO, max_new_tokens=4, batch_invariant=True)
    assert dec.calls == []


def test_seed_list_checks():
    gen, m = _model()
    with pytest.raises(ValueError, match="2 prompts"):
        gen(m, TWO, max_new_tokens=4, batch_invariant=True, do_sample=True, temperature=1.0, seed=[1, 2, 3])
    with pytest.raises(ValueError, match="batch_invariant"):
        gen(m, TWO, max_new_tokens=4, do_sample=True, temperature=1.0, seed=[1, 2])
    assert m.llm.calls == []


def test_grouping_of_19_prompts_and_per_row_seeds():
    from spatialrgpt_b200.llava_llama import batch_invariant_groups
    assert batch_invariant_groups(19, 8) == [(0, 8), (8, 16), (16, 19)]
    assert batch_invariant_groups(8, 8) == [(0, 8)] and batch_invariant_groups(2, 8) == [(0, 2)]
    gen, m = _model()
    ids = torch.arange(19 * 4).view(19, 4) + 1
    out = gen(m, ids, max_new_tokens=3, batch_invariant=True, do_sample=True, temperature=0.7, seed=5)
    rows = [c for c in m.llm.calls if c[0] == "rows"]
    assert [len(c[1]) for c in rows] == [8, 8, 3]
    assert [s for c in rows for s in c[3]["seeds"]] == sequence_seeds(5, 19)
    assert all(c[3]["sampling"]["temperature"] == 0.7 for c in rows)
    assert out[:, 0].tolist() == ids[:, 0].tolist()
    m.llm.calls.clear()
    gen(m, ids[:3], max_new_tokens=3, batch_invariant=True, do_sample=True, temperature=0.7, seed=[9, 8, 7])
    assert m.llm.calls[0][3]["seeds"] == [9, 8, 7]


def test_unpadded_rows_and_their_own_budgets():
    gen, m = _model()
    ids = torch.tensor([[0, 0, 4, 5, 6], [7, 8, 9, 10, 11], [0, 3, 2, 1, 1]])
    mask = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [0, 1, 1, 1, 1]])
    out, lg = gen(m, ids, attention_mask=mask, max_length=9, batch_invariant=True, output_logits=True)
    (kind, lens, budgets, kw), = m.llm.calls
    assert kind == "rows" and lens == [3, 5, 4] and budgets == [6, 4, 5]
    assert out.tolist() == [[4] * 6, [7] * 4 + [0, 0], [3] * 5 + [0]] and [x.shape[0] for x in lg] == [6, 4, 5]
    # B = 1 takes the ordinary path
    m.llm.calls.clear()
    gen(m, ids[1:2], max_new_tokens=2, batch_invariant=True)
    assert m.llm.calls[0][0] == "one"


def _rows_step_args(B, ptr, pt_stride=41):
    """The arguments of srgpt_llama_decode_rows_bf16 at Llama-3-8B shapes, every buffer `ptr`."""
    return [ptr, ptr, 1, ptr, ptr, ptr, B, 4096, 32, 8, 128, 14336, 1e-5, ptr, ptr, ptr, ptr, pt_stride, 16, ptr, ptr, 128256] + [ptr] * 8 + [None]


def test_host_argument_checks_of_the_rows_entry_points():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    fake = 0x1000  # never dereferenced: every call below is refused on the host
    for B in (0, -1, 9):
        assert lib.srgpt_rows_advance(fake, 100, None, B, fake, fake, 16, fake, fake, fake, None) == -1
        assert lib.srgpt_attention_decode_rows_bf16(fake, 4096, fake, 4096, fake, fake, 41, 16, fake, B, 32, 8, 128, 0.1, None) == -1
        assert lib.srgpt_gemv_rows_bf16(fake, 4096, fake, 4096, fake, 4096, B, 6144, 4096, fake, 1e-5, 32, 8, 128, fake, fake, fake, fake, fake,
                                        41, 16, None) == -1
        assert lib.srgpt_llama_decode_rows_bf16(*_rows_step_args(B, fake)) == -1
    # null buffers, a null pos_rows, a zero page-table stride, a sampled step without its ids
    assert lib.srgpt_rows_advance(None, 100, None, 2, fake, fake, 16, fake, fake, fake, None) == -1
    assert lib.srgpt_gemv_rows_bf16(fake, 4096, fake, 4096, fake, 4096, 2, 6144, 4096, fake, 1e-5, 32, 8, 128, fake, fake, None, fake, fake, 41,
                                    16, None) == -1
    assert lib.srgpt_llama_decode_rows_bf16(*_rows_step_args(2, None)) == -1
    assert lib.srgpt_llama_decode_rows_bf16(*_rows_step_args(2, fake, pt_stride=0)) == -1
    args = _rows_step_args(2, fake)
    args[27] = None  # ids
    assert lib.srgpt_llama_decode_rows_bf16(*args) == -1
    packed = _rows_step_args(2, fake)
    assert lib.srgpt_llama_decode_rows_packed_bf16(*packed[:2], None, *packed[2:21], None, *packed[21:]) == -1  # no packed array


def test_signatures_match_the_header_argument_counts():
    import os
    from spatialrgpt_b200 import _lib
    src = open(os.path.join(os.path.dirname(__file__), "..", "include", "srgpt_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    for name in ("srgpt_gemv_rows_bf16", "srgpt_gemv_rows_packed_bf16", "srgpt_gemv_rows_nf4_bf16", "srgpt_attention_decode_rows_bf16",
                 "srgpt_rows_advance", "srgpt_llama_decode_rows_bf16", "srgpt_llama_decode_rows_packed_bf16", "srgpt_llama_decode_rows_nf4_bf16"):
        decl = re.search(name + r"\s*\(([^;]*)\);", src).group(1)
        assert len(decl.split(",")) == len(_lib.SIGNATURES[name][1]), name


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_rows_kernels_use_no_local_memory(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    r = subprocess.run(["cuobjdump", "-res-usage", _lib.lib_path(elem)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    found = {}
    lines = r.stdout.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*(rows_advance_kernel|gemv_multi_kernel|attn_decode_kernel)\S*):", line)
        if m:
            found[m.group(1)] = lines[i + 1]
    assert any("rows_advance" in k for k in found) and any("gemv_multi" in k for k in found) and any("attn_decode" in k for k in found)
    for fn, usage in found.items():
        assert "LOCAL:0" in usage and "STACK:0" in usage, (fn, usage)


# ---- the drivers' --batch-size ----------------------------------------------------------------------------------------------------
class _RowStub:
    """A stand-in model whose answer to a prompt depends on that prompt alone (its unpadded ids, image and masks), like
    generate(batch_invariant=True); batched calls pad the rows with pad_token_id."""
    device = torch.device("cpu")
    dtype = torch.float16

    def __init__(self, config):
        self.config = config
        self.calls = []

    def to(self, dtype=None, **kw):
        self.dtype = dtype or self.dtype
        return self

    def generate(self, input_ids, images=None, depths=None, masks=None, attention_mask=None, **kw):
        self.calls.append((input_ids.shape[0], kw.get("batch_invariant", False)))
        rows = []
        for b in range(input_ids.shape[0]):
            ids = input_ids[b] if attention_mask is None else input_ids[b][attention_mask[b].bool()]
            key = int(ids.abs().sum()) + int(images[b].float().sum() * 100) + (0 if masks is None or masks[b] is None else int(masks[b].sum()))
            rows.append([3 + (key + k) % 7 for k in range(1 + key % 4)])
        n = max(len(r) for r in rows)
        pad = kw.get("pad_token_id")
        return torch.tensor([r + [-1 if pad is None else pad] * (n - len(r)) for r in rows])


def _spatial_setup(tmp_path, n_ann=5):
    import json
    import numpy as np
    from PIL import Image
    from transformers import SiglipImageProcessor
    from tests.golden.make_host_golden import ToyTokenizer
    proc = SiglipImageProcessor(size={"height": 28, "width": 28})
    tok = ToyTokenizer()
    tok.batch_decode = lambda ids, skip_special_tokens=True: [" ".join(str(int(i)) for i in ids[0])]
    for i in range(3):
        Image.fromarray(np.random.RandomState(i).randint(0, 255, (20, 30, 3), dtype=np.uint8)).save(tmp_path / f"{i}.jpg")
    ann = []
    for i in range(n_ann):
        conv = [{"from": "human", "value": "<image>\nDistance between <mask> and <mask>?"}, {"from": "gpt", "value": "2 m"}]
        conv += [{"from": "human", "value": f"And is <mask> closer {i}?"}, {"from": "gpt", "value": "yes"}] * (i % 3)
        ann.append({"id": i, "image_info": {"file_path": f"{i % 3}.jpg", "height": 20, "width": 30}, "text_q": f"q{i}", "qa_info": {},
                    "bbox": [[1, 1, 10, 10], [5, 5, 25 - i, 18]], "conversations": conv})
    (tmp_path / "ann.json").write_text(json.dumps(ann))
    return proc, tok


def test_eval_spatial_batch_size_writes_the_batch1_records(tmp_path):
    from spatialrgpt_b200 import eval_spatial as E
    proc, tok = _spatial_setup(tmp_path)
    files = {}
    for bs in (1, 3):
        model = _RowStub(types.SimpleNamespace(image_aspect_ratio="resize"))
        args = types.SimpleNamespace(model_path="m/x", model_base=None, image_folder=str(tmp_path), annotation_file=str(tmp_path / "ann.json"),
                                     answers_file=str(tmp_path / f"a{bs}.jsonl"), conv_mode="llava_v1", num_chunks=1, chunk_idx=0, temperature=0.0,
                                     top_p=None, num_beams=1, use_mask=True, batch_size=bs)
        n = E.eval_model(args, depth_predictor=None, loader=lambda p, name, base: (tok, model, proc, 4096))
        files[bs] = open(args.answers_file, "rb").read()
        assert n == 1 + 2 + 3 + 1 + 2
        assert all(b == 1 for b, _ in model.calls) if bs == 1 else any(b == 3 and inv for b, inv in model.calls)
    assert files[1] == files[3]
    for bad in (dict(prefix_cache=True), dict(prompt_lookup_num_tokens=3), dict(num_beams=2)):
        args = types.SimpleNamespace(**dict(dict(num_beams=1, batch_size=3, model_path="m/x"), **bad))
        with pytest.raises(ValueError, match="--batch-size"):
            E.eval_model(args, depth_predictor=None, loader=lambda *a: pytest.fail("loaded a model"))


def test_eval_region_cls_batch_size_writes_the_batch1_records(tmp_path):
    import json
    import os
    import numpy as np
    from PIL import Image
    from transformers import SiglipImageProcessor
    from spatialrgpt_b200 import eval_region_cls as R
    from tests.golden.make_host_golden import ToyTokenizer
    os.makedirs(tmp_path / "coco" / "val2017")
    Image.fromarray(np.random.RandomState(2).randint(0, 255, (60, 90, 3), dtype=np.uint8)).save(tmp_path / "coco" / "val2017" / "img1.jpg")
    anns = [{"id": i + 1, "image_id": 5, "category_id": 1 + i % 2, "iscrowd": 0, "bbox": [5 + 3 * i, 5, 20, 20 + i],
             "segmentation": [[5 + 3 * i, 5, 25 + 3 * i, 5, 25 + 3 * i, 25 + i, 5 + 3 * i, 25 + i]]} for i in range(7)]
    coco = {"images": [{"id": 5, "height": 60, "width": 90, "coco_url": "http://x/val2017/img1.jpg"}],
            "categories": [{"id": 1, "name": "Dog"}, {"id": 2, "name": "cat"}], "annotations": anns}
    (tmp_path / "ann.json").write_text(json.dumps(coco))
    proc = SiglipImageProcessor(size={"height": 28, "width": 28})
    tok = ToyTokenizer()
    tok.batch_decode = lambda ids, skip_special_tokens=True: [" ".join(str(int(i)) for i in ids[0])]
    files = {}
    for bs in (1, 3):
        model = _RowStub(types.SimpleNamespace(image_aspect_ratio="resize", mm_use_im_start_end=False))
        args = types.SimpleNamespace(model_path="m/tiny-cls", model_base=None, image_folder=str(tmp_path), annotation_file=str(tmp_path / "ann.json"),
                                     answers_file=str(tmp_path / f"r{bs}.jsonl"), conv_mode="llava_v1", num_chunks=1, chunk_idx=0, temperature=0.0,
                                     top_p=None, num_beams=1, dataset="coco", prompt_type="seg", batch_size=bs)
        assert R.eval_model(args, loader=lambda p, name, base: (tok, model, proc, 2048), seed=3) == 7
        files[bs] = open(args.answers_file, "rb").read()
    assert files[1] == files[3]
    for bad in (dict(num_beams=2), dict(score_categories=True)):
        args = types.SimpleNamespace(**dict(dict(num_beams=1, batch_size=3), **bad))
        with pytest.raises(ValueError, match="--batch-size"):
            R.eval_model(args, loader=lambda *a: pytest.fail("loaded a model"))
