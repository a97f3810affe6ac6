"""Host side of the prompt-prefix cache (generate(prefix_cache=True)): the reuse rule over splice plans, the decoder's record of
reusable prefill rows, and the C-ABI argument checks of the chunked-prefill kernels.  No GPU needed."""
import re
import subprocess

import pytest
import torch

from spatialrgpt_b200.constants import IMAGE_TOKEN_INDEX
from spatialrgpt_b200.conversation import conv_templates
from spatialrgpt_b200.mm_utils import tokenizer_image_token
from spatialrgpt_b200.splice_plan import SRC_IMAGE, SRC_MASK, build_splice_plan, reusable_prefix
from tests.golden.make_host_golden import ToyTokenizer

MASK_ID, DEPTH_ID, N_TOK = 500, 501, 9


class SubwordToyTokenizer(ToyTokenizer):
    """Whitespace words, split once more after a ':' (as a subword tokenizer splits 'ASSISTANT:USER:')."""

    def __call__(self, text):
        from types import SimpleNamespace
        words = [w for chunk in text.split() for w in re.findall(r"[^:]*:|[^:]+", chunk)]
        return SimpleNamespace(input_ids=[self.bos_token_id] + [self._id(w) for w in words])


def make_tok():
    tok = SubwordToyTokenizer()
    tok.vocab.update({"<mask>": MASK_ID, "<depth>": DEPTH_ID})
    return tok


def plan_of(ids, n_masks, depth=True):
    ids = torch.as_tensor(ids, dtype=torch.int64)[None]
    return build_splice_plan(ids, None, None, N_TOK, [n_masks], [True], MASK_ID, DEPTH_ID, True, depth)


def lcp(prev, new, image_equal=(True,), mask_equal=None, limit=None):
    n_masks = int((new.src_id == SRC_MASK).sum())
    mask_equal = [True] * max(n_masks, 8) if mask_equal is None else mask_equal
    limit = prev.src_id.numel() if limit is None else limit
    return reusable_prefix(prev.src_id, prev.src_row, new.src_id, new.src_row, N_TOK, list(image_equal), mask_equal, limit)


def turn_prompts(conv_mode, questions):
    conv, tok, out = conv_templates[conv_mode].copy(), make_tok(), []
    for q in questions:
        conv.append_message(conv.roles[0], q)
        conv.append_message(conv.roles[1], None)
        out.append(tokenizer_image_token(conv.get_prompt(), tok, IMAGE_TOKEN_INDEX, return_tensors="pt").tolist())
    return out


QUESTIONS = ["<image>\nhow far is <mask> <depth> from <mask> <depth> ?", "which is taller <mask> <depth> ?", "and <mask> <depth> wide ?"]


def test_pure_text_extension_reuses_the_whole_previous_prompt():
    a = plan_of([1, 20, 30, 40], 0)
    b = plan_of([1, 20, 30, 40, 50, 60], 0)
    assert lcp(a, b) == 4
    assert lcp(a, b, limit=3) == 3  # never more than the decoder still holds


@pytest.mark.parametrize("conv_mode", ["llava_v1", "llama_3"])
def test_multi_question_prompts_extend_the_previous_turn(conv_mode):
    """Each turn's prompt (TWO-style separators and llama_3 headers) starts with the whole previous prompt, image and
    region rows included, so everything but the new question is reused."""
    prompts = turn_prompts(conv_mode, QUESTIONS)
    plans = [plan_of(p, 2) for p in prompts]
    for k in range(2):
        assert prompts[k + 1][:len(prompts[k])] == prompts[k]
        n_prev = plans[k].src_id.numel()
        assert lcp(plans[k], plans[k + 1]) == n_prev
        assert int((plans[k].src_id[:n_prev] == SRC_IMAGE).sum()) == N_TOK


def test_changed_token_inside_the_prefix_stops_reuse_there():
    ids = turn_prompts("llama_3", QUESTIONS[:2])
    prev, new = list(ids[0]), list(ids[1])
    new[5] = new[5] + 1 if new[5] + 1 not in (MASK_ID, DEPTH_ID) else new[5] + 3
    assert lcp(plan_of(prev, 2), plan_of(new, 2)) == 5


def test_changed_image_reuses_no_image_row():
    prompts = turn_prompts("llama_3", QUESTIONS[:2])
    prev, new = plan_of(prompts[0], 2), plan_of(prompts[1], 2)
    first_image_row = int(torch.nonzero(new.src_id == SRC_IMAGE)[0, 0])
    assert lcp(prev, new, image_equal=[False]) == first_image_row
    assert first_image_row > 0


def test_changed_mask_stops_at_its_first_mask_row():
    prompts = turn_prompts("llama_3", QUESTIONS[:2])
    prev, new = plan_of(prompts[0], 2), plan_of(prompts[1], 2)
    rows_of_mask1 = torch.nonzero((new.src_id == SRC_MASK) & (new.src_row == 1)).flatten()
    assert lcp(prev, new, mask_equal=[True, False]) == int(rows_of_mask1[0])
    rows_of_mask0 = torch.nonzero((new.src_id == SRC_MASK) & (new.src_row == 0)).flatten()
    assert lcp(prev, new, mask_equal=[False, True]) == int(rows_of_mask0[0])
    assert int(rows_of_mask0[0]) < int(rows_of_mask1[0])


def test_reuse_is_capped_below_the_prompt_length():
    """The same prompt again: at most S - 1 rows are reused (the first new token needs the last row's hidden state)."""
    p = plan_of(turn_prompts("llama_3", QUESTIONS[:1])[0], 2)
    S = p.src_id.numel()
    assert lcp(p, p) == S
    assert lcp(p, p, limit=S - 1) == S - 1
    assert reusable_prefix(None, None, p.src_id, p.src_row, N_TOK, [True], [True, True], S - 1) == 0


def test_shorter_or_unrelated_prompt_reuses_nothing_past_the_difference():
    a = plan_of([1, 20, 30, 40, 50], 0)
    assert lcp(a, plan_of([1, 20, 30], 0)) == 3
    assert lcp(a, plan_of([2, 20, 30, 40, 50], 0)) == 0


def _stub_decoder(monkeypatch):
    """The bookkeeping half of LlamaDecoder over CPU tensors: the compute entry points are replaced by no-ops."""
    from spatialrgpt_b200 import llama_decoder as LD
    from spatialrgpt_b200 import ops
    monkeypatch.setattr(ops, "llama_prefill_layers", lambda x, *a, **k: x)
    monkeypatch.setattr(ops, "llama_prefill_chunk_layers", lambda x, *a, **k: x)
    d = LD.LlamaDecoder.__new__(LD.LlamaDecoder)
    d.dims = type("D", (), {"num_hidden_layers": 1, "num_key_value_heads": 1, "head_dim": 128})()
    d.device, d.dtype, d.max_seq_len = torch.device("cpu"), torch.bfloat16, 256
    d.cos = d.sin = d._layer_array = d.w = None
    d.prefix_rows, d.prefix_epoch = 0, 0
    d.cache = type("C", (), {})()
    d.cache.page_tables = torch.zeros((4, 17), dtype=torch.int32)
    d.cache.n_pages = 64
    d.cache.reserve = lambda seq, n: None
    return d


def test_record_is_invalidated_by_every_other_prefill(monkeypatch):
    """generate_batch / generate_beam / forward all prefill through prefill_packed or a fresh prefill_hidden; each of them
    drops the record, and the epoch moves so a model can tell that its cached prompt is gone."""
    d = _stub_decoder(monkeypatch)
    x = torch.zeros(10, 8)
    d._record_prefix(10)
    e0 = d.prefix_epoch
    d.prefill_packed(torch.zeros(12, 8), [5, 7])  # the batch and beam paths
    assert d.prefix_rows == 0 and d.prefix_epoch != e0
    d._record_prefix(10)
    e1 = d.prefix_epoch
    d.prefill_hidden(x, 0, 0)  # forward() at batch 1
    assert d.prefix_rows == 0 and d.prefix_epoch != e1
    d._record_prefix(10)
    d.prefill_hidden(x[:3], 0, 10)  # a chunk: the caller records the new length afterwards
    assert d.prefix_rows == 0


def test_reuse_rows_beyond_the_record_is_a_value_error(monkeypatch):
    d = _stub_decoder(monkeypatch)
    d._record_prefix(6)
    for bad in (7, 8, -1):  # more than recorded, the whole prompt (S - 1 = 7 at most), negative
        with pytest.raises(ValueError):
            d.generate_from_embeds(torch.zeros(8, 8), 4, reuse_rows=bad)
    with pytest.raises(ValueError):
        d.generate_from_embeds(torch.zeros(8, 8), 4, reuse_rows=3, seq=1)
    assert d.prefix_rows == 6  # a refused request leaves the record alone


# ---- C-ABI ------------------------------------------------------------------------------------------------------------------
P = 1 << 20  # a 16-byte aligned stand-in address: the checks below return before anything is dereferenced


def _paged(lib, **over):
    a = dict(q=P, q_ld=3 * 128 * 4, out=P, o_ld=128 * 4, kv_pages=P, n_pages=8, page_tables=P, stride=9, page_size=16, start_pos=P, cu=P,
             n_seqs=1, max_rows=4, total_rows=4, nh=4, nkv=2, hd=128)
    a.update(over)
    return lib.srgpt_attention_prefill_paged_bf16(a["q"], a["q_ld"], a["out"], a["o_ld"], a["kv_pages"], a["n_pages"], a["page_tables"], a["stride"],
                                                  a["page_size"], a["start_pos"], a["cu"], a["n_seqs"], a["max_rows"], a["total_rows"], a["nh"],
                                                  a["nkv"], a["hd"], 0.088, None)


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_paged_attention_rejects_unsupported_arguments_without_a_gpu(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    for bad in (dict(hd=64), dict(page_size=32), dict(q=None), dict(kv_pages=None), dict(page_tables=None), dict(start_pos=None), dict(cu=None),
                dict(nh=3, nkv=2), dict(total_rows=2)):
        assert _paged(lib, **bad) == -1, bad
        assert "invalid argument" in lib.srgpt_last_error().decode()
    assert lib.srgpt_rows_equal(None, P, 1, 16, P, None) == -1
    assert lib.srgpt_rows_equal(P, P, 0, 16, P, None) == -1


def test_chunk_composite_rejects_null_pointers_without_a_gpu():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    rc = lib.srgpt_llama_prefill_chunk_layers_bf16(P, P, 1, P, P, P, P, 4, 256, 2, 1, 128, 384, 1e-5, P, P, None, P, 9, 16, 8, 1, P, 4, None)
    assert rc == -1 and "invalid argument" in _lib.last_error()


def test_paged_attention_kernel_runs_on_wgmma_and_tma():
    """The paged kernel's own SASS carries the Hopper tensor-core (HGMMA) and TMA (UTMALDG) instructions."""
    from spatialrgpt_b200 import _lib
    _lib.load()
    r = subprocess.run(["cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    body = [f for f in funcs if f.startswith("_ZN5srgpt10attn_paged") and "attn_prefill_paged_kernel" in f.split("\n", 1)[0]]
    assert len(body) == 1, "paged attention kernel missing from the library"
    assert "HGMMA" in body[0] and "UTMALDG" in body[0]
