"""Chunked prefill over the paged KV cache and prompt-prefix reuse (generate(prefix_cache=True)) on the H100: the paged attention
kernel against fp32 torch, chunked vs one-pass prefill through the decoder, and multi-turn requests with and without the cache
against each other and against the CPU oracle."""
import numpy as np
import pytest
import torch

from oracle import srgpt_oracle as O
from tests.golden.make_golden import CASES
from tests.golden.make_host_golden import ToyTokenizer
from tests.test_gpu_pipeline import build_model
from tests.util import BF16_STAGE, assert_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
HD, PAGE = 128, 16
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def paged_case(nh, nkv, lens, starts, dtype, seed=0):
    """Random cache contents for positions [0, start + len) of each sequence over a random permutation of physical pages, and
    q rows as the q columns of a fused qkv buffer."""
    g = torch.Generator().manual_seed(seed)
    cap = max((s + n + PAGE - 1) // PAGE for s, n in zip(starts, lens)) + 1
    n_pages = len(lens) * cap + 3
    perm = torch.randperm(n_pages, generator=g)[:len(lens) * cap].to(torch.int32).view(len(lens), cap)
    pages = (torch.randn(n_pages, 2, PAGE, nkv, HD, generator=g) * 0.5).to(dtype)
    qkv = (torch.randn(sum(lens), (nh + 2 * nkv) * HD, generator=g) * 0.5).to(dtype)
    return qkv, pages, perm


def reference(qkv, pages, perm, lens, starts, nh, nkv):
    """Dense fp32 softmax over the gathered cache rows of every chunk."""
    out, o, grp = [], 0, nh // nkv
    pf = pages.float()
    for b, (n, s) in enumerate(zip(lens, starts)):
        P = s + n
        pos = torch.arange(P)
        rows = pf[perm[b, pos // PAGE].long(), :, pos % PAGE]  # [P, 2, nkv, HD]
        k = rows[:, 0].repeat_interleave(grp, dim=1)  # [P, nh, HD]
        v = rows[:, 1].repeat_interleave(grp, dim=1)
        q = qkv[o:o + n, :nh * HD].float().view(n, nh, HD)
        sc = torch.einsum("rhd,phd->hrp", q, k) * HD ** -0.5
        sc = sc.masked_fill(pos[None, None, :] > (s + torch.arange(n))[None, :, None], float("-inf"))
        out.append(torch.einsum("hrp,phd->rhd", sc.softmax(-1), v).reshape(n, nh * HD))
        o += n
    return torch.cat(out)


def run_paged(ops, qkv, pages, perm, lens, starts, nh, nkv):
    cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=DEV)
    sp = torch.tensor(starts, dtype=torch.int32, device=DEV)
    q = qkv.to(DEV)
    return ops.attention_prefill_paged(q[:, :nh * HD], pages.to(DEV), perm.to(DEV), PAGE, sp, cu, max(lens), nh, nkv, HD, HD ** -0.5)


@pytest.mark.parametrize("elem", list(DTYPES))
@pytest.mark.parametrize("nh,nkv", [(32, 8), (4, 2), (2, 1)])
@pytest.mark.parametrize("start", [0, 1, 15, 16, 17, 259, 1000])
def test_paged_attention_matches_fp32(ops, elem, nh, nkv, start):
    dtype = DTYPES[elem]
    with ops.elem_dtype(dtype):
        for n in (1, 7, 30, 64, 127, 128, 129, 300):
            qkv, pages, perm = paged_case(nh, nkv, [n], [start], dtype, seed=start * 1000 + n)
            out = run_paged(ops, qkv, pages, perm, [n], [start], nh, nkv)
            assert_close(out, reference(qkv, pages, perm, [n], [start], nh, nkv), rel_rms=1e-2, rel_max=8e-2,
                         what=f"paged attention {elem} nh{nh}/{nkv} start {start} rows {n}")


@pytest.mark.parametrize("elem", list(DTYPES))
def test_packed_chunks_equal_single_chunk_calls(ops, elem):
    dtype, nh, nkv = DTYPES[elem], 32, 8
    lens, starts = [30, 129, 7], [259, 16, 1000]
    with ops.elem_dtype(dtype):
        qkv, pages, perm = paged_case(nh, nkv, lens, starts, dtype, seed=11)
        packed = run_paged(ops, qkv, pages, perm, lens, starts, nh, nkv)
        assert_close(packed, reference(qkv, pages, perm, lens, starts, nh, nkv), rel_rms=1e-2, rel_max=8e-2, what="packed chunks")
        o = 0
        for b, (n, s) in enumerate(zip(lens, starts)):
            one = run_paged(ops, qkv[o:o + n].contiguous(), pages, perm[b:b + 1], [n], [s], nh, nkv)
            assert torch.equal(one, packed[o:o + n]), f"chunk {b} differs between the packed and the single call"
            o += n


@pytest.mark.parametrize("elem", list(DTYPES))
def test_start_zero_agrees_with_the_varlen_kernel(ops, elem):
    """With start_pos 0 the cache holds exactly the chunk's own K/V: the dense varlen kernel over the fused buffer computes the
    same attention (within one rounding)."""
    dtype, nh, nkv, n = DTYPES[elem], 4, 2, 300
    with ops.elem_dtype(dtype):
        qkv, pages, perm = paged_case(nh, nkv, [n], [0], dtype, seed=5)
        pos = torch.arange(n)
        rows = pages[perm[0, pos // PAGE].long(), :, pos % PAGE]  # the cached k / v of every row, into the fused buffer
        qkv[:, nh * HD:(nh + nkv) * HD] = rows[:, 0].reshape(n, nkv * HD)
        qkv[:, (nh + nkv) * HD:] = rows[:, 1].reshape(n, nkv * HD)
        paged = run_paged(ops, qkv, pages, perm, [n], [0], nh, nkv)
        d = qkv.to(DEV)
        cu = torch.tensor([0, n], dtype=torch.int32, device=DEV)
        dense = ops.attention_prefill_varlen(d[:, :nh * HD], d[:, nh * HD:(nh + nkv) * HD], d[:, (nh + nkv) * HD:], cu, n, nh, nkv, HD,
                                             HD ** -0.5, True)
        assert_close(paged, dense, rel_rms=4e-3, rel_max=5e-2, what="paged vs varlen at start 0")


# ---- decoder: chunked prefill vs one pass ----------------------------------------------------------------------------------
SPLITS = [1, 100, 128, 159, 299]


def test_chunked_prefill_matches_one_pass():
    kw = CASES["tiny_masks_gqa"][0]
    oc, sd, model = build_model(kw, 23)
    llm, S = model.llm, 300
    emb = (torch.randn(S, oc.hidden, generator=torch.Generator().manual_seed(1)) * 0.05).to(DEV, model.dtype)
    full = llm.prefill_hidden(emb, 0, 0).clone()
    pages_full = llm.cache.pages.clone()
    pt_full = list(llm.cache.owned[0])
    llm.cache.release(0)
    parts, lo = [], 0
    for hi in SPLITS + [S]:
        parts.append(llm.prefill_hidden(emb[lo:hi], 0, lo).clone())
        lo = hi
    chunked = torch.cat(parts)
    assert_close(chunked, full, **BF16_STAGE, what="final hidden state, chunked vs one pass")
    assert list(llm.cache.owned[0]) == pt_full  # the same physical pages: compare every layer's K/V rows directly
    n_pg = (S + PAGE - 1) // PAGE
    for l in range(oc.layers):
        a = pages_full[l, pt_full[:n_pg]].transpose(0, 1).reshape(2, -1)[:, :S * oc.kv_heads * HD]
        b = llm.cache.pages[l, pt_full[:n_pg]].transpose(0, 1).reshape(2, -1)[:, :S * oc.kv_heads * HD]
        assert_close(b, a, **BF16_STAGE, what=f"layer {l} KV pages")


def test_generate_continuing_a_prefix_matches_a_full_prefill():
    kw = CASES["tiny_masks_gqa"][0]
    oc, sd, model = build_model(kw, 29)
    llm, S, n_new = model.llm, 300, 12
    emb = (torch.randn(S, oc.hidden, generator=torch.Generator().manual_seed(2)) * 0.05).to(DEV, model.dtype)
    ids_full, lg_full = llm.generate_from_embeds(emb, n_new, return_logits=True)
    # oracle: greedy ids are compared where the fp32 reference's top-1 / top-2 margin is clear
    ref_ids, ref_lg = O.greedy_generate(oc, sd["llm"], emb.float().cpu(), n_new, return_logits=True)
    sigma = float(ref_lg.std())
    for split in SPLITS:
        llm.generate_from_embeds(emb[:split], 1)  # records `split` prefill rows
        assert llm.prefix_rows == split
        reuse = min(split, S - 1)
        ids, lg = llm.generate_from_embeds(emb, n_new, return_logits=True, reuse_rows=reuse)
        assert llm.prefix_rows == S
        assert float((lg.cpu() - lg_full.cpu()).abs().max()) <= 0.06 * sigma, f"split {split}: logits"
        assert ids.tolist() == ids_full.tolist(), f"split {split}: greedy ids"
        # graph decode after a chunked prefill equals eager decode
        llm.generate_from_embeds(emb[:split], 1)
        ids_graph = llm.generate_from_embeds(emb, n_new, reuse_rows=reuse, use_graph=True)
        assert ids_graph.tolist() == ids.tolist(), f"split {split}: graph vs eager decode"
    top2 = ref_lg.topk(2, -1).values
    safe = int(((top2[:, 0] - top2[:, 1]) > 0.08 * sigma).long().cumprod(0).sum())
    assert ids_full.tolist()[:safe] == ref_ids.tolist()[:safe]
    with pytest.raises(ValueError):
        llm.generate_from_embeds(emb, 2, reuse_rows=S)  # at most S - 1 rows


# ---- pipeline: multi-turn requests -----------------------------------------------------------------------------------------
PIPE_CASES = ["tiny_boxes", "tiny_masks_gqa", "tiny_nodepth"]
QUESTIONS = ["<image>\n how far is <mask> from <mask> ?", "which one is taller <mask> ?", "and how wide is <mask> ?"]


def pipeline_setup(name):
    from PIL import Image
    from transformers import SiglipImageProcessor
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    oc, sd, model = build_model(kw, 31)
    proc = SiglipImageProcessor(size={"height": oc.image_size, "width": oc.image_size})
    model.config.image_aspect_ratio = "resize"
    tok = ToyTokenizer()
    tok.vocab.update({"<mask>": oc.mask_token_id, "<depth>": oc.depth_token_id})
    tok.batch_decode = lambda ids, skip_special_tokens=True: [" ".join(str(int(i)) for i in ids[0])]
    rs = np.random.RandomState(3)
    image = Image.fromarray(rs.randint(0, 255, (40, 60, 3), dtype=np.uint8))
    depth = Image.fromarray(rs.randint(0, 255, (40, 60, 3), dtype=np.uint8)) if depth_on else None
    line = {"id": 1, "text_q": "q", "qa_info": {}, "conversations": []}
    for q in QUESTIONS:
        line["conversations"] += [{"from": "human", "value": q}, {"from": "gpt", "value": "gt"}]
    masks = torch.zeros(4, oc.image_size, oc.image_size)  # one per <mask> of the three questions, as the driver passes them
    for m, (y0, y1, x0, x1) in enumerate([(2, 20, 3, 30), (10, 40, 5, 25), (0, 12, 0, 50), (30, 55, 20, 40)]):
        masks[m, y0:y1, x0:x1] = 1
    return oc, sd, model, proc, tok, image, depth, line, masks


def turn_requests(model, proc, tok, image, depth, masks, conv_mode="llama_3"):
    """The tensors answer_questions builds for each turn."""
    from spatialrgpt_b200 import eval_spatial as E
    from spatialrgpt_b200.conversation import conv_templates
    from spatialrgpt_b200.mm_utils import process_images, tokenizer_image_token
    imgs = process_images([image], proc, model.config).to(DEV, dtype=model.dtype)
    deps = None if depth is None else process_images([depth], proc, model.config).to(DEV, dtype=model.dtype)
    conv, out = conv_templates[conv_mode].copy(), []
    for q in QUESTIONS:
        conv.append_message(conv.roles[0], E.question_with_depth_tokens(q) if depth is not None else q)
        conv.append_message(conv.roles[1], None)
        ids = tokenizer_image_token(conv.get_prompt(), tok, -200, return_tensors="pt").unsqueeze(0)
        out.append(ids)
    return imgs, deps, out


@pytest.mark.parametrize("name", PIPE_CASES)
def test_three_question_annotation_with_and_without_prefix_cache(name):
    from spatialrgpt_b200 import eval_spatial as E
    oc, sd, model, proc, tok, image, depth, line, masks = pipeline_setup(name)
    plain = E.answer_questions(line, model, tok, proc, image, depth, masks, "llama_3", "tiny", "a.jpg", max_new_tokens=8)
    reuse = []
    orig = model.generate

    def recording(*a, **k):
        r = orig(*a, **k)
        reuse.append(model.last_prefix_reuse)
        return r
    model.generate = recording
    cached = E.answer_questions(line, model, tok, proc, image, depth, masks, "llama_3", "tiny", "a.jpg", max_new_tokens=8, prefix_cache=True)
    model.generate = orig
    assert [r["pred"] for r in cached] == [r["pred"] for r in plain]

    imgs, deps, turns = turn_requests(model, proc, tok, image, depth, masks)
    md = [masks.to(DEV, dtype=model.dtype)]
    n_tok = model._tokens_per_image()
    rows = [int(t.shape[1]) - 1 + n_tok for t in turns]  # prompt rows: the <image> slot becomes n_tok rows
    assert reuse[0] == (0, rows[0], False)
    for k in (1, 2):
        assert reuse[k] == (rows[k - 1], rows[k] - rows[k - 1], True), f"turn {k + 1}: {reuse[k]}"

    # per-turn logits: cached vs plain, and both vs the CPU oracle's full re-prefill of the turn's whole prompt
    for k, ids in enumerate(turns):
        args = dict(images=imgs, depths=deps, masks=md, do_sample=False, max_new_tokens=4, output_logits=True)
        p_ids, p_lg = model.generate(ids.to(DEV), **args)
        c_ids, c_lg = model.generate(ids.to(DEV), prefix_cache=True, **args)
        ref_ids, enc = O.generate(oc, sd, ids, imgs.float().cpu(), None if deps is None else deps.float().cpu(), [masks], 4, return_all=True)
        sigma = float(enc["logits"].std())
        assert float((c_lg[0] - p_lg[0]).abs().max()) <= 0.06 * sigma, f"turn {k + 1}: cached vs plain logits"
        assert float((c_lg[0].cpu() - enc["logits"]).abs().max()) <= 0.06 * sigma, f"turn {k + 1}: cached vs oracle logits"
        top2 = enc["logits"].topk(2, -1).values
        safe = int(((top2[:, 0] - top2[:, 1]) > 0.08 * sigma).long().cumprod(0).sum())
        assert c_ids[0].tolist()[:safe] == ref_ids.tolist()[:safe] == p_ids[0].tolist()[:safe]


def assert_same_answer(c, p, what):
    """Cached vs plain request: logits within 0.06 sigma, greedy ids equal up to the first step whose top-1 / top-2 margin is
    within the noise (the new rows differ from a full prefill by rounding)."""
    (c_ids, c_lg), (p_ids, p_lg) = c, p
    n = min(c_lg[0].shape[0], p_lg[0].shape[0])
    sigma = float(p_lg[0].float().std())
    assert float((c_lg[0][:n] - p_lg[0][:n]).abs().max()) <= 0.06 * sigma, f"{what}: logits"
    top2 = p_lg[0][:n].topk(2, -1).values
    safe = int(((top2[:, 0] - top2[:, 1]) > 0.08 * sigma).long().cumprod(0).sum())
    assert c_ids[0].tolist()[:safe] == p_ids[0].tolist()[:safe], f"{what}: greedy ids"


def _requests(name):
    oc, sd, model, proc, tok, image, depth, line, masks = pipeline_setup(name)
    imgs, deps, turns = turn_requests(model, proc, tok, image, depth, masks)
    return oc, model, imgs, deps, turns, masks


def test_fallbacks_reuse_what_is_unchanged_and_match_the_plain_path_bitwise():
    oc, model, imgs, deps, turns, masks = _requests("tiny_masks_gqa")
    md = masks.to(DEV, dtype=model.dtype)
    n_tok = model._tokens_per_image()
    args = dict(do_sample=False, max_new_tokens=6, output_logits=True)
    first, second = turns[0].to(DEV), turns[1].to(DEV)
    S1, S2 = first.shape[1] - 1 + n_tok, second.shape[1] - 1 + n_tok
    img_row = int((turns[1][0] == -200).nonzero()[0, 0])  # the first image row

    def pair(ids, images, masks_, first_images=None, first_masks=None):
        model.generate(first, images=imgs if first_images is None else first_images, depths=deps, masks=[md if first_masks is None else first_masks],
                       prefix_cache=True, **args)
        c = model.generate(ids, images=images, depths=deps, masks=[masks_], prefix_cache=True, **args)
        info = model.last_prefix_reuse
        p = model.generate(ids, images=images, depths=deps, masks=[masks_], **args)
        return c, p, info

    # one changed pixel: no image row is reused, the encoders run again
    px = imgs.clone()
    px[0, 1, 5, 7] += 0.25
    c, p, info = pair(second, px, md)
    assert info == (img_row, S2 - img_row, False)
    assert_same_answer(c, p, "changed pixel")
    # a changed earlier mask: the prefix stops at that mask's first row, pooling reruns, encoders are skipped
    m2 = md.clone()
    m2[1, 0, 0] = 1 - m2[1, 0, 0]
    c, p, info = pair(second, imgs, m2)
    ids_rows = second[0].tolist()
    mask_tok = [i for i, t in enumerate(ids_rows) if t == oc.mask_token_id]
    first_mask1_row = mask_tok[1] - 1 + n_tok  # second <mask> of the prompt = region 1, after the image slot
    assert info == (first_mask1_row, S2 - first_mask1_row, True)
    assert_same_answer(c, p, "changed mask")
    # a changed earlier token
    tweaked = second.clone()
    pos = img_row + 3
    tweaked[0, pos] = tweaked[0, pos] + 1
    c, p, info = pair(tweaked, imgs, md)
    assert info == (pos - 1 + n_tok, S2 - (pos - 1 + n_tok), True)
    assert_same_answer(c, p, "changed token")
    # a different first token and image: nothing is reused, and the request is the plain path bit for bit
    ids0 = second.clone()
    ids0[0, 0] = ids0[0, 0] + 1
    c, p, info = pair(ids0, px, md)
    assert info == (0, S2, False)
    assert torch.equal(c[0], p[0]) and torch.equal(c[1][0], p[1][0])
    assert S1 < S2


def test_other_requests_in_between_drop_the_reuse():
    oc, model, imgs, deps, turns, masks = _requests("tiny_boxes")
    md = [masks.to(DEV, dtype=model.dtype)]
    args = dict(images=imgs, depths=deps, masks=md, do_sample=False, max_new_tokens=4)
    first, second = turns[0].to(DEV), turns[1].to(DEV)
    between = [
        lambda: model.generate(torch.cat([first, first]), images=torch.cat([imgs, imgs]), depths=torch.cat([deps, deps]), masks=md * 2,
                               do_sample=False, max_new_tokens=3),  # generate_batch
        lambda: model.generate(first, num_beams=2, **args),
        lambda: model.forward(input_ids=first, images=imgs, masks=md, depths=deps),
        lambda: model.generate(second, **args),  # a plain batch-1 request over other rows
    ]
    for other in between:
        model.generate(first, prefix_cache=True, **args)
        other()
        model.generate(second, prefix_cache=True, **args)
        assert model.last_prefix_reuse[0] == 0 and model.last_prefix_reuse[2] is True


def test_region_chat_follow_up_with_new_masks():
    from PIL import Image
    from transformers import SiglipImageProcessor

    from spatialrgpt_b200.chat import RegionChat
    kw = CASES["tiny_boxes"][0]
    oc, sd, model = build_model(kw, 37)
    model.config.image_aspect_ratio = "resize"
    proc = SiglipImageProcessor(size={"height": oc.image_size, "width": oc.image_size})
    tok = ToyTokenizer()
    tok.vocab.update({"<mask>": oc.mask_token_id, "<depth>": oc.depth_token_id})
    rs = np.random.RandomState(4)
    img = Image.fromarray(rs.randint(0, 255, (40, 50, 3), dtype=np.uint8))
    depth = Image.fromarray(rs.randint(0, 255, (40, 50, 3), dtype=np.uint8))
    segs = [np.zeros((40, 50), dtype=np.uint8) for _ in range(4)]
    for i, s in enumerate(segs):
        s[5 * i:5 * i + 8, 4:20] = 1
    answers, infos = {}, []
    for cache in (False, True):
        chat = RegionChat(model, tok, proc, conv_mode="llava_v1", max_new_tokens=6, prefix_cache=cache)
        a1 = chat.ask("Is <region2> behind <region0> ?", img, segs, depth_image=depth)
        infos.append(model.last_prefix_reuse)
        a2 = chat.ask("And how wide is <region3> ?", img, segs, depth_image=depth, follow_up=True)  # a third mask joins
        infos.append(model.last_prefix_reuse)
        answers[cache] = (a1, a2)
    assert answers[True] == answers[False]
    assert infos[3][2] is True and infos[3][0] > 0  # the follow-up: encoders skipped, pooling rerun over the 3 masks


def test_batch_beam_and_tensor_parallel_are_refused():
    oc, model, imgs, deps, turns, masks = _requests("tiny_boxes")
    md = [masks.to(DEV, dtype=model.dtype)]
    first = turns[0].to(DEV)
    with pytest.raises(NotImplementedError):
        model.generate(torch.cat([first, first]), images=torch.cat([imgs, imgs]), depths=torch.cat([deps, deps]), masks=md * 2, prefix_cache=True)
    with pytest.raises(NotImplementedError):
        model.generate(first, images=imgs, depths=deps, masks=md, num_beams=2, prefix_cache=True)
