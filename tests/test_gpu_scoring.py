"""Likelihood scoring on the H100: the row log-softmax kernel against torch, forward(labels=)'s loss against F.cross_entropy over the
logits it returns and against the oracle, and score() against forward() on every prompt ++ candidate, in one pass and several, for
bf16, fp16, NF4 (both modes) and FP8 decoders."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import srgpt_oracle as O
from tests.golden.make_golden import CASES
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


def _build(name, dtype, seed=None, golden_dir=None):
    from tests.test_gpu_fp16 import build_model
    kw = CASES[name][0]
    if seed is None:
        seed = int(load_npz(os.path.join(golden_dir, name + ".npz"))["weight_seed"])
    return build_model(kw, seed, dtype=dtype)


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("offset", [0, 3])  # 3: every row starts off a 16-byte boundary (head, vectors and tail)
def test_kernel_against_log_softmax(dtype, offset):
    from spatialrgpt_b200 import ops
    R, V = 37, 128259
    g = torch.Generator().manual_seed(7 + offset)
    buf = torch.zeros(R, (V + offset + 7) // 8 * 8, dtype=dtype, device=DEV)
    buf[:, offset:offset + V].copy_((torch.randn(R, V, generator=g) * 4).to(dtype))
    x = buf[:, offset:offset + V]
    rows = torch.randint(0, R, (500,), generator=g)
    tg = torch.randint(0, V, (500,), generator=g)
    tg[::7] = -100
    with ops.elem_dtype(dtype):
        lse, lp, loss = ops.token_logprobs(x, rows, tg, loss=True)
        lse2, lp2, loss2 = ops.token_logprobs(x, rows, tg, loss=True)
    ref = torch.log_softmax(x.float(), -1)
    torch.testing.assert_close(lse, torch.logsumexp(x.float(), -1), atol=1e-5, rtol=1e-5)
    keep = tg != -100
    want = torch.zeros(500, device=DEV)
    want[keep.to(DEV)] = ref[rows[keep].to(DEV), tg[keep].to(DEV)]
    torch.testing.assert_close(lp, want, atol=1e-5, rtol=1e-5)
    assert bool((lp[~keep.to(DEV)] == 0).all())
    torch.testing.assert_close(loss, F.cross_entropy(x.float()[rows.to(DEV)], tg.to(DEV), ignore_index=-100), atol=1e-5, rtol=1e-5)
    assert torch.equal(lse, lse2) and torch.equal(lp, lp2) and torch.equal(loss, loss2)  # bit-identical repeats
    # a NaN makes its row NaN; no pair at all, or only ignored ones, gives a NaN loss
    buf[5, offset + 1000] = float("nan")
    with ops.elem_dtype(dtype):
        lse, lp, _ = ops.token_logprobs(x, [5, 6], [3, 3])
        assert bool(torch.isnan(lse[5])) and bool(torch.isnan(lp[0])) and not bool(torch.isnan(lse).sum() > 1)
        assert math.isnan(float(ops.token_logprobs(x, [0, 1], [-100, -100], loss=True)[2]))
        assert math.isnan(float(ops.token_logprobs(x, [], [], loss=True)[2]))


# ---- forward(labels=) --------------------------------------------------------------------------------------------------------------
def _shifted_ce(logits, labels):
    V = logits.shape[-1]
    return F.cross_entropy(logits[:, :-1].reshape(-1, V).float(), labels[:, 1:].reshape(-1).to(logits.device), ignore_index=-100)


def _labels(ids, seed):
    g = torch.Generator().manual_seed(seed)
    lab = ids.clone()
    lab[torch.rand(ids.shape, generator=g) < 0.3] = -100
    return lab


@pytest.mark.parametrize("name", ["tiny_boxes", "tiny_masks_gqa"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_forward_loss_multimodal(golden_dir, name, dtype):
    from tests.test_gpu_pipeline import _batch_requests
    oc, sd, model = _build(name, dtype, golden_dir=golden_dir)
    _, n_regions, t_text, kind, _, _ = CASES[name]
    ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    args = dict(images=images.to(DEV, dtype), depths=depths.to(DEV, dtype), masks=[m.to(DEV, dtype) for m in masks])
    lab = _labels(ids, 1)
    out = model.forward(input_ids=ids.to(DEV), labels=lab.to(DEV), **args)
    spliced = model.prepare_inputs_labels_for_multimodal(ids.to(DEV), None, None, None, lab.to(DEV), args["images"], args["masks"], args["depths"])[5]
    want = _shifted_ce(out.logits, spliced)
    assert out.loss.dtype == torch.float32 and out.loss.dim() == 0
    assert abs(float(out.loss) - float(want)) <= 1e-5 * abs(float(want))
    plain = model.forward(input_ids=ids.to(DEV), **args)
    assert plain.loss is None and torch.equal(plain.logits, out.logits)  # the logits are what forward returns without labels
    # against the oracle's fp32 logits: a log-prob moves at most twice the largest logit error (0.06 sigma)
    enc = O.encode_multimodal(oc, sd, images, depths, masks)
    emb = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), ids, enc["image_features"], enc["mask_embeds"],
                              enc["depth_embeds"])[0]
    ref, _ = O.llama_forward(oc, sd["llm"], emb, None)
    assert abs(float(out.loss) - float(_shifted_ce(ref[None], spliced.cpu()))) <= 2 * 0.06 * float(ref.std())
    # every label ignored: NaN, as CrossEntropyLoss
    none = model.forward(input_ids=ids.to(DEV), labels=torch.full_like(ids, -100).to(DEV), **args)
    assert math.isnan(float(none.loss))
    # a padded batch of two requests, either padding side
    reqs, bids, am, bimages, bdepths, bmasks = _batch_requests(oc, [(2, 24, 1234), (1, 19, 9)])
    blab = _labels(bids, 2)
    for side in ("right", "left"):
        model.config.llama.tokenizer_padding_side = side
        bargs = dict(images=bimages.to(DEV, dtype), depths=bdepths.to(DEV, dtype), masks=[m.to(DEV, dtype) for m in bmasks])
        o = model.forward(input_ids=bids.to(DEV), attention_mask=am.to(DEV), labels=blab.to(DEV), **bargs)
        sl = model.prepare_inputs_labels_for_multimodal(bids.to(DEV), None, am.to(DEV), None, blab.to(DEV), bargs["images"], bargs["masks"],
                                                        bargs["depths"])[5]
        # equal_nan: the random fp16 tiny_boxes weights overflow on one of these rows, and then the returned logits hold NaN too
        torch.testing.assert_close(o.loss, _shifted_ce(o.logits, sl), rtol=1e-5, atol=0, equal_nan=True, msg=side)
    model.config.llama.tokenizer_padding_side = "right"


@pytest.mark.parametrize("dtype", DTYPES)
def test_forward_loss_text_only_padded(dtype):
    oc, sd, model = _build("tiny_masks_gqa", dtype, seed=3)
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(3, 1000, (3, 21), generator=g)
    for left in (False, True):
        am = torch.ones(3, 21, dtype=torch.long)
        for b, n in enumerate((21, 14, 9)):
            if left:
                am[b, :21 - n] = 0
            else:
                am[b, n:] = 0
        lab = ids.clone()
        lab[am == 0] = -100
        lab[0, 5] = -100
        lab[1, 17 if not left else 3] = 17  # a label at a padding position scores the zero logits row forward returns there
        am_d = am.to(DEV)
        o = model.forward(input_ids=ids.to(DEV), attention_mask=am_d, labels=lab.to(DEV))
        want = _shifted_ce(o.logits, lab)
        assert abs(float(o.loss) - float(want)) <= 1e-5 * abs(float(want)), left
        one = model.forward(input_ids=ids[:1].to(DEV), labels=lab[:1].to(DEV))
        assert abs(float(one.loss) - float(_shifted_ce(one.logits, lab[:1]))) <= 1e-5 * float(one.loss)
    with pytest.raises(ValueError, match="labels"):
        model.forward(input_ids=ids.to(DEV), labels=lab[:, :5].to(DEV))


# ---- score() -----------------------------------------------------------------------------------------------------------------------
CAND_SETS = {
    "one_token": [[5], [17], [900], [5]],
    "mixed": [[5], [17, 40], [3, 4, 5], [900, 901, 902, 903], [11, 12, 13, 14, 15], [40, 17]],
    "page_crossing": [[7] * 12, [8, 9] * 7 + [1], [2] * 20, [3]],
}


def _forward_logprobs(model, prompt_ids, cands):
    """token log-probs read from forward() on each prompt ++ candidate, [N, L_max], and the std of the logits."""
    S = prompt_ids.numel()
    L = max(len(c) for c in cands)
    out = torch.zeros(len(cands), L)
    sig = []
    for i, c in enumerate(cands):
        full = torch.cat([prompt_ids, torch.tensor(c)])[None]
        lg = model.forward(input_ids=full.to(DEV)).logits[0].float()
        ls = torch.log_softmax(lg, -1).cpu()
        for j, t in enumerate(c):
            out[i, j] = ls[S - 1 + j, t]
        sig.append(float(lg.std()))
    return out, max(sig)


@pytest.mark.parametrize("dtype", DTYPES)
def test_score_text_prompts_against_forward(dtype, golden_dir):
    oc, sd, model = _build("tiny_masks_gqa", dtype, golden_dir=golden_dir)
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(3, 1000, (n,), generator=g) for n in (32, 37)]  # S % 16 == 0 and != 0
    llm = model.llm
    for cname, cands in CAND_SETS.items():
        refs = [_forward_logprobs(model, p, cands) for p in prompts]
        for b, p in enumerate(prompts):
            r = model.score(p[None].to(DEV), candidates=cands)
            ref, sig = refs[b]
            assert r.token_logprobs.shape == (1, len(cands), ref.shape[1]) and r.lengths.tolist() == [len(c) for c in cands]
            assert (r.token_logprobs[0].cpu() - ref).abs().max() <= 2 * 0.03 * sig, (cname, b)
            for i, c in enumerate(cands):
                assert bool((r.token_logprobs[0, i, len(c):] == 0).all())
            torch.testing.assert_close(r.sequence_logprobs, r.token_logprobs.sum(-1))
            assert len(llm.cache.free) == llm.cache.n_pages and not llm.cache.forks
        # B = 2, right- and left-padded
        T = 37
        for left in (False, True):
            ids = torch.zeros(2, T, dtype=torch.long)
            am = torch.zeros(2, T, dtype=torch.long)
            for b, p in enumerate(prompts):
                sl = slice(T - p.numel(), T) if left else slice(0, p.numel())
                ids[b, sl], am[b, sl] = p, 1
            r = model.score(ids.to(DEV), attention_mask=am.to(DEV), candidates=cands)
            for b in range(2):
                ref, sig = refs[b]
                assert (r.token_logprobs[b].cpu() - ref).abs().max() <= 2 * 0.03 * sig, (cname, b, left)
        # several passes (a forced small row budget) agree with one, and a repeat is bit-identical
        x = torch.cat([llm.embed_tokens(p.to(DEV)) for p in prompts])
        one = llm.score_candidates(x, [32, 37], cands, 1000)
        many = llm.score_candidates(x, [32, 37], cands, max(len(c) for c in cands) - 1 if cname != "one_token" else 1)
        assert (one - many).abs().max() <= 2 * 0.03 * refs[0][1]
        assert torch.equal(one, llm.score_candidates(x, [32, 37], cands, 1000))
        assert len(llm.cache.free) == llm.cache.n_pages


def test_score_multimodal_and_generate_afterwards(golden_dir):
    name = "tiny_masks_gqa"
    gold = load_npz(os.path.join(golden_dir, name + ".npz"))
    from tests.test_gpu_pipeline import build_model
    oc, sd, model = build_model(CASES[name][0], int(gold["weight_seed"]))
    _, n_regions, t_text, kind, n_new, _ = CASES[name]
    ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    args = dict(images=images.to(DEV), depths=depths.to(DEV), masks=[m.to(DEV) for m in masks])
    cands = CAND_SETS["mixed"]
    r = model.score(ids.to(DEV), candidates=cands, **args)
    assert len(model.llm.cache.free) == model.llm.cache.n_pages
    S = model._last_seq_lens[0]
    ref = torch.zeros_like(r.token_logprobs[0]).cpu()
    sig = 0.0
    for i, c in enumerate(cands):
        full = torch.cat([ids[0], torch.tensor(c)])[None]
        lg = model.forward(input_ids=full.to(DEV), **args).logits[0].float()
        ls = torch.log_softmax(lg, -1).cpu()
        for j, t in enumerate(c):
            ref[i, j] = ls[S - 1 + j, t]
        sig = max(sig, float(lg.std()))
    assert (r.token_logprobs[0].cpu() - ref).abs().max() <= 2 * 0.03 * sig
    # the cache is whole again: generate() still returns the fixture's ids
    out = model.generate(ids.to(DEV), do_sample=False, max_new_tokens=n_new, **args)
    assert out[0].tolist() == gold["new_ids"].tolist()


def test_score_rejections():
    oc, sd, model = _build("tiny_boxes", torch.bfloat16, seed=3)
    p = torch.randint(3, 500, (1, 20))
    for bad, msg in (([], "non-empty"), ([[3], []], "empty"), ([[3, 512]], "outside"), ([[3] * 493], "max_seq_len")):
        with pytest.raises(ValueError, match=msg):
            model.score(p.to(DEV), candidates=bad)
    assert model.score(p.to(DEV), candidates=[[3] * 492]).token_logprobs.shape == (1, 1, 492)  # 20 + 492 = max_seq_len 512


# ---- quantized decoders ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_quantized_decoders_against_their_own_forward(dtype):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_beam_batch import _dims
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    lens = [133, 48]
    g = torch.Generator().manual_seed(3)
    x = torch.cat([(torch.randn(n, d.hidden_size, generator=g) * 0.3) for n in lens]).to(dtype).to(DEV)
    cands = [[5], [17, 40], [3, 4, 5], [900, 901, 902, 903, 904], [7] * 18]

    def check(dec, fp8=False):
        got = dec.score_candidates(x, lens, cands, 20)  # several passes
        assert len(dec.cache.free) == dec.cache.n_pages
        o, diffs = 0, []
        for b, S in enumerate(lens):
            for i, c in enumerate(cands):
                full = torch.cat([x[o:o + S], dec.embed_tokens(torch.tensor(c[:-1], dtype=torch.int64))]) if len(c) > 1 else x[o:o + S]
                lg = dec.logits_all(dec.prefill_hidden(full, 0, 0))
                ls = torch.log_softmax(lg, -1)
                ref = torch.stack([ls[S - 1 + j, t] for j, t in enumerate(c)])
                d = (got[b, i, :len(c)] - ref).abs() / float(lg.std())
                diffs.append(d)
                if not fp8:
                    assert float(d.max()) <= 2 * 0.03, (b, i)
            o += S
        if fp8:
            # E4M3 activations: the chunked rows' attention rounds differently from the full prefill's, and an activation moved by one ulp
            # across an E4M3 boundary changes its code by an eighth of its value; test_gpu_fp8.py bounds that path difference by 0.8 sigma
            # max and 0.15 sigma rms on the logits, doubled here for log-probs
            d = torch.cat(diffs)
            assert float(d.max()) <= 2 * 0.8 and float(d.pow(2).mean().sqrt()) <= 2 * 0.15, (float(d.max()), float(d.pow(2).mean().sqrt()))
        return got

    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512)
    assert dec.fp8
    check(dec, fp8=True)
    del dec
    sd = _llm_state_dict(d, 21)
    res = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512)
        assert dec.nf4_planes_only == (not copy)
        res[copy] = check(dec)
        del dec
    assert torch.equal(res[True], res[False])  # planes-only is bit-identical to copy mode
