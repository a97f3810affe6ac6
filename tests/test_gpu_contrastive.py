"""Contrastive search on the H100 (LlamaDecoder.generate_contrastive, generate(penalty_alpha=, top_k=)): the penalty and select kernels
against a float64 torch restatement, the KV broadcast against torch indexing of the page pool, every prompt against the 4.37.2 loop over
HF's LlamaForCausalLM (tests/golden/contrastive_kats.npz), the limit alpha -> 0 against greedy generate(), graph against eager, a prompt's
ids against its batch, the stopping rules, output_scores, the multimodal API against tests/contrastive_oracle.py and the quantized weight
formats.  Both element types."""
import dataclasses
import os

import numpy as np
import pytest
import torch

from oracle import srgpt_oracle as O
from tests.golden.make_cfg_golden import BEAM_WEIGHT_SEED
from tests.golden.make_golden import CASES
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "contrastive_kats.npz")
TOL = {torch.float16: 3e-3, torch.bfloat16: 2e-2}  # score margins below these may flip between the 16-bit step and HF's fp32 model


def _elem(dtype):
    from spatialrgpt_b200 import ops
    return ops.elem_dtype(dtype)


# ---- the kernels --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,k,lens,H", [(1, 2, [1], 512), (1, 4, [259], 256), (5, 8, [1, 259, 100, 4096, 33], 128), (5, 50, [70, 1, 259, 4096, 2000], 64),
                                        (1, 50, [4096], 4096), (2, 64, [31, 97], 128)])
def test_penalty_and_select_match_float64(dtype, B, k, lens, H):
    from spatialrgpt_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + k + H)
    L_cap, V = 4160 if max(lens) > 2000 else 300, 1003
    ctx = (torch.randn(B, L_cap, H, generator=g)).to(dtype)
    cand = (torch.randn(B * k, H, generator=g)).to(dtype)
    for gi in range(B):  # candidates near a context row, so the penalty is not the same everywhere
        for i in range(0, k, 3):
            cand[gi * k + i] = (ctx[gi, (7 * i) % lens[gi]].float() + 0.3 * torch.randn(H, generator=g)).to(dtype)
    logp = torch.log_softmax(torch.randn(B, k, generator=g) * 2, -1)
    toks = torch.randint(0, V, (B, k), generator=g, dtype=torch.int32)
    tie_g = B - 1  # a constructed tie: candidates 1 and 2 of the last prompt have the same row and the same probability
    if k > 2:
        cand[tie_g * k + 2] = cand[tie_g * k + 1]
        logp[tie_g, 2] = logp[tie_g, 1]
        logp[tie_g, 1:3] = logp[tie_g].max() + 1.0
    logits = torch.randn(B * k, V, generator=g).to(dtype)
    alpha = 0.6
    with _elem(dtype):
        d_ctx, d_cand = ctx.to(DEV), cand.to(DEV)
        d_lg = torch.zeros(B * k, 1008, dtype=dtype, device=DEV)[:, :V]
        d_lg.copy_(logits)
        nxt = torch.zeros(B, 1008, dtype=dtype, device=DEV)[:, :V]
        pos = torch.tensor([n for n in lens for _ in range(k)], dtype=torch.int32, device=DEV)
        partial = ops.contrastive_partial(B, k, L_cap, DEV)
        ops.contrastive_penalty(d_cand, d_ctx, pos, k, partial)
        a = torch.tensor([1.0 - alpha, alpha], dtype=torch.float64).float().to(DEV)
        step, ticket = torch.tensor([3], dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
        out = torch.full((8 * B,), -7, dtype=torch.int64, device=DEV)
        sel = torch.empty(B, dtype=torch.int32, device=DEV)
        pen, score = (torch.empty(B, k, dtype=torch.float32, device=DEV) for _ in range(2))
        ops.contrastive_select(logp.to(DEV), toks.to(DEV), partial, a, d_cand, d_lg, d_ctx, nxt, pos, out, step, ticket, sel, pen, score)
        torch.cuda.synchronize()
    c64, x64 = ctx.double(), cand.double()
    for gi, L in enumerate(lens):
        cn = c64[gi, :L] / c64[gi, :L].norm(dim=-1, keepdim=True)
        xn = x64[gi * k:(gi + 1) * k] / x64[gi * k:(gi + 1) * k].norm(dim=-1, keepdim=True)
        ref_pen = (xn @ cn.T).max(-1).values
        assert (pen[gi].double().cpu() - ref_pen).abs().max() <= 1e-5, (gi, (pen[gi].double().cpu() - ref_pen).abs().max())
        ref_score = (1 - alpha) * logp[gi].double().exp() - alpha * ref_pen
        top2 = ref_score.topk(2).values
        s = int(sel[gi])
        if gi == tie_g and k > 2:
            assert s == 1  # the lowest index of the tie
        elif float(top2[0] - top2[1]) > 1e-5:
            assert s == int(ref_score.argmax()), (gi, s, ref_score)
        assert int(out[3 * B + gi]) == int(toks[gi, s])
        r = gi * k + s
        assert torch.equal(d_ctx[gi, L].cpu().view(torch.int16), cand[r].view(torch.int16))  # the chosen row joins the context
        assert torch.equal(nxt[gi].cpu().view(torch.int16), logits[r].view(torch.int16))
    assert pos.cpu().tolist() == [n + 1 for n in lens for _ in range(k)] and int(step) == 4 and int(ticket) == 0
    assert int((out == -7).sum()) == 7 * B  # only row step 3 written


@pytest.mark.parametrize("dtype", DTYPES)
def test_kv_broadcast_matches_torch_indexing(dtype):
    from spatialrgpt_b200 import ops
    Lyr, n_pages, nkv, hd, k, G, cap = 3, 96, 2, 64, 4, 3, 6
    g = torch.Generator().manual_seed(5)
    pages = torch.randn(Lyr, n_pages, 2, 16, nkv, hd, generator=g).to(dtype).to(DEV)
    perm = torch.randperm(n_pages, generator=g)[: G * k * cap].view(G * k, cap).to(torch.int32)
    tables = torch.zeros(G * k + 2, cap + 1, dtype=torch.int32)
    tables[: G * k, :cap] = perm
    positions = [17, 40, 3]  # the position just written, per prompt
    pos = torch.tensor([p + 1 for p in positions for _ in range(k)], dtype=torch.int32)
    sel = torch.tensor([2, 0, 3], dtype=torch.int32)
    ref = pages.clone()
    for gi in range(G):
        p, s = positions[gi], int(sel[gi])
        src = ref[:, int(perm[gi * k + s, p // 16]), :, p % 16].clone()
        for i in range(k):
            ref[:, int(perm[gi * k + i, p // 16]), :, p % 16] = src
    with _elem(dtype):
        ops.kv_broadcast_rows(pages, tables.to(DEV), pos.to(DEV), -1, sel.to(DEV), k)
    torch.cuda.synchronize()
    assert torch.equal(pages.view(torch.int16), ref.view(torch.int16))  # the siblings' position, and nothing else, changed


# ---- the decoder against HF ---------------------------------------------------------------------------------------------------------
def _model(dtype, max_seq_len=512):
    from tests.test_gpu_fp16 import build_model
    return build_model(CASES["tiny_masks_gqa"][0], BEAM_WEIGHT_SEED, dtype=dtype, max_seq_len=max_seq_len)


def _agrees(ids, ref, margins, tol):
    """ids equal HF's up to the first step whose score margin is below tol (that step and the later ones may differ)."""
    m = next((t for t, x in enumerate(margins) if x < tol), None)
    return ids == ref if m is None else ids[:m] == ref[:m]


@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_hf_contrastive_search(dtype):
    """Every fixture prompt, batched as in the fixture (one prompt, two equal-length prompts); graph and eager steps give equal ids."""
    k = np.load(GOLDEN)
    oc, sd, model = _model(dtype)
    names = sorted({n.split("__")[0] for n in k.files if "__" in n})
    ok, full = [], []
    for name in names:
        ids = torch.from_numpy(k[f"{name}__input_ids"]).to(DEV)
        eos = int(k[f"{name}__eos"])
        packed = model.llm.embed_tokens(ids)
        lens = [ids.shape[1]] * ids.shape[0]
        kw = dict(eos_token_ids=None if eos < 0 else eos)
        out = model.llm.generate_contrastive(packed, lens, int(k[f"{name}__k"]), float(k[f"{name}__alpha"]), int(k["max_new"]), **kw)
        eager = model.llm.generate_contrastive(packed, lens, int(k[f"{name}__k"]), float(k[f"{name}__alpha"]), int(k["max_new"]),
                                               use_graph=False, **kw)
        assert [t.tolist() for t in out] == [t.tolist() for t in eager], name
        for b in range(ids.shape[0]):
            ref = k[f"{name}__ids{b}"].tolist()
            ok.append(_agrees(out[b].tolist(), ref, k[f"{name}__margin{b}"].tolist(), TOL[dtype]))
            full.append(out[b].tolist() == ref)
    print(f"contrastive {dtype}: prompts agreeing with HF up to the first near-tie: {sum(ok)} of {len(ok)}; equal throughout: {sum(full)}")
    assert all(ok), ok


@pytest.mark.parametrize("dtype", DTYPES)
def test_tiny_alpha_is_greedy(dtype):
    """penalty_alpha = 1e-6 ranks by probability alone wherever greedy's top-2 probability margin exceeds 1e-5."""
    oc, sd, model = _model(dtype)
    ids = torch.randint(3, 1000, (1, 30), generator=torch.Generator().manual_seed(8)).to(DEV)
    g = model.generate(ids, max_new_tokens=16, return_dict_in_generate=True, output_scores=True)
    c = model.generate(ids, max_new_tokens=16, penalty_alpha=1e-6, top_k=4)
    probs = torch.stack(g.scores)[:, 0].softmax(-1).topk(2).values
    margins = (probs[:, 0] - probs[:, 1]).tolist()
    m = next((t for t, x in enumerate(margins) if x <= 1e-5), len(margins))
    assert c[0, :m + 1].tolist() == g.sequences[0, :m + 1].tolist(), (m, c.tolist(), g.sequences.tolist())


def _long_prompts(H, dtype, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, H, generator=g) * 0.3).to(dtype).to(DEV) for n in lens]


def _composition_check(dec, prompts, k, n_new, alpha=0.6, eos=None):
    """Each prompt's ids do not depend on the other prompts of its batch (batches of 2 or more: batch 1 runs batch 1's prefill): every
    batch packs more than 128 prompt rows and has at most 128 rows per step, so each GEMM keeps one configuration."""
    def run(idx, **kw):
        return dec.generate_contrastive(torch.cat([prompts[i] for i in idx]), [prompts[i].shape[0] for i in idx], k, alpha, n_new,
                                        eos_token_ids=eos, **kw)
    n = len(prompts)
    base = run(list(range(n)))
    assert [t.tolist() for t in base] == [t.tolist() for t in run(list(range(n)), use_graph=False)]
    for idx in ([n - 1, 0], list(reversed(range(n))), [2, 0, 3] if n > 3 else [2, 0]):
        for i, t in zip(idx, run(idx)):
            assert t.tolist() == base[i].tolist(), (idx, i)
    one = dec.generate_contrastive(prompts[1], [prompts[1].shape[0]], k, alpha, n_new, eos_token_ids=eos)
    assert [t.tolist() for t in one] == [t.tolist() for t in dec.generate_contrastive(prompts[1], [prompts[1].shape[0]], k, alpha, n_new,
                                                                                       eos_token_ids=eos, use_graph=False)]
    return base


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_composition_invariance(dtype):
    oc, sd, model = _model(dtype)
    prompts = _long_prompts(oc.hidden, dtype, [131, 150, 129, 170, 140], 11)
    _composition_check(model.llm, prompts, 4, 12)
    _composition_check(model.llm, prompts[:4], 8, 10, alpha=0.3)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stopping_eos_criteria_and_max_length(dtype):
    oc, sd, model = _model(dtype)
    ids = torch.randint(3, 1000, (2, 20), generator=torch.Generator().manual_seed(3)).to(DEV)
    kw = dict(penalty_alpha=0.6, top_k=4)
    full = model.generate(ids, max_new_tokens=10, **kw)
    assert full.shape == (2, 10)
    eos = int(full[0, 2])
    if eos in full[1].tolist() or eos in full[0, :2].tolist():
        pytest.skip("the chosen EOS id comes earlier or in the other prompt too")
    stopped = model.generate(ids, max_new_tokens=10, eos_token_id=eos, pad_token_id=1, **kw)
    assert stopped[0].tolist() == full[0, :3].tolist() + [1] * 7  # padded after its EOS
    assert stopped[1].tolist() == full[1].tolist()

    class AtFive:
        def __call__(self, input_ids, scores):
            return input_ids.shape[-1] >= 5

    crit = model.generate(ids, max_new_tokens=10, stopping_criteria=[AtFive()], **kw)
    assert crit.tolist() == full[:, :5].tolist()
    short = model.generate(ids, max_length=24, **kw)
    assert short.tolist() == full[:, :4].tolist()


@pytest.mark.parametrize("dtype", DTYPES)
def test_output_scores(dtype):
    oc, sd, model = _model(dtype)
    ids = torch.randint(3, 1000, (2, 25), generator=torch.Generator().manual_seed(4)).to(DEV)
    greedy = model.generate(ids[:1], max_new_tokens=6, return_dict_in_generate=True, output_scores=True)
    r = model.generate(ids[:1], max_new_tokens=6, penalty_alpha=0.6, top_k=5, return_dict_in_generate=True, output_scores=True)
    assert torch.equal(r.scores[0], greedy.scores[0])  # both the prefill's last row through batch 1's lm_head
    plain = model.generate(ids[:1], max_new_tokens=6, penalty_alpha=0.6, top_k=5)
    assert torch.equal(r.sequences, plain)
    rb = model.generate(ids, max_new_tokens=6, penalty_alpha=0.6, top_k=5, return_dict_in_generate=True, output_scores=True)
    for res in (r, rb):
        assert len(res.scores) == res.sequences.shape[1]
        for t, row in enumerate(res.scores):
            top = row.topk(5, -1).indices
            for b in range(row.shape[0]):
                assert int(res.sequences[b, t]) in top[b].tolist(), (t, b)


def test_multimodal_generate_equals_the_oracle(golden_dir):
    from tests.contrastive_oracle import contrastive_generate
    from tests.test_gpu_fp16 import build_model
    name = "tiny_masks_gqa"
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    gd = load_npz(os.path.join(golden_dir, name + ".npz"))
    oc, sd, model = build_model(kw, int(gd["weight_seed"]), dtype=torch.float16)
    ok = 0
    for seed in (1234, 77):
        input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=seed, kind=kind)
        enc = O.encode_multimodal(oc, sd, images, depths, masks)
        embeds = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), input_ids, enc["image_features"], enc["mask_embeds"],
                                     enc["depth_embeds"])[0]
        ref, rec = contrastive_generate(oc, sd["llm"], embeds, 4, 0.6, 8)
        top2 = rec["score"].topk(2, -1).values
        h = lambda t: t.to(DEV, torch.float16)  # noqa: E731
        out = model.generate(input_ids.to(DEV), images=h(images), depths=h(depths), masks=[h(m) for m in masks], penalty_alpha=0.6, top_k=4,
                             max_new_tokens=8)
        ok += _agrees(out[0].tolist(), ref.tolist(), (top2[:, 0] - top2[:, 1]).tolist(), TOL[torch.float16])
        print("multimodal", seed, out[0].tolist(), ref.tolist())
    assert ok == 2


def _dims():
    from spatialrgpt_b200.config import LlamaDims
    return dataclasses.replace(LlamaDims(), hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16,
                               num_key_value_heads=4, head_dim=128, vocab_size=32003)


@pytest.mark.parametrize("dtype", DTYPES)
def test_fp8_and_nf4_decoders(dtype):
    """The FP8 and NF4 planes-only 4-layer decoders run contrastive search through the same step: graph equals eager and a prompt's ids
    do not depend on its batch, and NF4 planes-only equals NF4 copy mode bit for bit."""
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    prompts = _long_prompts(d.hidden_size, dtype, [131, 150, 129, 170], 5)
    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512, max_seqs=2)
    assert dec.fp8
    out = _composition_check(dec, prompts, 4, 10)
    assert all(t.numel() == 10 for t in out)
    del dec
    sd = _llm_state_dict(d, 21)
    res = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512, max_seqs=2)
        assert dec.nf4_planes_only == (not copy)
        res[copy] = [t.tolist() for t in _composition_check(dec, prompts, 4, 10)]
        del dec
    assert res[True] == res[False]
