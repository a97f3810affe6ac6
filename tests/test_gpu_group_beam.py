"""Diverse beam search on the H100 (generate(num_beams=k, num_beam_groups=G, diversity_penalty=lambda); LlamaDecoder.generate_beam_batch
with num_beam_groups, csrc/beam.cu group_select_kernel): the kernel against a torch restatement bit for bit, every prompt against the
restatement of transformers 4.37.2's group_beam_search over the fp32 oracle (tests/group_beam_oracle.py), graph against eager, the
multimodal and padded text API, and the packed, NF4 and FP8 weight formats."""
import dataclasses
import os

import pytest
import torch

from oracle import srgpt_oracle as O
from tests.golden.make_golden import CASES
from tests.group_beam_oracle import group_beam_generate
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


# ---- the kernel ---------------------------------------------------------------------------------------------------------------------
def _restated(logits, stats, scores, k, G, lam, eos, pad, done):
    """group_select_kernel in torch: each group's rows of logp = (v - m) - lse (the candidates kernel's m, lse) minus fl(lambda * c) for
    the earlier groups' choices of this step, plus the beam score, all in fp32; ranked by a stable float64 sort of the flattened group
    table; HF's process rule.  Returns (scores, beams, tokens) [P, G, n_cand] and (next beams, next tokens) [P * k]."""
    R, V = logits.shape
    P, gs = R // k, k // G
    n_cand = max(2, 1 + len(eos)) * gs
    logp = (logits.float() - stats[:, :1]) - stats[:, 1:]
    lam32 = torch.tensor(lam, dtype=torch.float32)
    out_s = torch.full((P, G, n_cand), float("-inf"))
    out_b = torch.full((P, G, n_cand), -1, dtype=torch.int32)
    out_t = torch.full((P, G, n_cand), -1, dtype=torch.int32)
    nb, nt = torch.full((R,), -1, dtype=torch.int32), torch.full((R,), -1, dtype=torch.int32)
    for p in range(P):
        chosen = []
        for g in range(G):
            r0 = p * k + g * gs
            if done[p, g]:
                nb[r0:r0 + gs], nt[r0:r0 + gs] = g * gs, pad
                chosen += [pad] * gs
                continue
            c = torch.bincount(torch.tensor(chosen, dtype=torch.long), minlength=V)[:V].float() if chosen else torch.zeros(V)
            pen = torch.where(c > 0, lam32 * c, torch.zeros(V))
            tab = torch.where(c > 0, logp[r0:r0 + gs] - pen, logp[r0:r0 + gs]) + scores[r0:r0 + gs, None]
            flat = tab.reshape(-1)
            order = torch.sort(-flat.double(), stable=True).indices[:n_cand]
            out_s[p, g], out_b[p, g], out_t[p, g] = flat[order], (order // V).int(), (order % V).int()
            n = 0
            for t, b in zip(out_t[p, g].tolist(), out_b[p, g].tolist()):
                if t in eos:
                    continue
                nb[r0 + n], nt[r0 + n] = g * gs + b, t
                chosen.append(t)
                n += 1
                if n == gs:
                    break
    return (out_s, out_b, out_t), (nb, nt)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k,G,V", [(2, 2, 1000), (4, 2, 1000), (4, 4, 32003), (6, 2, 1000), (6, 6, 1000), (8, 2, 128256), (8, 8, 1000)])
def test_group_select_matches_a_torch_restatement(dtype, k, G, V):
    from spatialrgpt_b200 import ops
    P = 5
    gs = k // G
    R = P * k
    gen = torch.Generator().manual_seed(k * 100 + G * 10 + V)
    eos, pad, lam = [3, 7], 3, 0.75
    with ops.elem_dtype(dtype):
        for trial in range(3):
            # small integer logits tie often (the rows' top tokens collide across groups); some rows are mostly -inf; beam scores mix 0,
            # exact halves, a value whose addition rounds, and -1e9 (the starting scores of a group's other beams)
            lg = torch.randint(-4, 4, (R, V), generator=gen).float() * (0.5 if trial else 1.0)
            lg[:, :8] += 3.0  # the EOS ids and their neighbours lead
            lg[1, 12:] = float("-inf")
            lg[R - 1, torch.randperm(V, generator=gen)[:V // 2]] = float("-inf")
            logits = lg.to(dtype)
            ld = (V + 7) // 8 * 8
            d_logits = torch.zeros(R, ld, dtype=dtype, device=DEV)[:, :V]
            d_logits.copy_(logits)
            choice = torch.tensor([0.0, -0.5, -1e9, -37.123457])
            scores = choice[torch.randint(0, 4, (R,), generator=gen)]
            scores[::gs] = torch.where(torch.rand(P * G, generator=gen) < 0.5, 0.0, -2.25)
            done = (torch.rand(P, G, generator=gen) < 0.25).int()
            done[0] = 0
            n_cand = max(2, 1 + len(eos)) * gs
            L = min(n_cand + k - gs, V)
            cs = torch.empty(R, L, dtype=torch.float32, device=DEV)
            ct = torch.empty(R, L, dtype=torch.int32, device=DEV)
            stats = torch.empty(R, 2, dtype=torch.float32, device=DEV)
            d_scores = scores.to(DEV)
            ops.beam_candidates_scored(d_logits, d_scores, cs, ct, stats)
            outs = [torch.empty(P, G, n_cand, dtype=t, device=DEV) for t in (torch.float32, torch.int32, torch.int32)]
            nxt = [torch.empty(R, dtype=torch.int32, device=DEV) for _ in range(2)]
            ops.beam_group_select(d_logits, stats, d_scores, ct, k, G, torch.tensor(eos, dtype=torch.int32, device=DEV), pad, lam,
                                  done.to(DEV), *outs, *nxt)
            st = stats.cpu()
            lf = logits.float().double()
            assert torch.equal(st[:, 0], logits.float().max(-1).values)  # the max is exact
            assert torch.allclose(st[:, 1].double(), torch.logsumexp(lf - lf.max(-1, keepdim=True).values, -1), atol=1e-5)
            (rs, rb, rt), (nb, nt) = _restated(logits, st, scores, k, G, lam, eos, pad, done)
            ds = done.bool()[:, :, None].expand_as(rs)
            assert torch.equal(outs[1].cpu()[~ds], rb[~ds]) and torch.equal(outs[2].cpu()[~ds], rt[~ds]), (trial,)
            assert torch.equal(outs[0].cpu()[~ds].view(torch.int32), rs[~ds].view(torch.int32)), (trial,)
            assert (outs[1].cpu()[ds] == -1).all() and (outs[2].cpu()[ds] == -1).all()
            assert torch.equal(nxt[0].cpu(), nb) and torch.equal(nxt[1].cpu(), nt), (trial,)
            # the candidate lists are each row's top L in (score desc, token asc) order of the fp32 score
            row_s = ((logits.float() - st[:, :1]) - st[:, 1:]) + scores[:, None]
            for r in (0, 1, R - 1):
                order = torch.sort(-row_s[r].double(), stable=True).indices[:L]
                assert ct[r].cpu().tolist() == order.tolist(), r


# ---- end to end ---------------------------------------------------------------------------------------------------------------------
# (num_beams, num_beam_groups, diversity_penalty, eos, max_new_tokens, length_penalty, early_stopping)
GROUP_CASES = [
    (4, 2, 0.5, None, 10, 1.0, False),
    (4, 4, 1.0, [460], 10, 1.0, False),
    (6, 3, 0.3, [38, 97], 12, 1.0, False),
    (4, 2, 0.7, [764], 16, 2.0, False),
    (4, 2, 0.7, [764], 16, 0.5, True),
    (2, 2, 5.0, [886], 10, 1.0, False),
]


def _model(dtype):
    from tests.test_gpu_fp16 import build_model
    g = load_npz(os.path.join(os.path.dirname(__file__), "golden", "beam_batch_kats.npz"))
    oc, sd, model = build_model(CASES["tiny_masks_gqa"][0], int(g["weight_seed"]), dtype=dtype)
    return g, oc, sd, model


@pytest.mark.parametrize("dtype,need", [(torch.float16, 18), (torch.bfloat16, 12)])
def test_group_beams_match_the_restatement(dtype, need):
    """B = 3 prompts of 20, 9 and 14 rows, and B = 1, against the restatement over the fp32 oracle: fp16 on every prompt of every case;
    bf16 rounds the logits to 8 bits of mantissa, which flips near-ties that the penalty then carries into later groups, so it matches
    12 of the 18 prompts (as measured on an H100).  Graph and eager steps give equal ids, and a prompt's ids do not depend on its batch."""
    g, oc, sd, model = _model(dtype)
    lens = [int(n) for n in g["seq_lens"]][:3]
    packed = g["packed_embeds"][:sum(lens)].to(DEV)
    offs = [0, lens[0], lens[0] + lens[1], sum(lens)]
    ok = []
    for i, (k, G, lam, eos, n_new, lp, es) in enumerate(GROUP_CASES):
        kw = dict(eos_token_ids=eos, length_penalty=lp, early_stopping=es, num_beam_groups=G, diversity_penalty=lam)
        out = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, k, n_new, **kw)]
        eager = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, k, n_new, use_graph=False, **kw)]
        assert out == eager, i
        one = model.llm.generate_beam_batch(packed[:lens[0]], lens[:1], k, n_new, **kw)[0].tolist()
        assert one == out[0], i
        for b in range(3):
            ref = group_beam_generate(oc, sd["llm"], g["packed_embeds"][offs[b]:offs[b + 1]], k, G, lam, n_new, eos, lp, es)["ids"]
            ok.append(out[b] == ref)
            if dtype == torch.float16:
                assert out[b] == ref, (i, b, out[b], ref)
    print(f"group beams {dtype}: prompts equal to the restatement: {sum(ok)} of {len(ok)} {ok}")
    assert sum(ok) >= need, ok


def test_stopping_criterion_and_plain_beams_are_unchanged():
    g, oc, sd, model = _model(torch.float16)
    lens = [int(n) for n in g["seq_lens"]][:3]
    packed = g["packed_embeds"][:sum(lens)].to(DEV)
    offs = [0, lens[0], lens[0] + lens[1], sum(lens)]
    stop = lambda ids: ids.numel() >= 5  # noqa: E731
    out = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, 4, 12, eos_token_ids=[460], stopping_fn=stop, num_beam_groups=2,
                                                              diversity_penalty=0.5)]
    for b in range(3):
        ref = group_beam_generate(oc, sd["llm"], g["packed_embeds"][offs[b]:offs[b + 1]], 4, 2, 0.5, 12, [460], stopping_fn=stop)["ids"]
        assert out[b] == ref, (b, out[b], ref)
    # one group is plain beam search on the plain path
    plain = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, 4, 10, eos_token_ids=[460])]
    assert plain == [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, 4, 10, eos_token_ids=[460], num_beam_groups=1)]


def test_generate_api_multimodal_and_padded_text_prompts():
    from tests.test_gpu_fp16 import build_model
    name = "tiny_masks_gqa"
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    gd = load_npz(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    oc, sd, model = build_model(kw, int(gd["weight_seed"]), dtype=torch.float16)
    reqs = [O.synth_request(oc, n_regions, t_text, seed=s, kind=kind) for s in (1234, 1234)]
    reqs[1] = (reqs[1][0],) + tuple(O.synth_request(oc, n_regions, t_text, seed=77, kind=kind)[1:])
    refs = []
    for input_ids, images, depths, masks in reqs:
        enc = O.encode_multimodal(oc, sd, images, depths, masks)
        embeds = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), input_ids, enc["image_features"], enc["mask_embeds"],
                                     enc["depth_embeds"])[0]
        refs.append(group_beam_generate(oc, sd["llm"], embeds, 4, 2, 0.8, 8)["ids"])
    h = lambda t: t.to(DEV, torch.float16)  # noqa: E731
    args = dict(images=h(torch.cat([r[1] for r in reqs])), depths=h(torch.cat([r[2] for r in reqs])),
                masks=[h(m) for r in reqs for m in r[3]])
    out = model.generate(torch.cat([r[0] for r in reqs]).to(DEV), num_beams=4, num_beam_groups=2, diversity_penalty=0.8, max_new_tokens=8,
                         **args)
    assert out.shape[0] == 2
    for b in range(2):
        assert out[b].tolist()[:len(refs[b])] == refs[b], (b, out[b].tolist(), refs[b])
    one = model.generate(reqs[0][0].to(DEV), num_beams=4, num_beam_groups=2, diversity_penalty=0.8, max_new_tokens=8,
                         images=h(reqs[0][1]), depths=h(reqs[0][2]), masks=[h(m) for m in reqs[0][3]])
    assert one[0].tolist()[:len(refs[0])] == refs[0]
    # text only, a left-padded batch: each row equals the batch-1 call of its unpadded prompt
    ids = torch.randint(3, 900, (2, 20), generator=torch.Generator().manual_seed(1)).to(DEV)
    mask = torch.ones_like(ids)
    mask[1, :6] = 0
    gk = dict(num_beams=4, num_beam_groups=4, diversity_penalty=2.0, max_new_tokens=6)
    model.config.llama.tokenizer_padding_side = "left"
    try:
        both = model.generate(ids, attention_mask=mask, pad_token_id=0, **gk)
        single = [model.generate(ids[0:1], **gk), model.generate(ids[1:2, 6:], **gk)]
    finally:
        model.config.llama.tokenizer_padding_side = "right"
    assert [both[b].tolist() for b in range(2)] == [single[b][0].tolist() for b in range(2)]


# ---- weight formats -------------------------------------------------------------------------------------------------------------------
def _dims():
    from spatialrgpt_b200.config import LlamaDims
    return dataclasses.replace(LlamaDims(), hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16,
                               num_key_value_heads=4, head_dim=128, vocab_size=32003)


def _prompts(H, dtype, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, H, generator=g) * 0.3).to(dtype).to(DEV) for n in lens]


def _run(dec, prompts, **kw):
    x = torch.cat(prompts)
    lens = [p.shape[0] for p in prompts]
    out = [t.tolist() for t in dec.generate_beam_batch(x, lens, 4, 10, num_beam_groups=2, diversity_penalty=0.6, **kw)]
    assert out == [t.tolist() for t in dec.generate_beam_batch(x, lens, 4, 10, num_beam_groups=2, diversity_penalty=0.6, use_graph=False, **kw)]
    assert all(1 <= len(t) <= 10 and all(0 <= v < dec.dims.vocab_size for v in t) for t in out)
    return out


def test_packed_weights_give_the_bf16_ids(monkeypatch):
    """The lossless 12-bit packing changes no logit, so the ids are the bf16 decoder's."""
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_packed_decode import _decoder
    dec1 = _decoder(monkeypatch, True)
    prompts = _prompts(dec1.dims.hidden_size, torch.bfloat16, [20, 33], 3)
    ids1 = _run(dec1, prompts)
    monkeypatch.setenv("SRGPT_DECODE_PACK", "0")
    dec0 = LlamaDecoder(dec1.dims, dec1.w, max_seq_len=256)
    del dec1
    torch.cuda.empty_cache()
    assert _run(dec0, prompts) == ids1


@pytest.mark.parametrize("dtype", DTYPES)
def test_nf4_and_fp8_decoders_run_group_beams(dtype):
    """The FP8 and NF4 decoders' logits differ from the 16-bit model's, so the case shows the call runs: graph equals eager and every
    id is valid; NF4 planes-only equals NF4 copy mode."""
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    prompts = _prompts(d.hidden_size, dtype, [131, 150, 129], 5)
    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512, max_seqs=2)
    assert dec.fp8
    _run(dec, prompts, eos_token_ids=[460])
    del dec
    sd = _llm_state_dict(d, 21)
    res = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512, max_seqs=2)
        res[copy] = _run(dec, prompts)
        del dec
    assert res[True] == res[False]
