"""generate(output_hidden_states=True, output_attentions=True, return_dict_in_generate=True) on the H100, in both element types: the
decode probability kernel against an fp64 softmax over the paged cache, the flags changing no id / score / logit bit on any weight
format, entry 0 against forward() bit for bit, graph against eager replay, and the outputs against the fp32 oracle
(tests/generate_outputs_oracle.py)."""
import pytest
import torch

from oracle import srgpt_oracle as O
from tests.generate_outputs_oracle import generate_outputs
from tests.golden.make_golden import CASES
from tests.test_gpu_forward_outputs import C2, FORMATS, FACTOR, _model, _text_batch, _ulp

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
FLAGS = dict(return_dict_in_generate=True, output_hidden_states=True, output_attentions=True)


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("R,nh,nkv", [(1, 8, 8), (3, 16, 4), (32, 8, 2)])
def test_decode_probability_kernel(dtype, R, nh, nkv):
    from spatialrgpt_b200 import ops
    hd, ps = 128, 16
    g = torch.Generator().manual_seed(R * 100 + nh)
    n_prompt = torch.randint(1, 400, (R,), generator=g)
    gen = torch.randint(1, 300, (R,), generator=g)  # keys generated so far, the step's own included
    if R == 1:
        n_prompt[0], gen[0] = 3000, 1096  # 4096 keys
    n_prompt[-1] = 17  # a prompt that ends one row past a page boundary
    P = n_prompt + gen
    T = int(n_prompt.max()) + 5
    offs = torch.tensor([(T - int(n)) if r % 2 == 0 else 0 for r, n in enumerate(n_prompt)])  # left and right padding
    n_cols = T + int(gen.max()) + 7
    cap = (int(P.max()) + ps - 1) // ps
    n_pages = R * cap + 3
    perm = torch.randperm(n_pages, generator=g)[:R * cap].view(R, cap).to(torch.int32)
    kv = (torch.randn(n_pages, 2, ps, nkv, hd, generator=g)).to(dtype)
    q = torch.randn(R, nh * hd, generator=g).to(dtype)
    scale = hd ** -0.5
    with ops.elem_dtype(dtype):
        out = torch.full((3, R, nh, n_cols), float("nan"), dtype=dtype, device=DEV)
        ws = ops.attention_probs_decode_ws(R, nh, n_cols, DEV)
        step = torch.tensor([2], dtype=torch.int32, device=DEV)  # writes slot step - 1 = 1
        ops.attention_probs_decode(q.to(DEV), kv.to(DEV), perm.to(DEV), ps, (P - 1).to(torch.int32).to(DEV), nh, nkv, hd, scale,
                                   offs.to(torch.int32).to(DEV), n_prompt.to(torch.int32).to(DEV), T, step, -1, out, ws)
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.isnan(out[0]).all() and torch.isnan(out[2]).all(), "only the device step's slot is written"
    for r in range(R):
        p, n, off = int(P[r]), int(n_prompt[r]), int(offs[r])
        keys = torch.cat([kv[int(perm[r, j // ps]), 0, j % ps] for j in range(p)]).view(p, nkv, hd).double()
        qr = q[r].double().view(nh, hd)
        s = torch.einsum("hd,khd->hk", qr, keys.repeat_interleave(nh // nkv, 1)) * scale
        ref = torch.softmax(s, -1)
        width = T + p - n
        row = out[1, r]
        assert not torch.isnan(row[:, :width]).any(), "every column of the row's view is written"
        assert torch.isnan(row[:, width:]).all(), "nothing past the row's view"
        cols = torch.cat([off + torch.arange(n), T + torch.arange(p - n)])
        got = row[:, cols].double()
        assert bool(((got - ref).abs() <= _ulp(ref, dtype)).all()), (r, float((got - ref).abs().max()))
        pad = torch.ones(width, dtype=torch.bool)
        pad[cols] = False
        assert bool((row[:, :width][:, pad] == 0).all()), "pad columns are 0"
        assert float((row[:, :width].double().sum(-1) - 1).abs().max()) <= 2 ** -6


# ---- the flags change nothing ------------------------------------------------------------------------------------------------------
def _ids_scores(out):
    return out.sequences, torch.stack(out.scores)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_flags_change_no_id_score_or_logit(dtype, fmt):
    from spatialrgpt_b200 import ops
    quant, copy = FORMATS[fmt]
    oc, _, model = _model(C2, dtype, quant, copy)
    modes = [dict(), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=7), dict(repetition_penalty=1.3, no_repeat_ngram_size=2)]
    for lens in ([37], [37, 12, 50, 25]):
        ids, am = _text_batch(oc.vocab, lens, True, seed=3)
        ids, am = ids.to(DEV), am.to(DEV)
        for mode in modes:
            kw = dict(max_new_tokens=9, return_dict_in_generate=True, output_scores=True, **mode)
            if len(lens) == 1:
                kw["output_logits"] = True
            model.generate(ids, attention_mask=am, **kw)  # captures this mode's graph: the counts below are replays
            n0 = ops.LAUNCHES
            ref = model.generate(ids, attention_mask=am, **kw)
            n1 = ops.LAUNCHES
            off = model.generate(ids, attention_mask=am, output_hidden_states=False, output_attentions=False, **kw)
            n2 = ops.LAUNCHES
            on = model.generate(ids, attention_mask=am, output_hidden_states=True, output_attentions=True, **kw)
            assert n2 - n1 == n1 - n0, "flags off launch exactly what no flags launch"
            assert off.hidden_states is None and off.attentions is None
            for r in (off, on):
                assert torch.equal(r.sequences, ref.sequences), (fmt, lens, mode)
                assert torch.equal(torch.stack(r.scores), torch.stack(ref.scores))
                if len(lens) == 1:
                    assert all(torch.equal(a, b) for a, b in zip(r.logits, ref.logits))
            n_max = ref.sequences.shape[1]
            assert len(on.hidden_states) == len(on.attentions) == n_max
            T = max(lens)
            for t in range(1, n_max):
                assert on.attentions[t][0].shape == (len(lens), oc.heads, 1, T + t)
                assert on.hidden_states[t][0].shape == (len(lens), 1, oc.hidden)
                for a in on.attentions[t]:  # decode rows sum to 1
                    assert float((a.float().sum(-1) - 1).abs().max()) <= 2 ** -5
            if not mode:  # greedy: hidden_states[L] through lm_head is the raw score row
                for t in range(1, n_max):
                    with ops.elem_dtype(dtype):
                        hn = on.hidden_states[t][-1][:, 0].contiguous()
                        lg = ops.gemm(hn, model.weights.llama.lm_head, out=model.llm._logits_buffer(hn.shape[0])).float()
                    sc = ref.scores[t]
                    tol = 4 * float(_ulp(sc.abs().max(), dtype))
                    assert float((lg - sc).abs().max()) <= tol, (t, float((lg - sc).abs().max()))
            del on


# ---- entry 0 is forward()'s; graphs equal eager steps ------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_prompt_entry_is_forward_bit_for_bit(dtype):
    oc, _, model = _model(CASES["tiny_masks_gqa"][0], dtype)
    for lens, left in (([23], True), ([23, 9, 31], True), ([23, 9, 31], False)):
        model.config.llama.tokenizer_padding_side = "left" if left else "right"
        ids, am = _text_batch(oc.vocab, lens, left, seed=4)
        ids, am = ids.to(DEV), am.to(DEV)
        fw = model.forward(input_ids=ids, attention_mask=am, output_hidden_states=True, output_attentions=True)
        gen = model.generate(ids, attention_mask=am, max_new_tokens=4, **FLAGS)
        assert all(torch.equal(a, b) for a, b in zip(gen.hidden_states[0], fw.hidden_states))
        assert all(torch.equal(a, b) for a, b in zip(gen.attentions[0], fw.attentions))
    model.config.llama.tokenizer_padding_side = "right"
    kw, n_regions, t_text, kind, _, _ = CASES["tiny_masks_gqa"]
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    mm = dict(images=images.to(DEV), depths=depths.to(DEV), masks=[m.to(DEV) for m in masks])
    fw = model.forward(input_ids=input_ids.to(DEV), output_hidden_states=True, output_attentions=True, **mm)
    gen = model.generate(input_ids.to(DEV), max_new_tokens=4, **FLAGS, **mm)
    assert all(torch.equal(a, b) for a, b in zip(gen.hidden_states[0], fw.hidden_states))
    assert all(torch.equal(a, b) for a, b in zip(gen.attentions[0], fw.attentions))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lens", [[30], [30, 11, 44]])
def test_graph_and_eager_steps_bit_identical(dtype, lens):
    oc, _, model = _model(CASES["tiny_masks_gqa"][0], dtype)
    ids, am = _text_batch(oc.vocab, lens, True, seed=6)
    g = model.generate(ids.to(DEV), attention_mask=am.to(DEV), max_new_tokens=7, **FLAGS)
    e = model.generate(ids.to(DEV), attention_mask=am.to(DEV), max_new_tokens=7, use_cuda_graph=False, **FLAGS)
    assert torch.equal(g.sequences, e.sequences)
    for a, b in zip(g.hidden_states + g.attentions, e.hidden_states + e.attentions):
        assert all(torch.equal(x, y) for x, y in zip(a, b))


# ---- against the fp32 oracle -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("lens", [[41], [41, 17, 29]])
def test_against_the_fp32_oracle(dtype, lens):
    """Margin-safe greedy cases (the oracle's ids are ours): every decode entry's hidden rows and attention rows within FACTOR times the
    oracle-in-dtype error."""
    oc, sd, model = _model(CASES["tiny_masks_gqa"][0], dtype)
    model.config.llama.tokenizer_padding_side = "left"
    g = torch.Generator().manual_seed(11)
    T, N = max(lens), 6
    emb = [(torch.randn(n, oc.hidden, generator=g) * 0.3).to(dtype).float() for n in lens]
    ref = [generate_outputs(oc, sd["llm"], e, N, off=T - e.shape[0], T=T) for e in emb]
    rdt = [generate_outputs(oc, sd["llm"], e, N, off=T - e.shape[0], T=T, dtype=dtype) for e in emb]
    packed = torch.cat(emb).to(DEV, dtype)
    with torch.no_grad():
        from spatialrgpt_b200 import ops
        with ops.elem_dtype(dtype):
            gen_out, gp = model._generate_probe(lens, T, N, True, True, True)
            r = (model.llm.generate_from_embeds(packed, N, outputs=gp) if len(lens) == 1 else
                 model.llm.generate_batch(packed, lens, N, outputs=gp))
    outs = [r] if len(lens) == 1 else r
    hs, att = model._generate_outputs(gen_out, N)
    checked = 0
    for b in range(len(lens)):
        if outs[b].tolist() != ref[b][0].tolist():  # a near-tie changed a greedy choice: the row is not margin-safe
            continue
        checked += 1
        for t in range(1, N):
            for l in range(oc.layers + 1):
                e_ours = float((hs[t][l][b].cpu().float() - ref[b][1][t][l]).abs().max())
                e_ref = float((rdt[b][1][t][l].float() - ref[b][1][t][l]).abs().max())
                assert e_ours <= FACTOR * e_ref + 1e-6, ("hidden", b, t, l, e_ours, e_ref)
            for l in range(oc.layers):
                e_ours = float((att[t][l][b].cpu().float() - ref[b][2][t][l]).abs().max())
                e_ref = float((rdt[b][2][t][l].float() - ref[b][2][t][l]).abs().max())
                assert e_ours <= FACTOR * e_ref + 1e-6, ("attn", b, t, l, e_ours, e_ref)
    if checked == 0:
        pytest.skip("every row met a near-tie; not margin-safe")
