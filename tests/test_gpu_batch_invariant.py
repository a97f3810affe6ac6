"""Batch-invariant decoding on the H100: the rows kernels (QKV GEMV over rows of different sequences, rows attention, pick / advance)
against their one-token kernels byte for byte, LlamaDecoder.generate_rows against batch-1 generate_from_embeds for every weight format
and both element types, and generate(batch_invariant=True) against batch-1 generate() for text and multimodal prompts."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


def _rand(shape, seed, dtype, std=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).to(dtype).to(DEV)


# ---- kernels ---------------------------------------------------------------------------------------------------------------------
NH, NKV, HD, H = 32, 8, 128, 4096
PS, CAP = 16, 40  # page size, pages per sequence


def _rope(dtype):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    return build_rope_tables(LlamaDims(), CAP * PS, DEV, dtype)


def _tables(B, n_pages, seed):
    """B page tables [B, CAP + 1] over disjoint pages of a cache of n_pages, shuffled."""
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed))[:B * CAP].view(B, CAP)
    t = torch.zeros(B, CAP + 1, dtype=torch.int32)
    t[:, :CAP] = perm
    return t.to(DEV)


def _matrices(dtype):
    """The qkv matrix of one layer as the element-type weight, its 12-bit packing (bf16) and its NF4 planes (with their dequantized copy)."""
    from spatialrgpt_b200 import ops
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    from spatialrgpt_b200.config import LlamaDims
    d = dataclasses.replace(LlamaDims(), num_hidden_layers=1, vocab_size=1024)
    lw = _llama(d, _llm_state_dict(d, 3), dtype, True).layers[0]
    out = {"plain": (lw.qkv_w, {}), "nf4": (lw.nf4["qkv"], {})}
    if dtype == torch.bfloat16:
        pk, why = ops.pack12(lw.qkv_w)
        assert why is None
        out["packed"] = (lw.qkv_w, {"packed": pk})
    return out, lw


@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_qkv_gemv_equals_one_token_calls(dtype):
    """B rows at different positions, each through its own page table: y and the written K/V pages equal B one-token gemv calls."""
    from spatialrgpt_b200 import ops
    cos, sin = _rope(dtype)
    mats, lw = _matrices(dtype)
    qd = NH * HD
    for B in (1, 3, 8):
        pos = torch.tensor([5, 200, 17, 0, 399, 63, 64, 128][:B], dtype=torch.int32, device=DEV)
        tables = _tables(B, B * CAP + 7, B)
        x = _rand((B, H), 40 + B, dtype)
        for name, (w, kw) in mats.items():
            with ops.elem_dtype(dtype):
                pages_r = torch.zeros(B * CAP + 7, 2, PS, NKV, HD, dtype=dtype, device=DEV)
                pages_1 = pages_r.clone()
                y_r = torch.full((B, qd), float("nan"), dtype=dtype, device=DEV)
                ops.gemv_rows(x, w, y_r, lw.in_norm, 1e-5, NH, NKV, HD, cos, sin, pos, pages_r, tables, PS, **kw)
                y_1 = torch.full((B, qd), float("nan"), dtype=dtype, device=DEV)
                for b in range(B):
                    one = {"nf4": ops.gemv_nf4, "packed": ops.gemv_packed, "plain": ops.gemv}[name]
                    wt = kw["packed"] if name == "packed" else w
                    yb = torch.empty(qd + 2 * NKV * HD, dtype=dtype, device=DEV)
                    one(x[b], wt, yb, lw.in_norm, 1e-5, None, ops.GEMV_QKV_ROPE, NH, NKV, HD, cos, sin, pos[b:b + 1], pages_1, tables[b], PS)
                    y_1[b] = yb[:qd]
                torch.cuda.synchronize()
            assert torch.equal(y_r.view(torch.int16), y_1.view(torch.int16)), (name, B)
            assert torch.equal(pages_r.view(torch.int16), pages_1.view(torch.int16)), (name, B)
            assert bool(pages_r.view(torch.int16).ne(0).any())


@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_attention_equals_one_token_attention(dtype):
    from spatialrgpt_b200 import ops
    B = 8
    n_pages = B * CAP + 3
    pages = _rand((n_pages, 2, PS, NKV, HD), 7, dtype)
    tables = _tables(B, n_pages, 11)
    pos = torch.tensor([0, 1, 15, 16, 255, 256, 300, 639], dtype=torch.int32, device=DEV)
    q = _rand((B, NH * HD), 8, dtype)
    scale = HD ** -0.5
    with ops.elem_dtype(dtype):
        out = torch.full((B, NH * HD), float("nan"), dtype=dtype, device=DEV)
        ops.attention_decode_rows(q, out, pages, tables, PS, pos, NH, NKV, HD, scale)
        ref = torch.full((B, NH * HD), float("nan"), dtype=dtype, device=DEV)
        for b in range(B):
            ops.attention_decode(q[b].contiguous(), ref[b], pages, tables[b].contiguous(), PS, pos[b:b + 1], NH, NKV, HD, scale)
        torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("dtype", DTYPES)
def test_pick_and_advance_equals_the_one_token_arg_max(dtype):
    """lm_head over B rows + rows_advance: each row's token (ties at the top included: the lowest index) equals lm_head_argmax of that row,
    and out_ids / the next embedding rows / pos_rows / step advance as documented."""
    from spatialrgpt_b200 import ops
    B, V, K = 5, 32003, 2048
    W = _rand((V, K), 1, dtype, 0.02)
    W[1000:1010] = W[20000]  # ties: rows 1000..1009 and 20000 score the same
    W[30000] = W[20000]
    emb = _rand((V, K), 2, dtype)
    norm = torch.ones(K, dtype=dtype, device=DEV)
    x = _rand((B, K), 4, dtype)
    x[2] = (W[20000].float() * 50).to(dtype)  # row 2's top is the tie
    ws = torch.zeros(B * int(ops.lm_head_workspace(V, DEV).numel()), dtype=torch.uint8, device=DEV)
    with ops.elem_dtype(dtype):
        ops.lm_head_multi(x, W, norm, 1e-5, ws)
        out = torch.full((3 * B,), -1, dtype=torch.int64, device=DEV)
        step = torch.tensor([1], dtype=torch.int32, device=DEV)
        pos = torch.tensor([10, 20, 30, 40, 50], dtype=torch.int32, device=DEV)
        nxt = torch.zeros(B, K, dtype=dtype, device=DEV)
        ops.rows_advance(ws, V, None, B, emb, nxt, out, step, pos)
        want = []
        for b in range(B):
            o = torch.zeros(1, dtype=torch.int64, device=DEV)
            ops.lm_head_argmax(x[b], W, norm, 1e-5, ops.lm_head_workspace(V, DEV), o, torch.zeros(1, dtype=torch.int32, device=DEV),
                               torch.zeros(1, dtype=torch.int32, device=DEV))
            want.append(int(o))
        torch.cuda.synchronize()
    assert out[B:2 * B].tolist() == want and want[2] == 1000
    assert out[:B].tolist() == [-1] * B and out[2 * B:].tolist() == [-1] * B
    assert int(step) == 2 and pos.tolist() == [11, 21, 31, 41, 51]
    assert torch.equal(nxt, emb[torch.tensor(want, device=DEV)])
    # given ids (a draw): the same advance
    ids = torch.tensor([7, 8, 9, 10, 11], dtype=torch.int64, device=DEV)
    with ops.elem_dtype(dtype):
        ops.rows_advance(None, V, ids, B, emb, nxt, out, step, pos)
        torch.cuda.synchronize()
    assert out[2 * B:].tolist() == [7, 8, 9, 10, 11] and int(step) == 3 and pos.tolist() == [12, 22, 32, 42, 52]
    assert torch.equal(nxt, emb[7:12])


# ---- the decoder -----------------------------------------------------------------------------------------------------------------
def _prompts(lens, H, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, H, generator=g) * 0.3).to(dtype).to(DEV) for n in lens]


def _batch1(dec, embeds, n, **kw):
    out = []
    for b, e in enumerate(embeds):
        r = dec.generate_from_embeds(e, n[b] if isinstance(n, list) else n, **{k: (v[b] if k == "sampling" and isinstance(v, list) else v)
                                                                                for k, v in kw.items()})
        out.append(r)
    return out


def _same(rows, ref, logits=False):
    if logits:
        (ri, rl), ref = rows, ref
        assert [o.tolist() for o in ri] == [o[0].tolist() for o in ref]
        for a, (_, b) in zip(rl, ref):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    else:
        assert [o.tolist() for o in rows] == [o.tolist() for o in ref]


def test_rows_equal_batch1_bf16_packed_and_plain(monkeypatch):
    """Llama-3-8B widths, 2 layers: packed (the default bf16 decode step) and plain weights; ragged prompts, B in 2, 3, 8; ids and fp32
    logits bit-identical to batch 1; graph = eager; EOS at different steps; neighbours and position in the batch do not matter."""
    from spatialrgpt_b200 import ops
    from tests.test_gpu_packed_decode import _decoder
    for pack in (True, False):
        dec = _decoder(monkeypatch, pack, layers=2)
        H = dec.dims.hidden_size
        lens = [37, 5, 120, 64, 17, 99, 1, 80]
        P = _prompts(lens, H, torch.bfloat16, 3)
        ref = _batch1(dec, P, 12, return_logits=True)
        for B in (2, 3, 8):
            _same(dec.generate_rows(P[:B], 12, return_logits=True), ref[:B], logits=True)
        g = dec.generate_rows(P, 12)
        _same(g, [r[0] for r in ref])
        _same(dec.generate_rows(P, 12, use_graph=False), [r[0] for r in ref])
        # other neighbours, other slots
        order = [5, 2, 7, 0]
        _same(dec.generate_rows([P[i] for i in order], 12), [ref[i][0] for i in order])
        # EOS per row, and per-row budgets
        eos = [int(ref[0][0][3]), int(ref[2][0][7])]
        cut = dec.generate_rows(P, [12, 9, 12, 4, 12, 12, 7, 12], eos_token_ids=eos)
        for b in range(8):
            ids = ref[b][0].tolist()[: [12, 9, 12, 4, 12, 12, 7, 12][b]]
            stop = next((k + 1 for k, t in enumerate(ids) if t in eos), len(ids))
            assert cut[b].tolist() == ids[:stop], b
        # stopping criterion that fires on a row-specific length
        fn = lambda ids: ids.numel() == 6 and int(ids[0]) == int(ref[1][0][0])  # noqa: E731
        st = dec.generate_rows(P[:3], 12, stopping_fn=fn)
        assert [o.numel() for o in st] == [12 if int(ref[b][0][0]) != int(ref[1][0][0]) else 6 for b in range(3)]
        # launches: one graph replay per step
        l0 = ops.LAUNCHES
        dec.generate_rows(P[:4], 12)
        extra = ops.LAUNCHES - l0
        l0 = ops.LAUNCHES
        dec.generate_rows(P[:4], 8)
        assert extra - (ops.LAUNCHES - l0) == 4 * dec.stack.rows_kernels
        del dec


def test_rows_sampled_equal_batch1(monkeypatch):
    from tests.test_gpu_packed_decode import _decoder
    dec = _decoder(monkeypatch, True, layers=2)
    lens = [30, 8, 77]
    P = _prompts(lens, dec.dims.hidden_size, torch.bfloat16, 5)
    smp = dict(temperature=0.9, top_p=0.95, top_k=40)
    seeds = [11, 12345, 7]
    ref = _batch1(dec, P, 10, sampling=[dict(smp, seed=s) for s in seeds])
    _same(dec.generate_rows(P, 10, sampling=smp, seeds=seeds), ref)
    _same(dec.generate_rows(P, 10, sampling=smp, seeds=seeds, use_graph=False), ref)
    ref_l = _batch1(dec, P, 10, sampling=[dict(smp, seed=s) for s in seeds], return_logits=True)
    _same(dec.generate_rows(P, 10, sampling=smp, seeds=seeds, return_logits=True), ref_l, logits=True)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_equal_batch1_nf4_and_fp8_refused(dtype):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_beam_batch import _dims
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    lens = [131, 150, 9]
    P = _prompts(lens, d.hidden_size, dtype, 5)
    sd = _llm_state_dict(d, 21)
    got = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512)
        ref = _batch1(dec, P, 10, return_logits=True)
        _same(dec.generate_rows(P, 10, return_logits=True), ref, logits=True)
        got[copy] = dec.generate_rows(P, 10)
        _same(got[copy], [r[0] for r in ref])
        del dec
    _same(got[True], got[False])
    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512)
    with pytest.raises(NotImplementedError):
        dec.generate_rows(P, 4)


def test_rows_fp16_plain():
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_beam_batch import _dims
    from tests.test_gpu_nf4_planes import _llm_state_dict
    from spatialrgpt_b200.weights import LlamaLayerW, LlamaW, interleave_rows
    d = _dims()
    sd = _llm_state_dict(d, 4)
    g = lambda k: sd[k].to(DEV, torch.float16).contiguous()  # noqa: E731
    layers = []
    for l in range(d.num_hidden_layers):
        p = f"model.layers.{l}."
        qkv = torch.cat([g(p + "self_attn.q_proj.weight"), g(p + "self_attn.k_proj.weight"), g(p + "self_attn.v_proj.weight")]).contiguous()
        gu = interleave_rows(g(p + "mlp.gate_proj.weight"), g(p + "mlp.up_proj.weight")).contiguous()
        layers.append(LlamaLayerW(in_norm=g(p + "input_layernorm.weight"), qkv_w=qkv, o_w=g(p + "self_attn.o_proj.weight"),
                                  post_norm=g(p + "post_attention_layernorm.weight"), gateup_w=gu, down_w=g(p + "mlp.down_proj.weight")))
    dec = LlamaDecoder(d, LlamaW(embed=g("model.embed_tokens.weight"), norm=g("model.norm.weight"), lm_head=g("lm_head.weight"), layers=layers),
                       max_seq_len=512)
    P = _prompts([40, 3, 200, 66, 12, 90, 31, 7], d.hidden_size, torch.float16, 9)
    ref = _batch1(dec, P, 9, return_logits=True)
    _same(dec.generate_rows(P, 9, return_logits=True), ref, logits=True)
    _same(dec.generate_rows(P, 9), [r[0] for r in ref])


# ---- generate() ------------------------------------------------------------------------------------------------------------------
def _model():
    from tests.golden.make_golden import CASES
    from tests.test_gpu_fp16 import build_model
    oc, sd, model = build_model(CASES["tiny_masks_gqa"][0], 3, dtype=torch.float16)
    return oc, model


@pytest.mark.parametrize("side", ["left", "right"])
def test_generate_text_padded_batches(side):
    oc, model = _model()
    B, T = 11, 24
    tok = torch.randint(3, 900, (B, T), generator=torch.Generator().manual_seed(1)).to(DEV)
    mask = torch.ones_like(tok)
    for b in range(B):
        k = (3 * b) % 13
        if side == "left":
            mask[b, :k] = 0
        else:
            mask[b, T - k:] = 0
    model.config.llama.tokenizer_padding_side = side
    try:
        for kw in (dict(max_new_tokens=10), dict(max_length=30), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=4, max_new_tokens=9),
                   dict(do_sample=True, temperature=0.8, seed=list(range(100, 100 + B)), max_new_tokens=9)):
            kw = dict(kw, eos_token_id=None, output_logits=True)
            got, lg = model.generate(tok, attention_mask=mask, batch_invariant=True, **kw)
            assert torch.equal(model.generate(tok, attention_mask=mask, batch_invariant=True, use_cuda_graph=False, **dict(kw, output_logits=False)),
                               got)
            from spatialrgpt_b200.llama_decoder import sequence_seeds
            for b in range(B):
                row = tok[b][mask[b].bool()][None]
                one = dict(kw)
                if "seed" in kw:
                    one["seed"] = kw["seed"][b] if isinstance(kw["seed"], list) else sequence_seeds(kw["seed"], B)[b]
                ids, l1 = model.generate(row, **one)
                n = ids.shape[1]
                assert got[b, :n].tolist() == ids[0].tolist(), (kw, b)
                assert torch.equal(lg[b].view(torch.int32), l1[0].view(torch.int32)), (kw, b)
    finally:
        model.config.llama.tokenizer_padding_side = "right"


def test_generate_multimodal_rows_and_eos():
    from oracle import srgpt_oracle as O
    from tests.golden.make_golden import CASES
    oc, model = _model()
    _, n_regions, t_text, kind, _, _ = CASES["tiny_masks_gqa"]
    reqs = [O.synth_request(oc, n_regions, t_text, seed=s, kind=kind) for s in (1234, 77, 5)]
    h = lambda t: t.to(DEV, torch.float16)  # noqa: E731
    T = max(r[0].shape[1] for r in reqs)
    ids = torch.zeros(len(reqs), T, dtype=torch.int64)
    mask = torch.zeros(len(reqs), T, dtype=torch.int64)
    for b, r in enumerate(reqs):
        ids[b, :r[0].shape[1]] = r[0][0]
        mask[b, :r[0].shape[1]] = 1
    args = dict(images=h(torch.cat([r[1] for r in reqs])), depths=h(torch.cat([r[2] for r in reqs])), masks=[h(m) for r in reqs for m in r[3]])
    kw = dict(max_new_tokens=12, eos_token_id=None)
    alone = [model.generate(r[0].to(DEV), images=h(r[1]), depths=h(r[2]), masks=[h(m) for m in r[3]], output_logits=True, **kw) for r in reqs]
    got, lg = model.generate(ids.to(DEV), attention_mask=mask.to(DEV), batch_invariant=True, output_logits=True, **args, **kw)
    for b, (a, al) in enumerate(alone):
        assert got[b, :a.shape[1]].tolist() == a[0].tolist(), b
        assert torch.equal(lg[b].view(torch.int32), al[0].view(torch.int32)), b
    eos = int(alone[1][0][0, 4])
    cut = model.generate(ids.to(DEV), attention_mask=mask.to(DEV), batch_invariant=True, **args, **dict(kw, eos_token_id=eos))
    for b, (a, _) in enumerate(alone):
        want = a[0].tolist()
        want = want[:want.index(eos) + 1] if eos in want else want
        assert cut[b, :len(want)].tolist() == want, b


def test_fp8_model_refused_before_gpu_work(monkeypatch):
    oc, model = _model()
    monkeypatch.setattr(model.llm, "fp8", True)
    tok = torch.randint(3, 900, (2, 8), generator=torch.Generator().manual_seed(1)).to(DEV)
    with pytest.raises(NotImplementedError):
        model.generate(tok, batch_invariant=True, max_new_tokens=4)


def test_eval_spatial_batch_size_4_writes_the_batch1_answers_file(tmp_path):
    """The SpatialRGPT-Bench driver on a synthetic checkpoint: --batch-size 4 (annotations with different images, regions, depth maps
    and numbers of turns) writes the same bytes as --batch-size 1."""
    import json
    from types import SimpleNamespace

    import numpy as np
    from PIL import Image
    from transformers import SiglipImageProcessor

    from spatialrgpt_b200 import eval_spatial as E
    from tests.golden.make_host_golden import ToyTokenizer
    from tests.test_gpu_pipeline import build_model
    from tests.golden.make_golden import CASES
    oc, sd, model = build_model(CASES["tiny_boxes"][0], 17)
    proc = SiglipImageProcessor(size={"height": oc.image_size, "width": oc.image_size})
    model.config.image_aspect_ratio = "resize"
    tok = ToyTokenizer()
    tok.vocab.update({"<mask>": oc.mask_token_id, "<depth>": oc.depth_token_id})
    tok.batch_decode = lambda ids, skip_special_tokens=True: [" ".join(str(int(i)) for i in ids[0])]
    for i in range(3):
        Image.fromarray(np.random.RandomState(i).randint(0, 255, (40, 60, 3), dtype=np.uint8)).save(tmp_path / f"{i}.jpg")
    ann = []
    for i in range(6):
        conv = [{"from": "human", "value": "<image>\n how far is <mask> from <mask> ?"}, {"from": "gpt", "value": "gt"}]
        conv += [{"from": "human", "value": f"is <mask> left of <mask> {i} ?"}, {"from": "gpt", "value": "yes"}] * (i % 3)
        ann.append({"id": i, "image_info": {"file_path": f"{i % 3}.jpg", "height": 40, "width": 60}, "text_q": "q", "qa_info": {},
                    "bbox": [[2 + i, 3, 30, 30], [10, 5, 55 - i, 38]], "conversations": conv})
    (tmp_path / "ann.json").write_text(json.dumps(ann))

    def depth_predictor(rgb):
        return torch.tensor(rgb[::2, ::2, 0], dtype=torch.float32)[None]

    out = {}
    for bs in (1, 4):
        args = SimpleNamespace(model_path="m/tiny", model_base=None, image_folder=str(tmp_path), annotation_file=str(tmp_path / "ann.json"),
                               answers_file=str(tmp_path / f"ans{bs}.jsonl"), conv_mode="llava_v1", num_chunks=1, chunk_idx=0, temperature=0.0,
                               top_p=None, num_beams=1, use_mask=False, batch_size=bs)
        assert E.eval_model(args, depth_predictor=depth_predictor, loader=lambda p, name, base: (tok, model, proc, 4096)) == 12
        out[bs] = open(args.answers_file, "rb").read()
    assert out[1] == out[4]
    assert len({json.loads(l)["pred"] for l in out[1].decode().splitlines()}) > 1
