"""forward(output_hidden_states=True, output_attentions=True) on the H100: the probability kernel against an fp64 softmax and the flash
kernels, the probed prefill against the unprobed one bit for bit on every weight format, the outputs against the fp32 oracle
(tests/forward_outputs_oracle.py), a multimodal request's region rows, and padded batches on either side, in both element types."""
import functools

import pytest
import torch

from oracle import srgpt_oracle as O
from tests.forward_outputs_oracle import llama_forward_outputs
from tests.golden.make_golden import CASES
from tests.test_gpu_configs import WIDTHS

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
MANT = {torch.bfloat16: 7, torch.float16: 10}


def _model(case_kw, dtype, quantization=None, copy=True, seed=17, max_seq_len=512):
    from spatialrgpt_b200 import LlavaConfig, LlamaDims, VisionConfig
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    from spatialrgpt_b200.weights import from_state_dicts
    oc = O.OracleConfig(**case_kw)
    cfg = LlavaConfig(
        vision=VisionConfig(image_size=oc.image_size, patch_size=oc.patch_size, hidden_size=oc.v_hidden, num_hidden_layers=oc.v_layers,
                            num_attention_heads=oc.v_heads, intermediate_size=oc.v_inter, layer_norm_eps=oc.v_eps),
        llama=LlamaDims(hidden_size=oc.hidden, num_hidden_layers=oc.layers, num_attention_heads=oc.heads, num_key_value_heads=oc.kv_heads,
                        head_dim=oc.head_dim, intermediate_size=oc.inter, vocab_size=oc.vocab, rope_theta=oc.rope_theta, rms_norm_eps=oc.rms_eps),
        enable_region=oc.enable_region, enable_depth=oc.enable_depth, mm_vision_select_layer=oc.select_layer)
    cfg.llm_mask_token_id, cfg.llm_depth_token_id = oc.mask_token_id, oc.depth_token_id
    sd = _weights(tuple(sorted(case_kw.items())), seed)
    w = from_state_dicts(cfg, sd, DEV, dtype=dtype, quantization=quantization, nf4_dequantized_copy=copy)
    return oc, sd, LlavaLlamaModel(cfg, w, max_seq_len=max_seq_len)


@functools.lru_cache(maxsize=2)
def _weights(kw_items, seed):
    return O.make_weights(O.OracleConfig(**dict(kw_items)), seed=seed)


def _ulp(ref: torch.Tensor, dtype) -> torch.Tensor:
    """One element-type ulp at |ref| (the subnormal spacing below the smallest normal)."""
    fi = torch.finfo(dtype)
    a = ref.abs().clamp_min(fi.smallest_normal)
    return torch.exp2(torch.floor(torch.log2(a)) - MANT[dtype])


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nh,nkv", [(8, 2), (4, 4)])
def test_probability_kernel(dtype, nh, nkv):
    from spatialrgpt_b200 import ops
    hd, lens, offs, R = 128, [37, 130, 64, 200], [0, 5, 70, 1], 203
    g = torch.Generator().manual_seed(nh * 10 + nkv)
    T = sum(lens)
    q = torch.randn(T, nh * hd, generator=g).to(dtype).to(DEV)
    k = torch.randn(T, nkv * hd, generator=g).to(dtype).to(DEV)
    v = torch.randn(T, nkv * hd, generator=g).to(dtype).to(DEV)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    row_off = torch.tensor(offs, dtype=torch.int32, device=DEV)
    scale = hd ** -0.5
    with ops.elem_dtype(dtype):
        out = torch.full((len(lens), nh, R, R), float("nan"), dtype=dtype, device=DEV)
        ops.attention_probs(q, k, nh, nkv, hd, scale, out, cu_seqlens=cu, max_seqlen=max(lens), row_off=row_off)
        flash = ops.attention_prefill_varlen(q, k, v, cu, max(lens), nh, nkv, hd, scale, True)
    torch.cuda.synchronize()
    out, flash = out.cpu(), flash.cpu()
    assert not torch.isnan(out).any(), "an entry of the output blocks was not written"
    o = 0
    for b, (n, off) in enumerate(zip(lens, offs)):
        qb = q[o:o + n].cpu().double().view(n, nh, hd).transpose(0, 1)
        kb = k[o:o + n].cpu().double().view(n, nkv, hd).transpose(0, 1).repeat_interleave(nh // nkv, 0)
        vb = v[o:o + n].cpu().double().view(n, nkv, hd).transpose(0, 1).repeat_interleave(nh // nkv, 0)
        s = (qb @ kb.transpose(1, 2)) * scale
        causal = torch.arange(n)[None, :] <= torch.arange(n)[:, None]
        ref = torch.softmax(s.masked_fill(~causal, float("-inf")), -1)
        blk = out[b, :, off:off + n, off:off + n].double()
        assert bool(((blk - ref).abs() <= _ulp(ref, dtype)).all()), float((blk - ref).abs().max())
        assert bool((blk[:, ~causal] == 0).all())
        rest = out[b].clone()
        rest[:, off:off + n, off:off + n] = 0
        assert bool((rest == 0).all()), "entries outside the sequence's block must be 0"
        # P V from the returned probabilities against the flash kernel, both against fp64
        pv = (blk @ vb).transpose(0, 1).reshape(n, nh * hd)
        exact = (ref @ vb).transpose(0, 1).reshape(n, nh * hd)
        fl = flash[o:o + n].double()
        assert float((pv - exact).abs().max()) <= 2 * float((fl - exact).abs().max()) + 4 * 2.0 ** -MANT[dtype], b
        o += n


# ---- flags on, off and absent ------------------------------------------------------------------------------------------------------
C2 = dict(WIDTHS["c2_llama3_8b_448"][0])
FORMATS = {"elem": (None, True), "nf4_copy": ("nf4", True), "nf4_planes": ("nf4", False), "fp8": ("fp8", True)}


def _text_batch(vocab, lens, left, seed=5):
    g = torch.Generator().manual_seed(seed)
    T = max(lens)
    ids = torch.randint(3, vocab - 3, (len(lens), T), generator=g)
    am = torch.zeros(len(lens), T, dtype=torch.int64)
    for b, n in enumerate(lens):
        if left:
            am[b, T - n:] = 1
        else:
            am[b, :n] = 1
    return ids, am


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_flags_do_not_change_logits_loss_or_launches(dtype, fmt):
    from spatialrgpt_b200 import ops
    quant, copy = FORMATS[fmt]
    oc, _, model = _model(C2, dtype, quant, copy)
    for lens, left in (([70], True), ([70, 33, 129], True), ([70, 33, 129], False)):
        ids, am = _text_batch(oc.vocab, lens, left)
        ids, am = ids.to(DEV), am.to(DEV)
        labels = ids.clone()
        labels[am == 0] = -100
        n0 = ops.LAUNCHES
        ref = model.forward(input_ids=ids, attention_mask=am, labels=labels)
        n1 = ops.LAUNCHES
        off = model.forward(input_ids=ids, attention_mask=am, labels=labels, output_hidden_states=False, output_attentions=None)
        n2 = ops.LAUNCHES
        on = model.forward(input_ids=ids, attention_mask=am, labels=labels, output_hidden_states=True, output_attentions=True)
        assert n2 - n1 == n1 - n0, "flags off must launch exactly what no flags launch"
        assert off.hidden_states is None and off.attentions is None
        for r in (off, on):
            assert torch.equal(r.logits, ref.logits) and torch.equal(r.loss, ref.loss)
        L = oc.layers
        assert len(on.hidden_states) == L + 1 and len(on.attentions) == L
        assert on.hidden_states[0].dtype == dtype and on.attentions[0].shape == (len(lens), oc.heads, max(lens), max(lens))
        rows = [slice(max(lens) - n, max(lens)) if left else slice(0, n) for n in lens]
        with ops.elem_dtype(dtype):  # the valid rows packed as forward() packs them: the same GEMM shape as its lm_head call
            hn = torch.cat([on.hidden_states[-1][b, r] for b, r in enumerate(rows)]).contiguous()
            lg = ops.gemm(hn, model.weights.llama.lm_head, out=model.llm._logits_buffer(hn.shape[0])).float()
        assert torch.equal(lg, torch.cat([ref.logits[b, r] for b, r in enumerate(rows)])), "hidden_states[-1] must be the rows lm_head reads"
        del on


# ---- against the fp32 oracle -------------------------------------------------------------------------------------------------------
def _errors(model, oc, sd, emb, dtype):
    """(our error, the oracle-in-dtype error) against the fp32 oracle: max abs over hidden states and attentions, each pair."""
    out = model.forward(inputs_embeds=emb[None].to(DEV, dtype), output_hidden_states=True, output_attentions=True)
    _, h32, a32 = llama_forward_outputs(oc, sd["llm"], emb, torch.float32)
    _, hdt, adt = llama_forward_outputs(oc, sd["llm"], emb, dtype)
    res = {}
    for name, ours, r32, rdt in (("hidden", out.hidden_states, h32, hdt), ("attn", out.attentions, a32, adt)):
        e_ours = max(float((o[0].cpu().float() - r.float()).abs().max()) for o, r in zip(ours, r32))
        e_ref = max(float((d.float() - r.float()).abs().max()) for d, r in zip(rdt, r32))
        res[name] = (e_ours, e_ref)
    return res


FACTOR = 4  # ours may be this many times the oracle-in-dtype error: GEMM blockings and fp32 softmax order differ from torch's


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["tiny_masks_gqa", "c1_sheared_336", "c2_llama3_8b_448"])
def test_against_the_fp32_oracle(dtype, name):
    kw = CASES[name][0] if name in CASES else WIDTHS[name][0]
    oc, sd, model = _model(kw, dtype)
    g = torch.Generator().manual_seed(9)
    emb = (torch.randn(97, oc.hidden, generator=g) * 0.3).to(dtype).float()
    for what, (ours, ref) in _errors(model, oc, sd, emb, dtype).items():
        assert ours <= FACTOR * ref + 1e-6, (what, ours, ref)


@pytest.mark.parametrize("dtype", DTYPES)
def test_multimodal_mask_rows_over_the_image(dtype):
    """tiny_masks_gqa with an image, masks and depth: the attention rows of the <mask> rows over the image-patch columns (located through
    the splice plan) against the oracle over the same spliced rows."""
    from spatialrgpt_b200.splice_plan import SRC_TOKENS
    kw, n_regions, t_text, kind, _, _ = CASES["tiny_masks_gqa"]
    oc, sd, model = _model(kw, dtype)
    input_ids, images, depths, masks = O.synth_request(oc, n_regions, t_text, seed=1234, kind=kind)
    out = model.forward(input_ids=input_ids.to(DEV), images=images.to(DEV), depths=depths.to(DEV), masks=[m.to(DEV) for m in masks],
                        output_hidden_states=True, output_attentions=True)
    src_id, _ = model._last_plan_rows
    src = src_id.reshape(-1)[:out.attentions[0].shape[-1]]
    image_cols = torch.nonzero(src == 1).flatten()
    mask_rows = torch.nonzero(src == 2).flatten()
    assert image_cols.numel() > 0 and mask_rows.numel() > 0 and SRC_TOKENS == 0
    emb = out.hidden_states[0][0].float().cpu()
    _, _, a32 = llama_forward_outputs(oc, sd["llm"], emb, torch.float32)
    _, _, adt = llama_forward_outputs(oc, sd["llm"], emb, dtype)
    for l in range(oc.layers):
        sel = lambda a: a[:, mask_rows][:, :, image_cols].float()  # noqa: E731
        ours, r32, rdt = sel(out.attentions[l][0].cpu()), sel(a32[l]), sel(adt[l])
        assert float((ours - r32).abs().max()) <= FACTOR * float((rdt - r32).abs().max()) + 1e-6, l


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("left", [True, False])
def test_padded_batches_equal_batch_one(dtype, left):
    oc, _, model = _model(CASES["tiny_masks_gqa"][0], dtype)
    lens = [40, 13, 77]
    ids, am = _text_batch(oc.vocab, lens, left, seed=2)
    batch = model.forward(input_ids=ids.to(DEV), attention_mask=am.to(DEV), output_hidden_states=True, output_attentions=True)
    T = max(lens)
    for b, n in enumerate(lens):
        rows = slice(T - n, T) if left else slice(0, n)
        one = model.forward(input_ids=ids[b:b + 1, rows].to(DEV), output_hidden_states=True, output_attentions=True)
        for hb, h1 in zip(batch.hidden_states, one.hidden_states):
            assert torch.allclose(hb[b, rows].float(), h1[0].float(), rtol=2e-2, atol=2e-2 * float(h1.float().abs().max()))
            rest = hb[b].clone()
            rest[rows] = 0
            assert bool((rest == 0).all())
        for ab, a1 in zip(batch.attentions, one.attentions):
            assert torch.allclose(ab[b][:, rows, rows].float(), a1[0].float(), atol=2e-2)
            rest = ab[b].clone()
            rest[:, rows, rows] = 0
            assert bool((rest == 0).all())
