"""The 12-bit lossless packing of decode weights on the H100: the device packer against the numpy reference, every packed GEMV
mode against the plain kernel bit for bit (with planted exceptions and an odd vocabulary), graph decode steps of a Llama-3-8B
shaped decoder with packing on and off, the matrices that stay plain, and the round-trip check."""
import dataclasses

import numpy as np
import pytest
import torch

from tests.test_packed_weights_cpu import pack12_np

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def weights(N, K, seed, std=0.02, n_planted=0):
    """bf16 [N, K] ~ N(0, std) with n_planted extra exceptions (exponent 1, far below any row's window) spread over the rows,
    including the first and last chunk of lanes 0 and 31 of a batch."""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) * std).to(torch.bfloat16)
    if n_planted:
        bits = w.view(torch.int16)
        rows = torch.randint(0, N, (n_planted,), generator=g)
        cols = torch.randint(0, K, (n_planted,), generator=g)
        cols[:4] = torch.tensor([0, 8 * 31 + 7, K - 8 * 32, K - 1])
        bits[rows, cols] = (bits[rows, cols] & -32641) | 0x0080  # keep sign and mantissa (0x807F), exponent field 1
    return w.to(DEV)


def test_device_packer_matches_the_numpy_reference(ops):
    w = weights(96, 3072, 0, n_planted=40)
    p, why = ops.pack12(w)
    assert why is None
    ref, _ = pack12_np(w.view(torch.int16).cpu().numpy().view(np.uint16))
    for k in ("sm", "ex", "base", "row_ptr"):
        assert np.array_equal(getattr(p, k).cpu().numpy().view(ref[k].dtype), ref[k]), k
    n = int(p.row_ptr[-1])
    assert n >= 40 and np.array_equal(p.exc[:n].cpu().numpy(), ref["exc"])
    assert torch.equal(ops.unpack12(p).view(torch.int16), w.view(torch.int16))


def _same(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a, b.view(torch.int16) if b.dtype == torch.bfloat16 else b)


@pytest.mark.parametrize("K", [1024, 4096, 14336])
def test_plain_and_swiglu_modes_are_bit_identical(ops, K):
    N = 2048
    w = weights(N, K, K, n_planted=300)
    p, why = ops.pack12(w)
    assert why is None and int(p.row_ptr[-1]) >= 300
    x = (torch.randn(K, generator=torch.Generator().manual_seed(1)) * 0.5).to(torch.bfloat16).to(DEV)
    res = torch.randn(N, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).to(DEV)
    y0, y1 = torch.empty(N, dtype=torch.bfloat16, device=DEV), torch.empty(N, dtype=torch.bfloat16, device=DEV)
    ops.gemv(x, w, y0, residual=res)
    ops.gemv_packed(x, p, y1, residual=res)
    assert _same(y0, y1)
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(3))).to(torch.bfloat16).to(DEV)
    a0, a1 = torch.empty(N // 2, dtype=torch.bfloat16, device=DEV), torch.empty(N // 2, dtype=torch.bfloat16, device=DEV)
    ops.gemv(x, w, a0, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
    ops.gemv_packed(x, p, a1, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
    assert _same(a0, a1)


def test_qkv_rope_mode_is_bit_identical(ops):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, K, page = 32, 8, 128, 4096, 16
    N = (nh + 2 * nkv) * hd
    w = weights(N, K, 7, n_planted=200)
    p, _ = ops.pack12(w)
    cos, sin = build_rope_tables(LlamaDims(), 512, DEV)
    x = torch.randn(K, generator=torch.Generator().manual_seed(8)).to(torch.bfloat16).to(DEV)
    nw = torch.ones(K, dtype=torch.bfloat16, device=DEV)
    pos = torch.tensor([300], dtype=torch.int32, device=DEV)
    pt = torch.arange(40, dtype=torch.int32, device=DEV).flip(0).contiguous()
    outs = []
    for packed in (False, True):
        pages = torch.zeros(40, 2, page, nkv, hd, dtype=torch.bfloat16, device=DEV)
        y = torch.empty(nh * hd, dtype=torch.bfloat16, device=DEV)
        kw = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, cos_tab=cos, sin_tab=sin, pos=pos,
                  kv_pages=pages, page_table=pt, page_size=page)
        (ops.gemv_packed(x, p, y, **kw) if packed else ops.gemv(x, w, y, **kw))
        outs.append((y, pages))
    assert _same(outs[0][0], outs[1][0]) and _same(outs[0][1], outs[1][1])
    assert outs[0][1].abs().sum() > 0


def test_lm_head_with_an_odd_vocabulary_is_bit_identical(ops):
    V, K = 128259, 4096
    w = weights(V, K, 11, std=0.08, n_planted=500)
    p, why = ops.pack12(w)
    assert why is None
    x = torch.randn(K, generator=torch.Generator().manual_seed(12)).to(torch.bfloat16).to(DEV)
    nw = torch.ones(K, dtype=torch.bfloat16, device=DEV)
    embed = torch.randn(V, K, generator=torch.Generator().manual_seed(13)).to(torch.bfloat16).to(DEV)
    ws = ops.lm_head_workspace(V, DEV)
    res = []
    for packed in (False, True):
        ids = torch.zeros(4, dtype=torch.int64, device=DEV)
        step, pos = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
        logits = torch.empty(V, dtype=torch.float32, device=DEV)
        nxt = torch.empty(K, dtype=torch.bfloat16, device=DEV)
        f = ops.lm_head_argmax_packed if packed else ops.lm_head_argmax
        f(x, p if packed else w, nw, 1e-5, ws, ids, step, pos, embed_table=embed, next_x=nxt, logits_out=logits)
        res.append((logits, ids, nxt))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and _same(res[0][2], res[1][2])
    assert int(res[0][1][0]) == int(res[0][0].argmax())


def test_matrices_that_must_stay_plain(ops):
    w = weights(64, 1024, 20)
    for bad in (float("inf"), float("-inf"), float("nan")):
        v = w.clone()
        v[5, 17] = bad
        p, why = ops.pack12(v)
        assert p is None and "Inf or NaN" in why
    dense = (torch.randn(64, 1024) * torch.exp(torch.empty(64, 1024).uniform_(-30, 0))).to(torch.bfloat16).to(DEV)
    assert ops.pack12(dense)[0] is None
    row = w.clone()
    row.view(torch.int16)[3, :40] = 0x0080  # 40 exceptions in one row: more than a lane register per entry can hold
    p, why = ops.pack12(row)
    assert p is None and why.startswith("a row has")
    assert ops.pack12(weights(64, 1000, 21))[1].startswith("K = 1000")


def test_round_trip_check_raises_on_a_corrupted_plane(ops):
    w = weights(64, 2048, 30, n_planted=10)
    p, _ = ops.pack12(w)
    ops.verify12(p, w)
    for plane, idx in (("sm", (7, 100)), ("ex", (9, 5)), ("exc", (0,))):
        t = getattr(p, plane)
        t[idx] ^= 1
        with pytest.raises(ops.SrgptError):
            ops.verify12(p, w)
        t[idx] ^= 1
    ops.verify12(p, w)


def _decoder(monkeypatch, pack, layers=2):
    """A Llama-3-8B-shaped decoder (full width, `layers` layers) with seeded weights; layer 0's down_proj has a row with 40
    exceptions, so it stays plain while the other matrices are packed."""
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from spatialrgpt_b200.weights import LlamaLayerW, LlamaW
    monkeypatch.setenv("SRGPT_DECODE_PACK", "1" if pack else "0")
    d = dataclasses.replace(LlamaDims(), num_hidden_layers=layers)
    H, I, V = d.hidden_size, d.intermediate_size, d.vocab_size
    qkv_n = (d.num_attention_heads + 2 * d.num_key_value_heads) * d.head_dim
    norm = lambda s: (1 + 0.05 * torch.randn(H, generator=torch.Generator().manual_seed(s))).to(torch.bfloat16).to(DEV)  # noqa: E731
    lws = []
    for l in range(layers):
        down = weights(H, I, 100 + 10 * l + 3)
        if l == 0:
            down.view(torch.int16)[5, :40] = 0x0080
        lws.append(LlamaLayerW(in_norm=norm(l), qkv_w=weights(qkv_n, H, 100 + 10 * l), o_w=weights(H, H, 100 + 10 * l + 1), post_norm=norm(50 + l),
                               gateup_w=weights(2 * I, H, 100 + 10 * l + 2), down_w=down))
    w = LlamaW(embed=weights(V, H, 1, std=0.3), norm=norm(99), lm_head=weights(V, H, 2, std=0.08), layers=lws)
    return LlamaDecoder(d, w, max_seq_len=256)


def test_graph_decode_with_packing_matches_the_bf16_step(ops, monkeypatch):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    dec1 = _decoder(monkeypatch, True)
    assert dec1.decode_pack["layers.0.down"].startswith("a row has")
    assert all(v == "packed" for k, v in dec1.decode_pack.items() if k != "layers.0.down")
    x = (torch.randn(20, 4096, generator=torch.Generator().manual_seed(5)) * 0.3).to(torch.bfloat16).to(DEV)
    ids1 = dec1.generate_from_embeds(x, 40)
    ids1_l, lg1 = dec1.generate_from_embeds(x, 40, use_graph=False, return_logits=True)
    monkeypatch.setenv("SRGPT_DECODE_PACK", "0")
    dec0 = LlamaDecoder(dec1.dims, dec1.w, max_seq_len=256)  # the same bf16 weights
    del dec1
    torch.cuda.empty_cache()
    assert dec0.decode_pack == {} and dec0._packed_array is None
    ids0 = dec0.generate_from_embeds(x, 40)
    ids0_l, lg0 = dec0.generate_from_embeds(x, 40, use_graph=False, return_logits=True)
    assert ids0.numel() == 40 and torch.equal(ids0, ids1)
    assert torch.equal(ids0_l, ids1_l) and torch.equal(ids0, ids0_l)
    assert torch.equal(lg0, lg1)
