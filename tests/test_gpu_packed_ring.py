"""The packed decode GEMV's shared-memory ring on the H100: every mode is bit-identical to the plain bf16 kernel, with exceptions
planted in the first, a middle and the last batch of a row and a row holding the most exceptions a row may have.  The K cover
the ring clamped to 0, 1 and 2 slots (1, 2 and >= 3 batches per row)."""
import pytest
import torch

from tests.test_gpu_packed_decode import _same, weights

pytestmark = pytest.mark.gpu
DEV = "cuda"
KS = [1024, 2048, 4096, 5120, 14336]


@pytest.fixture(scope="module")
def ops():
    from spatialrgpt_b200 import ops as _ops
    return _ops


def planted(N, K, seed, std=0.02):
    """weights() with exceptions (exponent field 1) in rows 1 and N - 1 in the first, a middle and the last batch, and row 6 holding
    32 of them spread over the row (its other weights share one exponent, so it has no natural ones)."""
    w = weights(N, K, seed, std=std)
    bits = w.view(torch.int16)
    nb = K // 1024
    cols = torch.tensor([0, 8 * 31 + 7, (nb // 2) * 1024 + 8 * 45 + 2, K - 8 * 32, K - 1], device=DEV)
    for r in (1, N - 1):
        bits[r, cols] = (bits[r, cols] & -32641) | 0x0080  # keep sign and mantissa (0x807F)
    g = torch.Generator().manual_seed(seed + 1)
    row = (torch.randint(0, 1 << 16, (K,), generator=g) & 0x807F) | (120 << 7)
    bits[6] = torch.where(row >= 1 << 15, row - (1 << 16), row).to(torch.int16).to(DEV)
    full = torch.linspace(0, K - 1, 32).long().to(DEV)
    bits[6, full] = (bits[6, full] & -32641) | 0x0080
    return w


def pack(ops, w):
    p, why = ops.pack12(w)
    assert why is None, why
    n = p.row_ptr.cpu()
    assert int(n[7] - n[6]) == 32 and int(n[2] - n[1]) >= 5
    return p


@pytest.mark.parametrize("K", KS)
def test_plain_and_swiglu_modes_at_every_depth(ops, K):
    N = 1024
    w = planted(N, K, K)
    p = pack(ops, w)
    x = (torch.randn(K, generator=torch.Generator().manual_seed(1)) * 0.5).to(torch.bfloat16).to(DEV)
    res = torch.randn(N, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).to(DEV)
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(3))).to(torch.bfloat16).to(DEV)
    y0 = torch.empty(N, dtype=torch.bfloat16, device=DEV)
    a0 = torch.empty(N // 2, dtype=torch.bfloat16, device=DEV)
    ops.gemv(x, w, y0, residual=res)
    ops.gemv(x, w, a0, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)

    y, a = torch.full_like(y0, 7.0), torch.full_like(a0, 7.0)
    ops.gemv_packed(x, p, y, residual=res)
    ops.gemv_packed(x, p, a, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
    assert _same(y0, y), f"plain, K={K}"
    assert _same(a0, a), f"swiglu, K={K}"


@pytest.mark.parametrize("K", KS)
def test_qkv_rope_mode_at_every_depth(ops, K):
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.llama_decoder import build_rope_tables
    nh, nkv, hd, page = 8, 2, 128, 16
    N = (nh + 2 * nkv) * hd
    w = planted(N, K, 7 + K)
    p = pack(ops, w)
    cos, sin = build_rope_tables(LlamaDims(), 512, DEV)
    x = torch.randn(K, generator=torch.Generator().manual_seed(8)).to(torch.bfloat16).to(DEV)
    nw = (1 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(9))).to(torch.bfloat16).to(DEV)
    pos = torch.tensor([300], dtype=torch.int32, device=DEV)
    pt = torch.arange(40, dtype=torch.int32, device=DEV).flip(0).contiguous()

    def run(packed):
        pages = torch.zeros(40, 2, page, nkv, hd, dtype=torch.bfloat16, device=DEV)
        y = torch.empty(nh * hd, dtype=torch.bfloat16, device=DEV)
        kw = dict(norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=nh, n_kv_heads=nkv, head_dim=hd, cos_tab=cos, sin_tab=sin, pos=pos,
                  kv_pages=pages, page_table=pt, page_size=page)
        (ops.gemv_packed(x, p, y, **kw) if packed else ops.gemv(x, w, y, **kw))
        return y, pages

    y0, pages0 = run(False)
    assert pages0.abs().sum() > 0
    y, pages = run(True)
    assert _same(y0, y) and _same(pages0, pages), f"K={K}"


@pytest.mark.parametrize("K", KS)
def test_lm_head_with_an_odd_vocabulary_at_every_depth(ops, K):
    V = 4099
    w = planted(V, K, 11 + K, std=0.08)
    p = pack(ops, w)
    x = torch.randn(K, generator=torch.Generator().manual_seed(12)).to(torch.bfloat16).to(DEV)
    nw = torch.ones(K, dtype=torch.bfloat16, device=DEV)
    embed = torch.randn(V, K, generator=torch.Generator().manual_seed(13)).to(torch.bfloat16).to(DEV)
    ws = ops.lm_head_workspace(V, DEV)

    def run(packed):
        ids = torch.zeros(4, dtype=torch.int64, device=DEV)
        step, pos = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
        logits = torch.empty(V, dtype=torch.float32, device=DEV)
        nxt = torch.empty(K, dtype=torch.bfloat16, device=DEV)
        f = ops.lm_head_argmax_packed if packed else ops.lm_head_argmax
        f(x, p if packed else w, nw, 1e-5, ws, ids, step, pos, embed_table=embed, next_x=nxt, logits_out=logits)
        return logits, ids, nxt

    lg0, ids0, nxt0 = run(False)
    assert int(ids0[0]) == int(lg0.argmax())
    lg, ids, nxt = run(True)
    assert torch.equal(lg0, lg) and torch.equal(ids0, ids) and _same(nxt0, nxt), f"K={K}"
