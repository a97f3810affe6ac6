"""torch.Tensor-facing wrappers over the C-ABI (one function per exported kernel group).

torch is used for device memory and streams only; every computation below is a hand-written
sm_90a kernel in ``csrc/``.  All wrappers raise ``SrgptError`` on any failure (no fallbacks).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import SrgptError
from ._lib import check as _check_rc
from .weights import Fp8W, Nf4W, Packed12W

_KERNELS_PER_CALL = {"srgpt_lm_head_local_best_bf16": 2, "srgpt_mask_pool_bf16": 2, "srgpt_mask_weights": 2, "srgpt_lm_head_argmax_bf16": 2, "srgpt_depth_to_u8x3": 3,
                     "srgpt_lm_head_argmax_packed_bf16": 2, "srgpt_nf4_double_quant": 2}


def check(rc: int, what: str) -> None:
    global LAUNCHES
    _check_rc(rc, what)
    LAUNCHES += _KERNELS_PER_CALL.get(what, 1)

EPI_NONE, EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GELU_ERF, EPI_BIAS_RESIDUAL, EPI_SWIGLU, EPI_BIAS_QUICK_GELU = range(7)
GEMV_PLAIN, GEMV_SWIGLU, GEMV_QKV_ROPE = range(3)
ORDER_ROWMAJOR, ORDER_NESTED = 0, 2

BF16 = torch.bfloat16
F16 = torch.float16
_ELEM_NAMES = {torch.bfloat16: "bf16", torch.float16: "f16"}
_ELEM_DTYPES = {v: k for k, v in _ELEM_NAMES.items()}


def ELEM() -> torch.dtype:
    """The 16-bit element type the ops currently compute in (which build of the library ``_lib.load()`` hands out)."""
    return _ELEM_DTYPES[_lib.current_elem()]


class elem_dtype:
    """``with ops.elem_dtype(torch.float16): ...`` - route the ops through the IEEE-half build of the kernels (the reference loader's
    default dtype, llava/model/builder.py:62) instead of the bfloat16 one.  The models wrap their public entry points in this with their
    own dtype, so a bf16 and an fp16 model can live in one process (one thread at a time: the setting is process-wide)."""

    def __init__(self, dtype: torch.dtype):
        if dtype not in _ELEM_NAMES:
            raise SrgptError(f"unsupported compute dtype {dtype}: the kernels are built for torch.bfloat16 and torch.float16")
        self.name = _ELEM_NAMES[dtype]

    def __enter__(self):
        self.prev = _lib.set_elem(self.name)
        return self

    def __exit__(self, *exc):
        _lib.set_elem(self.prev)
        return False


def in_own_dtype(fn):
    """Method decorator: run the method with the kernels of ``self.dtype`` (torch.bfloat16 / torch.float16)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        with elem_dtype(self.dtype):
            return fn(self, *a, **k)

    return wrapped


# number of OUR kernels launched through this module (bench.py's `gpu_launches`); CUDA-graph replays
# are added by the decoder (kernels_per_decode_step per replay)
LAUNCHES = 0


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise SrgptError(f"{name}: expected a CUDA tensor (the sm_90a kernels have no CPU fallback)")
    if t.dtype != dtype:
        raise SrgptError(f"{name}: expected dtype {dtype}, got {t.dtype}")


def _rowmajor2d(t: torch.Tensor, name: str) -> int:
    if t.dim() != 2 or t.stride(1) != 1:
        raise SrgptError(f"{name}: expected a 2-D tensor with unit inner stride, got shape {tuple(t.shape)} strides {t.stride()}")
    return t.stride(0)


# workspace of the short-prompt GEMM configuration (include/srgpt_b200.h: srgpt_gemm_set_workspace): owned here, one per process,
# registered on the first GEMM call on a device (the library keeps only the pointer)
_GEMM_WS = {}  # element type -> buffer (each build of the library keeps its own registration)


def _ensure_gemm_workspace(device) -> None:
    elem = _lib.current_elem()
    if elem in _GEMM_WS:
        return
    lib = _lib.load()
    n = int(lib.srgpt_gemm_workspace_bytes())
    ws = _GEMM_WS[elem] = torch.zeros(n + 1024, dtype=torch.uint8, device=device)
    off = (-ws.data_ptr()) % 1024
    torch.cuda.synchronize(device)  # the zero fill is complete before any kernel polls the flags
    check(lib.srgpt_gemm_set_workspace(ws.data_ptr() + off, n), "srgpt_gemm_set_workspace")
    global LAUNCHES
    LAUNCHES -= 1


# ------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         epilogue: int = EPI_NONE, out: Optional[torch.Tensor] = None, out_fp32: bool = False,
         res_row_mod: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue(a[M,K] @ w[N,K]^T) on the Hopper tensor cores (wgmma)."""
    _need(a, ELEM(), "gemm.a"); _need(w, ELEM(), "gemm.w")
    _ensure_gemm_workspace(a.device)
    lda, ldw = _rowmajor2d(a, "gemm.a"), _rowmajor2d(w, "gemm.w")
    M, K = a.shape
    N, K2 = w.shape
    if K != K2:
        raise SrgptError(f"gemm: K mismatch {K} vs {K2}")
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float32 if out_fp32 else ELEM(), device=a.device)
    else:
        _need(out, torch.float32 if out_fp32 else ELEM(), "gemm.out")
        if out.shape != (M, n_out):
            raise SrgptError(f"gemm.out: expected {(M, n_out)}, got {tuple(out.shape)}")
    ldc = _rowmajor2d(out, "gemm.out")
    ldr = 0
    if residual is not None:
        _need(residual, ELEM(), "gemm.residual")
        ldr = _rowmajor2d(residual, "gemm.residual")
    if bias is not None:
        _need(bias, ELEM(), "gemm.bias")
    check(_lib.load().srgpt_gemm_bf16(_p(a), lda, _p(w), ldw, _p(out), ldc, M, N, K, _p(bias), _p(residual), ldr,
                                      res_row_mod, epilogue, 1 if out_fp32 else 0, _stream()), "srgpt_gemm_bf16")
    return out


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float, act: int = 0,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need(x, ELEM(), "layernorm.x")
    ldx = _rowmajor2d(x, "layernorm.x")
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=ELEM(), device=x.device)
    check(_lib.load().srgpt_layernorm_bf16(_p(x), ldx, _p(weight), _p(bias), _p(out), _rowmajor2d(out, "layernorm.out"),
                                           rows, cols, eps, act, _stream()), "srgpt_layernorm_bf16")
    return out


def downsample_layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> torch.Tensor:
    """x [n, side*side, C] -> [n, ceil(side/2)^2, 4C] (DownSampleBlock + LayerNorm)."""
    _need(x, ELEM(), "downsample_layernorm.x")
    if x.dim() != 3 or not x.is_contiguous():
        raise SrgptError("downsample_layernorm: expected contiguous [n, side*side, C]")
    n, hw, c = x.shape
    side = int(round(hw ** 0.5))
    if side * side != hw:
        raise SrgptError(f"downsample_layernorm: {hw} tokens is not a square grid")
    half = (side + 1) // 2
    out = torch.empty((n, half * half, 4 * c), dtype=ELEM(), device=x.device)
    check(_lib.load().srgpt_downsample_layernorm_bf16(_p(x), _p(weight), _p(bias), _p(out), n, side, c, eps, _stream()),
          "srgpt_downsample_layernorm_bf16")
    return out


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need(x, ELEM(), "rmsnorm.x")
    ldx = _rowmajor2d(x, "rmsnorm.x")
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=ELEM(), device=x.device)
    check(_lib.load().srgpt_rmsnorm_bf16(_p(x), ldx, _p(weight), _p(out), _rowmajor2d(out, "rmsnorm.out"), rows, cols, eps,
                                         _stream()), "srgpt_rmsnorm_bf16")
    return out


def patchify(images: torch.Tensor, patch: int, ldk: int) -> torch.Tensor:
    if not images.is_cuda or images.dim() != 4 or images.shape[1] != 3 or not images.is_contiguous():
        raise SrgptError("patchify: expected a contiguous CUDA tensor [n, 3, R, R]")
    if images.dtype not in (torch.float32, ELEM()):
        raise SrgptError(f"patchify: unsupported dtype {images.dtype}")
    n, _, R, R2 = images.shape
    if R != R2:
        raise SrgptError("patchify: square images only")
    P = R // patch
    out = torch.empty((n * P * P, ldk), dtype=ELEM(), device=images.device)
    check(_lib.load().srgpt_patchify_bf16(_p(images), 1 if images.dtype == ELEM() else 0, _p(out), n, R, patch, ldk, _stream()),
          "srgpt_patchify_bf16")
    return out


def splice_rows(src0: torch.Tensor, src1, src2, src3, src_id: torch.Tensor, src_row: torch.Tensor,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[r] = row src_row[r] of source src_id[r] (a fresh [rows, cols] tensor, or ``out``, contiguous)."""
    _need(src0, ELEM(), "splice.src0"); _need(src_id, torch.int32, "splice.src_id"); _need(src_row, torch.int32, "splice.src_row")
    cols = src0.shape[-1]
    rows = src_id.numel()
    for s in (src1, src2, src3):
        if s is not None:
            _need(s, ELEM(), "splice.src")
            if s.shape[-1] != cols or not s.is_contiguous():
                raise SrgptError("splice: all sources must be contiguous with the same width")
    if out is None:
        out = torch.empty((rows, cols), dtype=ELEM(), device=src0.device)
    else:
        _need(out, ELEM(), "splice.out")
        if tuple(out.shape) != (rows, cols) or not out.is_contiguous():
            raise SrgptError(f"splice: out must be contiguous [{rows}, {cols}], got shape {tuple(out.shape)}")
    check(_lib.load().srgpt_splice_rows_bf16(_p(src0), _p(src1), _p(src2), _p(src3), _p(src_id), _p(src_row), _p(out), rows,
                                             cols, _stream()), "srgpt_splice_rows_bf16")
    return out


# ------------------------------------------------------------------------------------------------
def mask_weights(masks: torch.Tensor, side: int, order: int) -> torch.Tensor:
    """masks [n_img, M, IH, IW] (fp32 or bf16) -> normalised bf16 pooling weights [n_img, M, side*side]."""
    if not masks.is_cuda or masks.dim() != 4 or not masks.is_contiguous():
        raise SrgptError("mask_weights: expected a contiguous CUDA tensor [n_img, M, IH, IW]")
    if masks.dtype not in (torch.float32, ELEM()):
        raise SrgptError(f"mask_weights: unsupported dtype {masks.dtype}")
    n, M, IH, IW = masks.shape
    # base_extractor.py:53-57: scale_factor = (L / (IH*IW)) ** 0.5 in Python doubles; ATen then uses
    # static_cast<float>(1.0 / scale_factor) as the source-index scale.
    scale_factor = ((side * side) / (IH * IW)) ** 0.5
    if int(IH * scale_factor) != side or int(IW * scale_factor) != side:
        raise SrgptError(f"mask_weights: floor({IH}x{IW} * {scale_factor}) != {side} (non-square masks are unsupported)")
    rscale = float(torch.tensor(1.0 / scale_factor, dtype=torch.float64).to(torch.float32))
    lib = _lib.load()
    L = side * side
    ld = (L + 7) // 8 * 8  # rows padded to 16 bytes (include/srgpt_b200.h); the returned view hides the pad
    w = torch.empty((n, M, ld), dtype=ELEM(), device=masks.device)[:, :, :L]
    ws = torch.empty(lib.srgpt_mask_weights_workspace(n, M, side), dtype=torch.uint8, device=masks.device)
    check(lib.srgpt_mask_weights(_p(masks), 1 if masks.dtype == ELEM() else 0, _p(w), _p(ws), n, M, IH, IW, side, rscale, order,
                                 _stream()), "srgpt_mask_weights")
    return w


def mask_pool(x: torch.Tensor, w: torch.Tensor, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [n_img, L, C] bf16, w [n_img, M, L] bf16 -> [n_img, M, C] bf16."""
    _need(x, ELEM(), "mask_pool.x"); _need(w, ELEM(), "mask_pool.w")
    if x.dim() != 3 or w.dim() != 3 or not x.is_contiguous():
        raise SrgptError("mask_pool: expected contiguous x [n, L, C] and w [n, M, L]")
    n, L, Cc = x.shape
    n2, M, L2 = w.shape
    ld = (L2 + 7) // 8 * 8
    if w.stride(2) != 1 or w.stride(1) != ld or w.stride(0) != M * ld:
        raise SrgptError("mask_pool: w must be the [n, M, L] view of a [n, M, round_up(L, 8)] buffer (what mask_weights returns)")
    if n != n2 or L != L2:
        raise SrgptError("mask_pool: shape mismatch between x and w")
    need = _lib.load().srgpt_mask_pool_workspace(n, M, L, Cc)
    if workspace is None or workspace.numel() * workspace.element_size() < need:
        workspace = torch.empty((need + 3) // 4, dtype=torch.float32, device=x.device)
    out = torch.empty((n, M, Cc), dtype=ELEM(), device=x.device)
    check(_lib.load().srgpt_mask_pool_bf16(_p(x), _p(w), _p(out), _p(workspace), n, M, L, Cc, _stream()), "srgpt_mask_pool_bf16")
    return out


def adaptive_avgpool(x: torch.Tensor, side: int, out_side: int, order: int) -> torch.Tensor:
    _need(x, ELEM(), "adaptive_avgpool.x")
    n, L, Cc = x.shape
    if L != side * side or not x.is_contiguous():
        raise SrgptError("adaptive_avgpool: expected contiguous [n, side*side, C]")
    y = torch.empty((n, out_side * out_side, Cc), dtype=ELEM(), device=x.device)
    check(_lib.load().srgpt_adaptive_avgpool_bf16(_p(x), _p(y), n, side, out_side, Cc, order, _stream()),
          "srgpt_adaptive_avgpool_bf16")
    return y


def reorder_rows(x: torch.Tensor, side: int, from_order: int, to_order: int) -> torch.Tensor:
    _need(x, ELEM(), "reorder_rows.x")
    n, L, Cc = x.shape
    if L != side * side or not x.is_contiguous():
        raise SrgptError("reorder_rows: expected contiguous [n, side*side, C]")
    y = torch.empty_like(x)
    check(_lib.load().srgpt_reorder_rows_bf16(_p(x), _p(y), n, side, Cc, from_order, to_order, _stream()), "srgpt_reorder_rows_bf16")
    return y


def depth_to_u8x3(depth: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """depth [h, w] or [1, h, w] fp32 -> [H, W, 3] uint8 (eval_spatial.py:99-105)."""
    _need(depth, torch.float32, "depth_to_u8x3.depth")
    d = depth.reshape(depth.shape[-2], depth.shape[-1]).contiguous()
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=depth.device)
    ws = torch.empty(H * W + 2, dtype=torch.float32, device=depth.device)
    check(_lib.load().srgpt_depth_to_u8x3(_p(d), d.shape[0], d.shape[1], _p(out), H, W, _p(ws), _stream()), "srgpt_depth_to_u8x3")
    return out


# ------------------------------------------------------------------------------------------------
def attention_prefill(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int, seqlen: int, n_heads: int,
                      n_kv_heads: int, head_dim: int, scale: float, causal: bool,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v: 2-D row-major views [batch*seqlen, heads*head_dim] (may be column slices of a fused qkv buffer)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _need(t, ELEM(), f"attention_prefill.{nm}")
    q_ld, k_ld, v_ld = _rowmajor2d(q, "q"), _rowmajor2d(k, "k"), _rowmajor2d(v, "v")
    if k_ld != v_ld:
        raise SrgptError("attention_prefill: k and v must share a row stride")
    if out is None:
        out = torch.empty((batch * seqlen, n_heads * head_dim), dtype=ELEM(), device=q.device)
    check(_lib.load().srgpt_attention_prefill_bf16(_p(q), _p(k), _p(v), _p(out), q_ld, k_ld, _rowmajor2d(out, "out"), batch,
                                                   seqlen, n_heads, n_kv_heads, head_dim, scale, 1 if causal else 0, _stream()),
          "srgpt_attention_prefill_bf16")
    return out


def attention_prefill_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int,
                             n_heads: int, n_kv_heads: int, head_dim: int, scale: float, causal: bool) -> torch.Tensor:
    """Packed sequences: rows [cu_seqlens[b], cu_seqlens[b+1]) belong to sequence b (modeling_llama.py:540-562)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _need(t, ELEM(), f"attention_prefill_varlen.{nm}")
    _need(cu_seqlens, torch.int32, "attention_prefill_varlen.cu_seqlens")
    q_ld, k_ld, v_ld = _rowmajor2d(q, "q"), _rowmajor2d(k, "k"), _rowmajor2d(v, "v")
    if k_ld != v_ld:
        raise SrgptError("attention_prefill_varlen: k and v must share a row stride")
    out = torch.empty((q.shape[0], n_heads * head_dim), dtype=ELEM(), device=q.device)
    check(_lib.load().srgpt_attention_prefill_varlen_bf16(_p(q), _p(k), _p(v), _p(out), q_ld, k_ld, _rowmajor2d(out, "out"),
                                                          cu_seqlens.numel() - 1, _p(cu_seqlens), max_seqlen, q.shape[0], n_heads, n_kv_heads,
                                                          head_dim, scale, 1 if causal else 0, _stream()),
          "srgpt_attention_prefill_varlen_bf16")
    return out


def rope_kv_append_varlen(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, cos_tab: torch.Tensor, sin_tab: torch.Tensor,
                          start_pos: torch.Tensor, kv_pages: torch.Tensor, page_tables: torch.Tensor, page_size: int,
                          cu_seqlens: torch.Tensor) -> None:
    _need(qkv, ELEM(), "rope_kv_append_varlen.qkv")
    if not qkv.is_contiguous() or qkv.shape[1] != (n_heads + 2 * n_kv_heads) * head_dim:
        raise SrgptError("rope_kv_append_varlen: qkv must be contiguous [rows, (nh + 2 nkv) * hd]")
    for t, nm in ((start_pos, "start_pos"), (page_tables, "page_tables"), (cu_seqlens, "cu_seqlens")):
        _need(t, torch.int32, f"rope_kv_append_varlen.{nm}")
    n_seqs = cu_seqlens.numel() - 1
    if page_tables.dim() != 2 or page_tables.shape[0] < n_seqs or page_tables.stride(1) != 1 or start_pos.numel() < n_seqs:
        raise SrgptError("rope_kv_append_varlen: page_tables [n_seqs, cap] / start_pos [n_seqs] expected")
    check(_lib.load().srgpt_rope_kv_append_varlen_bf16(_p(qkv), qkv.shape[0], n_heads, n_kv_heads, head_dim, _p(cos_tab), _p(sin_tab),
                                                       _p(start_pos), _p(kv_pages), _p(page_tables), page_tables.stride(0), page_size,
                                                       n_seqs, _p(cu_seqlens), _stream()), "srgpt_rope_kv_append_varlen_bf16")


def rope_kv_append(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, cos_tab: torch.Tensor,
                   sin_tab: torch.Tensor, start_pos: torch.Tensor, kv_pages: torch.Tensor, page_table: torch.Tensor,
                   page_size: int) -> None:
    _need(qkv, ELEM(), "rope_kv_append.qkv")
    if not qkv.is_contiguous() or qkv.shape[1] != (n_heads + 2 * n_kv_heads) * head_dim:
        raise SrgptError("rope_kv_append: qkv must be contiguous [rows, (nh + 2 nkv) * hd]")
    _need(start_pos, torch.int32, "rope_kv_append.start_pos"); _need(page_table, torch.int32, "rope_kv_append.page_table")
    check(_lib.load().srgpt_rope_kv_append_bf16(_p(qkv), qkv.shape[0], n_heads, n_kv_heads, head_dim, _p(cos_tab), _p(sin_tab),
                                                _p(start_pos), _p(kv_pages), _p(page_table), page_size, _stream()),
          "srgpt_rope_kv_append_bf16")


def attention_prefill_paged(q: torch.Tensor, kv_pages: torch.Tensor, page_tables: torch.Tensor, page_size: int, start_pos: torch.Tensor,
                            cu_seqlens: torch.Tensor, max_rows: int, n_heads: int, n_kv_heads: int, head_dim: int, scale: float,
                            out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Chunked prefill attention: q [rows, >= n_heads*hd] (row-strided view, e.g. the q columns of a fused qkv buffer) of n_seqs
    chunks packed by cu_seqlens [n_seqs+1]; chunk b continues sequence b at start_pos[b] and attends causally over its pages
    (kv_pages = one layer [n_pages, 2, page_size, nkv, hd], page_tables [>= n_seqs, cap])."""
    _need(q, ELEM(), "attention_prefill_paged.q"); _need(kv_pages, ELEM(), "attention_prefill_paged.kv_pages")
    for t, nm in ((page_tables, "page_tables"), (start_pos, "start_pos"), (cu_seqlens, "cu_seqlens")):
        _need(t, torch.int32, f"attention_prefill_paged.{nm}")
    n_seqs = cu_seqlens.numel() - 1
    if page_tables.dim() != 2 or page_tables.shape[0] < n_seqs or page_tables.stride(1) != 1 or start_pos.numel() < n_seqs:
        raise SrgptError("attention_prefill_paged: page_tables [n_seqs, cap] / start_pos [n_seqs] expected")
    if not kv_pages.is_contiguous():
        raise SrgptError("attention_prefill_paged: kv_pages must be contiguous [n_pages, 2, page_size, nkv, hd]")
    if out is None:
        out = torch.empty((q.shape[0], n_heads * head_dim), dtype=ELEM(), device=q.device)
    check(_lib.load().srgpt_attention_prefill_paged_bf16(_p(q), _rowmajor2d(q, "q"), _p(out), _rowmajor2d(out, "out"), _p(kv_pages), kv_pages.shape[0],
                                                         _p(page_tables), page_tables.stride(0), page_size, _p(start_pos), _p(cu_seqlens), n_seqs,
                                                         max_rows, q.shape[0], n_heads, n_kv_heads, head_dim, scale, _stream()),
          "srgpt_attention_prefill_paged_bf16")
    return out


def rows_equal(a: torch.Tensor, b: torch.Tensor, flags: torch.Tensor) -> torch.Tensor:
    """flags[r] (int32, device) = 1 when a[r] and b[r] are bitwise equal; a, b contiguous CUDA tensors of one shape and dtype."""
    if not (a.is_cuda and b.is_cuda and a.is_contiguous() and b.is_contiguous()) or a.shape != b.shape or a.dtype != b.dtype or a.dim() < 1:
        raise SrgptError("rows_equal: expected two contiguous CUDA tensors of the same shape and dtype")
    _need(flags, torch.int32, "rows_equal.flags")
    rows = a.shape[0]
    if flags.numel() < rows or not flags.is_contiguous():
        raise SrgptError("rows_equal: flags must be a contiguous int32 vector of at least one entry per row")
    check(_lib.load().srgpt_rows_equal(_p(a), _p(b), rows, a[0].numel() * a.element_size(), _p(flags), _stream()), "srgpt_rows_equal")
    return flags


def attention_decode(q: torch.Tensor, out: torch.Tensor, kv_pages: torch.Tensor, page_table: torch.Tensor, page_size: int,
                     pos: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, scale: float) -> torch.Tensor:
    check(_lib.load().srgpt_attention_decode_bf16(_p(q), _p(out), _p(kv_pages), _p(page_table), page_size, _p(pos), n_heads,
                                                  n_kv_heads, head_dim, scale, _stream()), "srgpt_attention_decode_bf16")
    return out


def gemv(x: torch.Tensor, w: torch.Tensor, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
         residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0,
         head_dim: int = 0, cos_tab=None, sin_tab=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0) -> torch.Tensor:
    N, K = w.shape
    check(_lib.load().srgpt_gemv_bf16(_p(x), _p(w), w.stride(0), _p(y), N, K, _p(norm_weight), eps, _p(residual), mode, n_heads,
                                      n_kv_heads, head_dim, _p(cos_tab), _p(sin_tab), _p(pos), _p(kv_pages), _p(page_table),
                                      page_size, _stream()), "srgpt_gemv_bf16")
    return y


# ---- 12-bit lossless packing of decode weights (pack12.cu; DESIGN.md §3) -------------------------------------------
PACK12_BATCH = 1024          # K must be a multiple: one 4-chunk step of a warp's 32 lanes
PACK12_MAX_EXC_RATE = 0.01   # a matrix with more exceptions than this stays plain bf16
PACK12_MAX_EXC_PER_ROW = 32  # the GEMV holds a row's exception list in one register per lane


def _packed_desc(p) -> "_lib.Packed12":
    d = _lib.Packed12()
    if p is not None:
        d.sm, d.ex, d.base, d.row_ptr, d.exc = (t.data_ptr() for t in (p.sm, p.ex, p.base, p.row_ptr, p.exc))
    return d


def pack12(w: torch.Tensor, verify: bool = True):
    """Pack a bf16 matrix [N, K] for the decode GEMV.  Returns (Packed12W, None), or (None, reason) when the matrix must stay
    plain: K not a multiple of 1024, Inf / NaN, more than 1 % exceptions or more than 32 in one row.  With ``verify`` the packed
    matrix is unpacked on the device and compared bit for bit with ``w``; a difference raises SrgptError."""
    _need(w, torch.bfloat16, "pack12.w")
    ldw = _rowmajor2d(w, "pack12.w")
    N, K = w.shape
    if K % PACK12_BATCH:
        return None, f"K = {K} is not a multiple of {PACK12_BATCH}"
    dev, lib = w.device, _lib.load()
    base = torch.empty(N, dtype=torch.uint8, device=dev)
    n_exc = torch.empty(N, dtype=torch.int32, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.srgpt_pack12_scan_bf16(_p(w), ldw, N, K, _p(base), _p(n_exc), _p(n_bad), _stream()), "srgpt_pack12_scan_bf16")
    total, worst, bad = (int(v) for v in torch.stack([n_exc.sum(), n_exc.max(), n_bad[0]]).cpu())
    if bad:
        return None, f"{bad} rows hold Inf or NaN"
    if total > PACK12_MAX_EXC_RATE * N * K:
        return None, f"{total / (N * K):.2%} of the weights are exceptions"
    if worst > PACK12_MAX_EXC_PER_ROW:
        return None, f"a row has {worst} exceptions"
    row_ptr = torch.zeros(N + 1, dtype=torch.int32, device=dev)
    row_ptr[1:] = torch.cumsum(n_exc, 0, dtype=torch.int32)
    p = Packed12W(sm=torch.empty((N, K), dtype=torch.uint8, device=dev), ex=torch.empty((N, K // 2), dtype=torch.uint8, device=dev), base=base,
                  row_ptr=row_ptr, exc=torch.empty(max(total, 1), dtype=torch.int32, device=dev))
    check(lib.srgpt_pack12_bf16(_p(w), ldw, N, K, _p(base), _p(row_ptr), _p(p.sm), _p(p.ex), _p(p.exc), _stream()), "srgpt_pack12_bf16")
    if verify:
        verify12(p, w)
    return p, None


def verify12(p, w: torch.Tensor) -> None:
    """Raises SrgptError unless the Packed12W ``p`` unpacks to exactly the bits of ``w``."""
    if not torch.equal(unpack12(p).view(torch.int16), w.view(torch.int16)):
        raise SrgptError(f"pack12: the packed {list(w.shape)} matrix does not unpack to the original bits")


def unpack12(p) -> torch.Tensor:
    """The bf16 matrix [N, K] a Packed12W holds (through the GEMV's own decoder)."""
    N, K = p.sm.shape
    out = torch.empty((N, K), dtype=torch.bfloat16, device=p.sm.device)
    d = _packed_desc(p)
    check(_lib.load().srgpt_unpack12_bf16(C.byref(d), N, K, _p(out), K, _stream()), "srgpt_unpack12_bf16")
    return out


def gemv_packed(x: torch.Tensor, p, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
                residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0,
                head_dim: int = 0, cos_tab=None, sin_tab=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0) -> torch.Tensor:
    """gemv() over a Packed12W: bit-identical results, 12 instead of 16 bits of weight stream per element."""
    N, K = p.sm.shape
    d = _packed_desc(p)
    check(_lib.load().srgpt_gemv_packed_bf16(_p(x), C.byref(d), _p(y), N, K, _p(norm_weight), eps, _p(residual), mode, n_heads, n_kv_heads,
                                             head_dim, _p(cos_tab), _p(sin_tab), _p(pos), _p(kv_pages), _p(page_table), page_size, _stream()),
          "srgpt_gemv_packed_bf16")
    return y


# ---- NF4 weight-only quantization of the decoder-layer matrices (nf4.cu; DESIGN.md §3) ------------------------------
NF4_BLOCK = 64     # weights per scale; a matrix's in_features must be a multiple
NF4_BATCH = 1024   # K must be a multiple for the decode GEMV's lane-ordered planes
_NF4_MAPS = {}


def nf4_dynamic_map(device) -> torch.Tensor:
    """The 256 fp32 values of bitsandbytes' create_dynamic_map(signed=True), the second-level code of double quantization: for
    i = 0..6, +-10^(i-6) times the midpoints of linspace(0.1, 1, 2^i + 1), plus 0 and 1, sorted.  The linspace points are
    fl32(0.1 + 0.9 j / (n - 1)) computed in fp64, the midpoints and products in fp32."""
    key = str(device)
    if key not in _NF4_MAPS:
        import numpy as np
        vals = []
        for i in range(7):
            n = 2 ** i + 1
            b = np.array([0.1 + 0.9 * j / (n - 1) for j in range(n)], dtype=np.float32)
            means = (b[:-1] + b[1:]) * np.float32(0.5)
            s = np.float32(10.0 ** (i - 6))
            vals += list(s * means) + list(-(s * means))
        vals += [np.float32(0.0), np.float32(1.0)]
        _NF4_MAPS[key] = torch.from_numpy(np.sort(np.array(vals, dtype=np.float32))).to(device)
    return _NF4_MAPS[key]


def nf4_quantize(w: torch.Tensor):
    """NF4 codes of an element-type matrix [N, K] (K a multiple of 64): (codes [N, K/2] uint8 in natural order, scale [N, K/64]
    fp32 resolved scales).  Raises NotImplementedError for K % 64 != 0 and SrgptError when w holds Inf or NaN."""
    _need(w, ELEM(), "nf4_quantize.w")
    ldw = _rowmajor2d(w, "nf4_quantize.w")
    N, K = w.shape
    if K % NF4_BLOCK:
        raise NotImplementedError(f"NF4 quantization needs in_features to be a multiple of {NF4_BLOCK}, got {K}")
    dev, lib = w.device, _lib.load()
    codes = torch.empty((N, K // 2), dtype=torch.uint8, device=dev)
    absmax = torch.empty((N, K // NF4_BLOCK), dtype=torch.float32, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int32, device=dev)
    check(lib.srgpt_nf4_quantize_bf16(_p(w), ldw, N, K, _p(codes), _p(absmax), _p(n_bad), _stream()), "srgpt_nf4_quantize_bf16")
    if int(n_bad[0]):
        raise SrgptError(f"nf4_quantize: the {list(w.shape)} matrix holds Inf or NaN in {int(n_bad[0])} blocks of {NF4_BLOCK}")
    offset = torch.empty(1, dtype=torch.float32, device=dev)
    scale = torch.empty_like(absmax)
    check(lib.srgpt_nf4_double_quant(_p(absmax), absmax.numel(), _p(nf4_dynamic_map(dev)), _p(offset), _p(scale), _stream()),
          "srgpt_nf4_double_quant")
    return codes, scale


def nf4_dequantize(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """The element-type matrix [N, K] of natural-order codes and scales: round_to_elem(fl32(code_value * scale))."""
    N, K = codes.shape[0], codes.shape[1] * 2
    out = torch.empty((N, K), dtype=ELEM(), device=codes.device)
    check(_lib.load().srgpt_nf4_dequantize_bf16(_p(codes), _p(scale), N, K, _p(out), K, _stream()), "srgpt_nf4_dequantize_bf16")
    return out


def _nf4_desc(p) -> "_lib.Nf4":
    d = _lib.Nf4()
    if p is not None:
        d.q, d.scale = p.q.data_ptr(), p.scale.data_ptr()
    return d


def nf4_planes(codes: torch.Tensor, scale: torch.Tensor, deq: torch.Tensor):
    """The decode GEMV's planes of a (fused) matrix: (Nf4W, None), or (None, reason) when K is not a multiple of 1024 and the decode
    step reads the dequantized matrix instead.  The lane-ordered planes must dequantize to exactly ``deq``; SrgptError otherwise."""
    N, K = codes.shape[0], codes.shape[1] * 2
    if K % NF4_BATCH:
        return None, f"K = {K} is not a multiple of {NF4_BATCH}"
    q = torch.empty_like(codes)
    check(_lib.load().srgpt_nf4_lane_order(_p(codes), N, K, _p(q), _stream()), "srgpt_nf4_lane_order")
    p = Nf4W(q=q, scale=scale.contiguous())
    if not torch.equal(nf4_unpack(p).view(torch.int16), deq.view(torch.int16)):
        raise SrgptError(f"nf4: the lane-ordered planes of the {list(deq.shape)} matrix do not dequantize to its resident copy")
    return p, None


def nf4_unpack(p) -> torch.Tensor:
    """The element-type matrix [N, K] an Nf4W's lane-ordered planes hold (through the GEMV's own dequantization)."""
    N, K = p.q.shape[0], p.q.shape[1] * 2
    out = torch.empty((N, K), dtype=ELEM(), device=p.q.device)
    d = _nf4_desc(p)
    check(_lib.load().srgpt_nf4_unpack_bf16(C.byref(d), N, K, _p(out), K, _stream()), "srgpt_nf4_unpack_bf16")
    return out


def gemv_nf4(x: torch.Tensor, p, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
             residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0,
             head_dim: int = 0, cos_tab=None, sin_tab=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0) -> torch.Tensor:
    """gemv() over an Nf4W: bit-identical to gemv() over the dequantized matrix, 4.5 bits of weight stream per element."""
    N, K = p.q.shape[0], p.q.shape[1] * 2
    d = _nf4_desc(p)
    check(_lib.load().srgpt_gemv_nf4_bf16(_p(x), C.byref(d), _p(y), N, K, _p(norm_weight), eps, _p(residual), mode, n_heads, n_kv_heads,
                                          head_dim, _p(cos_tab), _p(sin_tab), _p(pos), _p(kv_pages), _p(page_table), page_size, _stream()),
          "srgpt_gemv_nf4_bf16")
    return y


def gemm_nf4(a: torch.Tensor, w, residual: Optional[torch.Tensor] = None, epilogue: int = EPI_NONE,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemm() with the weight [N, K] read from an Nf4W's planes (K a multiple of 1024; epilogue EPI_NONE, EPI_BIAS_RESIDUAL without bias
    or EPI_SWIGLU): the producer warpgroup dequantizes each weight tile in shared memory, so no element-type copy of the matrix is read
    or kept.  Bit-identical to gemm() over the dequantized matrix."""
    _need(a, ELEM(), "gemm_nf4.a")
    _ensure_gemm_workspace(a.device)
    lda = _rowmajor2d(a, "gemm_nf4.a")
    M, K = a.shape
    N, K2 = w.q.shape[0], w.q.shape[1] * 2
    if K != K2:
        raise SrgptError(f"gemm_nf4: K mismatch {K} vs {K2}")
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=ELEM(), device=a.device)
    _need(out, ELEM(), "gemm_nf4.out")
    if out.shape != (M, n_out):
        raise SrgptError(f"gemm_nf4.out: expected {(M, n_out)}, got {tuple(out.shape)}")
    ldr = 0
    if residual is not None:
        _need(residual, ELEM(), "gemm_nf4.residual")
        ldr = _rowmajor2d(residual, "gemm_nf4.residual")
    d = _nf4_desc(w)
    check(_lib.load().srgpt_gemm_nf4_bf16(_p(a), lda, C.byref(d), _p(out), _rowmajor2d(out, "gemm_nf4.out"), M, N, K, _p(residual), ldr, epilogue,
                                          _stream()), "srgpt_gemm_nf4_bf16")
    return out


# ---- FP8 (E4M3) W8A8 quantization of the decoder-layer linears (fp8.cu, gemm_wgmma.cu; DESIGN.md §3) ------------------------------
FP8_K_MULTIPLE = 16  # in_features must be a multiple (16-byte rows for TMA)


def fp8_quantize_weight(w: torch.Tensor, name: str = "matrix"):
    """Per-row E4M3 codes of an element-type matrix [N, K]: (q [N, K] uint8, scale [N] fp32), include/srgpt_b200.h's definition.  Raises
    NotImplementedError for K % 16 != 0 and SrgptError when w holds Inf or NaN; `name` names the matrix in both."""
    N, K = w.shape
    if K % FP8_K_MULTIPLE:
        raise NotImplementedError(f"FP8 quantization needs in_features to be a multiple of {FP8_K_MULTIPLE}; {name} has {K}")
    _need(w, ELEM(), "fp8_quantize_weight.w")
    ldw = _rowmajor2d(w, "fp8_quantize_weight.w")
    q = torch.empty((N, K), dtype=torch.uint8, device=w.device)
    scale = torch.empty(N, dtype=torch.float32, device=w.device)
    n_bad = torch.zeros(1, dtype=torch.int32, device=w.device)
    check(_lib.load().srgpt_fp8_quantize_weight_bf16(_p(w), ldw, N, K, _p(q), _p(scale), _p(n_bad), _stream()), "srgpt_fp8_quantize_weight_bf16")
    if int(n_bad[0]):
        raise SrgptError(f"fp8_quantize_weight: {name} {list(w.shape)} holds Inf or NaN in {int(n_bad[0])} rows")
    return q, scale


def fp8_quantize_act(x: torch.Tensor, q: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None):
    """The activation quantizer: per-row E4M3 codes of x [M, K] -> (q [M, K] uint8, scale [M] fp32), the weights' definition."""
    _need(x, ELEM(), "fp8_quantize_act.x")
    ldx = _rowmajor2d(x, "fp8_quantize_act.x")
    M, K = x.shape
    q = torch.empty((M, K), dtype=torch.uint8, device=x.device) if q is None else q
    scale = torch.empty(M, dtype=torch.float32, device=x.device) if scale is None else scale
    _need(q, torch.uint8, "fp8_quantize_act.q"); _need(scale, torch.float32, "fp8_quantize_act.scale")
    if q.shape != (M, K) or scale.numel() < M:
        raise SrgptError(f"fp8_quantize_act: q {tuple(q.shape)} / scale {tuple(scale.shape)} do not fit x {(M, K)}")
    check(_lib.load().srgpt_fp8_quantize_act_bf16(_p(x), ldx, M, K, _p(q), _rowmajor2d(q, "fp8_quantize_act.q"), _p(scale), _stream()),
          "srgpt_fp8_quantize_act_bf16")
    return q, scale


def gemm_fp8(q: torch.Tensor, sx: torch.Tensor, w, residual: Optional[torch.Tensor] = None, epilogue: int = EPI_NONE,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M, N] = epilogue(acc * (sx[m] * w.scale[n])) with acc = q [M, K] · w.q [N, K]^T over E4M3 codes (an Fp8W), on the FP8 tensor
    cores.  Epilogues: EPI_NONE, EPI_BIAS_RESIDUAL (no bias), EPI_SWIGLU."""
    _need(q, torch.uint8, "gemm_fp8.q"); _need(sx, torch.float32, "gemm_fp8.sx")
    _ensure_gemm_workspace(q.device)
    lda, ldw = _rowmajor2d(q, "gemm_fp8.q"), _rowmajor2d(w.q, "gemm_fp8.w")
    M, K = q.shape
    N, K2 = w.q.shape
    if K != K2:
        raise SrgptError(f"gemm_fp8: K mismatch {K} vs {K2}")
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=ELEM(), device=q.device)
    _need(out, ELEM(), "gemm_fp8.out")
    if out.shape != (M, n_out):
        raise SrgptError(f"gemm_fp8.out: expected {(M, n_out)}, got {tuple(out.shape)}")
    ldr = 0
    if residual is not None:
        _need(residual, ELEM(), "gemm_fp8.residual")
        ldr = _rowmajor2d(residual, "gemm_fp8.residual")
    check(_lib.load().srgpt_gemm_fp8_bf16(_p(q), lda, _p(sx), _p(w.q), ldw, _p(w.scale), _p(out), _rowmajor2d(out, "gemm_fp8.out"), M, N, K,
                                          _p(residual), ldr, epilogue, _stream()), "srgpt_gemm_fp8_bf16")
    return out


def linear_fp8(x: torch.Tensor, w, residual: Optional[torch.Tensor] = None, epilogue: int = EPI_NONE, out: Optional[torch.Tensor] = None,
               q: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A W8A8 linear over the element-type activation x [M, K]: the activation quantizer (into q / scale when given), then gemm_fp8."""
    q, scale = fp8_quantize_act(x, q, scale)
    return gemm_fp8(q, scale, w, residual=residual, epilogue=epilogue, out=out)


def gemv_fp8(x: torch.Tensor, w, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
             residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0,
             head_dim: int = 0, cos_tab=None, sin_tab=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0) -> torch.Tensor:
    """gemv() over an Fp8W: x (RMS-normalised first with norm_weight) quantized in the kernel by the activation definition, the W8A8
    linear of fp8_quantize_act + gemm_fp8 at M = 1 with the one-token GEMV's modes and rounding points; 1 byte of weight stream per element."""
    _need(x, ELEM(), "gemv_fp8.x"); _need(y, ELEM(), "gemv_fp8.y")
    N, K = w.q.shape
    d = _fp8_desc(w)
    check(_lib.load().srgpt_gemv_fp8_bf16(_p(x), C.byref(d), _p(y), N, K, _p(norm_weight), eps, _p(residual), mode, n_heads, n_kv_heads, head_dim,
                                          _p(cos_tab), _p(sin_tab), _p(pos), _p(kv_pages), _p(page_table), page_size, _stream()),
          "srgpt_gemv_fp8_bf16")
    return y


def _fp8_desc(p) -> "_lib.Fp8":
    d = _lib.Fp8()
    d.q, d.scale = p.q.data_ptr(), p.scale.data_ptr()
    return d


# ---- host preprocessing on the GPU (preprocess.py) ---------------------------------------------------------------
def resample_u8(img: torch.Tensor, axis: int, out_size: int, kk: torch.Tensor, bounds: torch.Tensor, ksize: int) -> torch.Tensor:
    _need(img, torch.uint8, "resample_u8.img"); _need(kk, torch.int32, "resample_u8.kk"); _need(bounds, torch.int32, "resample_u8.bounds")
    H, W, Cc = img.shape
    out = torch.empty((out_size, W, Cc) if axis == 0 else (H, out_size, Cc), dtype=torch.uint8, device=img.device)
    check(_lib.load().srgpt_resample_u8(_p(img), _p(out), H, W, Cc, axis, out_size, _p(kk), _p(bounds), ksize, _stream()), "srgpt_resample_u8")
    return out


def u8_to_normalized_chw(img: torch.Tensor, scale: float, mean, std, do_normalize: bool = True) -> torch.Tensor:
    import ctypes
    _need(img, torch.uint8, "u8_to_normalized_chw.img")
    H, W, Cc = img.shape
    out = torch.empty((Cc, H, W), dtype=torch.float32, device=img.device)
    m3 = (ctypes.c_float * 3)(*([float(v) for v in mean] + [0.0] * 3)[:3])
    s3 = (ctypes.c_float * 3)(*([float(v) for v in std] + [1.0] * 3)[:3])
    check(_lib.load().srgpt_u8_to_normalized_chw(_p(img), _p(out), H, W, Cc, float(scale), m3, s3, 1 if do_normalize else 0, _stream()),
          "srgpt_u8_to_normalized_chw")
    return out


def resize_nearest_u8(img: torch.Tensor, out_h: int, out_w: int, ys: torch.Tensor, xs: torch.Tensor) -> torch.Tensor:
    _need(img, torch.uint8, "resize_nearest_u8.img"); _need(ys, torch.int32, "resize_nearest_u8.ys"); _need(xs, torch.int32, "resize_nearest_u8.xs")
    H, W = img.shape
    out = torch.empty((out_h, out_w), dtype=torch.float32, device=img.device)
    check(_lib.load().srgpt_resize_nearest_u8(_p(img), _p(out), H, W, out_h, out_w, _p(ys), _p(xs), _stream()), "srgpt_resize_nearest_u8")
    return out


# ---- batched decode ----------------------------------------------------------------------------------------------
def attention_decode_batched(q: torch.Tensor, out: torch.Tensor, kv_pages: torch.Tensor, page_tables: torch.Tensor, page_size: int, pos: torch.Tensor,
                             n_heads: int, n_kv_heads: int, head_dim: int, scale: float) -> torch.Tensor:
    """q [B, >= n_heads*hd] (row-strided view, e.g. the q columns of a fused qkv buffer), out [B, n_heads*hd], page_tables [>= B, cap],
    pos int32 [B] = position of every sequence's newest row."""
    _need(q, ELEM(), "attention_decode_batched.q"); _need(out, ELEM(), "attention_decode_batched.out")
    _need(page_tables, torch.int32, "attention_decode_batched.page_tables"); _need(pos, torch.int32, "attention_decode_batched.pos")
    B = q.shape[0]
    check(_lib.load().srgpt_attention_decode_batched_bf16(_p(q), _rowmajor2d(q, "q"), _p(out), _rowmajor2d(out, "out"), _p(kv_pages), _p(page_tables),
                                                          page_tables.stride(0), page_size, _p(pos), B, n_heads, n_kv_heads, head_dim, scale, _stream()),
          "srgpt_attention_decode_batched_bf16")
    return out


def decode_batch_advance(ids: torch.Tensor, embed_table: torch.Tensor, h: torch.Tensor, out_ids: torch.Tensor, step: torch.Tensor, pos: torch.Tensor,
                         ticket: torch.Tensor) -> None:
    _need(ids, torch.int64, "decode_batch_advance.ids"); _need(out_ids, torch.int64, "decode_batch_advance.out_ids")
    B, H = h.shape
    check(_lib.load().srgpt_decode_batch_advance(_p(ids), _p(embed_table), _p(h), H, _p(out_ids), _p(step), _p(pos), B, _p(ticket), _stream()),
          "srgpt_decode_batch_advance")


# ---- tensor-parallel decode (one rank's share) ---------------------------------------------------------------------
def gemv_tp_qkv(x, w_local, y_local, norm_weight, eps: float, n_heads_local: int, n_kv_local: int, head_dim: int, cos_tab, sin_tab, pos,
                kv_pages, page_table, page_size: int, kv_heads_total: int, kv_head_off: int) -> torch.Tensor:
    """RMSNorm + this rank's q/k/v rows + RoPE; K/V rows are appended to the full-layout cache at kv head `kv_head_off`."""
    N, K = w_local.shape
    check(_lib.load().srgpt_gemv_tp_bf16(_p(x), _p(w_local), w_local.stride(0), _p(y_local), N, K, _p(norm_weight), eps, GEMV_QKV_ROPE, n_heads_local,
                                         n_kv_local, head_dim, _p(cos_tab), _p(sin_tab), _p(pos), _p(kv_pages), _p(page_table), page_size,
                                         kv_heads_total, kv_head_off, None, _stream()), "srgpt_gemv_tp_bf16")
    return y_local


def gemv_tp_partial(x_local, w_local, partial_f32) -> torch.Tensor:
    """Row-parallel linear: fp32 partial sums over this rank's K slice (all-reduced by the caller)."""
    N, K = w_local.shape
    _need(partial_f32, torch.float32, "gemv_tp_partial.partial")
    check(_lib.load().srgpt_gemv_tp_bf16(_p(x_local), _p(w_local), w_local.stride(0), None, N, K, None, 0.0, GEMV_PLAIN, 0, 0, 0, None, None, None,
                                         None, None, 0, 0, 0, _p(partial_f32), _stream()), "srgpt_gemv_tp_bf16")
    return partial_f32


def attention_decode_tp(q_local, out_local, kv_pages, page_table, page_size: int, pos, n_heads_local: int, group: int, n_kv_total: int,
                        kv_head_off: int, head_dim: int, scale: float) -> torch.Tensor:
    check(_lib.load().srgpt_attention_decode_tp_bf16(_p(q_local), _p(out_local), _p(kv_pages), _p(page_table), page_size, _p(pos), n_heads_local, group,
                                                     n_kv_total, kv_head_off, head_dim, scale, _stream()), "srgpt_attention_decode_tp_bf16")
    return out_local


def tp_residual_add(h, partial_f32) -> None:
    check(_lib.load().srgpt_tp_residual_add_bf16(_p(h), _p(partial_f32), h.numel(), _stream()), "srgpt_tp_residual_add_bf16")


def lm_head_local_best(x, w_local, norm_weight, eps: float, workspace, index_base: int, best) -> None:
    V, K = w_local.shape
    _need(best, torch.int32, "lm_head_local_best.best")
    check(_lib.load().srgpt_lm_head_local_best_bf16(_p(x), _p(w_local), w_local.stride(0), V, K, _p(norm_weight), eps, _p(workspace), index_base, _p(best),
                                                    _stream()), "srgpt_lm_head_local_best_bf16")


def tp_pick_token(best_all, world: int, embed_table, next_x, out_ids, step, pos) -> None:
    _need(best_all, torch.int32, "tp_pick_token.best_all")
    K = 0 if embed_table is None else embed_table.shape[1]
    check(_lib.load().srgpt_tp_pick_token(_p(best_all), world, _p(embed_table), _p(next_x), K, _p(out_ids), _p(step), _p(pos), _stream()),
          "srgpt_tp_pick_token")


def tp_allreduce_residual(peer_bases, rank: int, world: int, slot_off: int, idx: int, epoch, step, h) -> None:
    """All-reduce of the ranks' fp32 partial sums (slot `slot_off` of every rank's symmetric buffer) over NVLink peer memory, fused
    with h = bf16(bf16(sum) + h).  ``peer_bases`` = ctypes array of the peer-mapped buffer addresses."""
    check(_lib.load().srgpt_tp_allreduce_residual_bf16(peer_bases, rank, world, slot_off, idx, _p(epoch), _p(step), _p(h), h.numel(), _stream()),
          "srgpt_tp_allreduce_residual_bf16")


def tp_allgather_pick(peer_bases, rank: int, world: int, slot_off: int, idx: int, epoch, embed_table, next_x, out_ids, step, pos) -> None:
    K = 0 if embed_table is None else embed_table.shape[1]
    check(_lib.load().srgpt_tp_allgather_pick_token(peer_bases, rank, world, slot_off, idx, _p(epoch), _p(embed_table), _p(next_x), K, _p(out_ids), _p(step),
                                                    _p(pos), _stream()), "srgpt_tp_allgather_pick_token")


def lm_head_workspace(V: int, device) -> torch.Tensor:
    return torch.empty(_lib.load().srgpt_lm_head_workspace(V), dtype=torch.uint8, device=device)


def lm_head_argmax(x: torch.Tensor, w: torch.Tensor, norm_weight: Optional[torch.Tensor], eps: float, workspace: torch.Tensor,
                   out_ids: torch.Tensor, step: torch.Tensor, pos: torch.Tensor, embed_table: Optional[torch.Tensor] = None,
                   next_x: Optional[torch.Tensor] = None, logits_out: Optional[torch.Tensor] = None) -> None:
    V, K = w.shape
    check(_lib.load().srgpt_lm_head_argmax_bf16(_p(x), _p(w), w.stride(0), V, K, _p(norm_weight), eps, _p(logits_out),
                                                _p(workspace), _p(embed_table), _p(next_x), _p(out_ids), _p(step), _p(pos),
                                                _stream()), "srgpt_lm_head_argmax_bf16")


def lm_head_argmax_packed(x: torch.Tensor, p, norm_weight: Optional[torch.Tensor], eps: float, workspace: torch.Tensor,
                          out_ids: torch.Tensor, step: torch.Tensor, pos: torch.Tensor, embed_table: Optional[torch.Tensor] = None,
                          next_x: Optional[torch.Tensor] = None, logits_out: Optional[torch.Tensor] = None) -> None:
    """lm_head_argmax() over a Packed12W lm_head (bit-identical)."""
    V, K = p.sm.shape
    d = _packed_desc(p)
    check(_lib.load().srgpt_lm_head_argmax_packed_bf16(_p(x), C.byref(d), V, K, _p(norm_weight), eps, _p(logits_out), _p(workspace),
                                                       _p(embed_table), _p(next_x), _p(out_ids), _p(step), _p(pos), _stream()),
          "srgpt_lm_head_argmax_packed_bf16")


def sample_top_p(logits: torch.Tensor, params: torch.Tensor, seed, step: torch.Tensor, step_offset: int, out_ids: torch.Tensor,
                 embed_table: Optional[torch.Tensor] = None, next_x: Optional[torch.Tensor] = None, scores: Optional[torch.Tensor] = None,
                 step_stride: int = 0) -> None:
    """One token from softmax(logits / T) restricted to its top-p nucleus -> out_ids[step + step_offset] (and next_x = embed row).
    ``params`` = device float32 [temperature, top_p, top_k (0 = off)]; ``step`` = device int32 [1]; ``seed`` = device int64 [1]
    (read by the kernel at run time - graph-capturable), or a Python int for one-off eager calls.
    ``params`` of 6 floats [temperature, top_p, top_k, typical_p, epsilon_cutoff, eta_cutoff] adds HF's typical, epsilon and eta
    warpers after top-p (srgpt_sample_warped_f32; off at typical_p >= 1 and cutoffs outside (0, 1)).
    ``scores`` (fp32, optional): the warped row the draw picked from (logits / T where kept, -inf elsewhere) goes to
    scores.view(-1)[(step + step_offset) * step_stride:][:V]."""
    if not isinstance(seed, torch.Tensor):
        seed = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF], dtype=torch.int64, device=logits.device)
    _need(seed, torch.int64, "sample_top_p.seed")
    _need(logits, torch.float32, "sample_top_p.logits"); _need(params, torch.float32, "sample_top_p.params")
    _need(step, torch.int32, "sample_top_p.step"); _need(out_ids, torch.int64, "sample_top_p.out_ids")
    if logits.dim() != 1 or not logits.is_contiguous() or params.numel() < 3:
        raise SrgptError("sample_top_p: logits must be a contiguous fp32 vector [V] and params [temperature, top_p, top_k]")
    K = 0 if embed_table is None else embed_table.shape[1]
    if params.numel() == 6:
        return _sample_warped(logits, params, seed, step, step_offset, out_ids, embed_table, next_x, K, scores, step_stride)
    if scores is not None:
        _need(scores, torch.float32, "sample_top_p.scores")
        check(_lib.load().srgpt_sample_top_p_scores_f32(_p(logits), logits.numel(), _p(params), _p(seed), _p(step), step_offset, _p(out_ids),
                                                        _p(embed_table), _p(next_x), K, _p(scores), int(step_stride), _stream()),
              "srgpt_sample_top_p_scores_f32")
        return
    check(_lib.load().srgpt_sample_top_p_f32(_p(logits), logits.numel(), _p(params), _p(seed), _p(step), step_offset,
                                             _p(out_ids), _p(embed_table), _p(next_x), K, _stream()), "srgpt_sample_top_p_f32")


def _sample_warped(logits, params, seed, step, step_offset: int, out_ids, embed_table, next_x, K: int, scores, step_stride: int) -> None:
    if scores is not None:
        _need(scores, torch.float32, "sample_top_p.scores")
        check(_lib.load().srgpt_sample_warped_scores_f32(_p(logits), logits.numel(), _p(params), _p(seed), _p(step), step_offset, _p(out_ids),
                                                         _p(embed_table), _p(next_x), K, _p(scores), int(step_stride), _stream()),
              "srgpt_sample_warped_scores_f32")
        return
    check(_lib.load().srgpt_sample_warped_f32(_p(logits), logits.numel(), _p(params), _p(seed), _p(step), step_offset, _p(out_ids),
                                              _p(embed_table), _p(next_x), K, _stream()), "srgpt_sample_warped_f32")


def sample_rows(logits: torch.Tensor, params: torch.Tensor, seeds: torch.Tensor, step: torch.Tensor, step_offset: int,
                ids: torch.Tensor, scores: Optional[torch.Tensor] = None) -> None:
    """One token per row of ``logits`` ([R, V] fp32 or the element type, unit inner stride, e.g. the batched lm_head's rows) in one
    launch -> ids int64 [R].  Row r draws with seeds[r] (device int64 [R]) at counter step + step_offset, the token sample_top_p draws
    from that row in fp32 with that seed and counter.  ``params`` and ``step`` as for sample_top_p (6 params: srgpt_sample_rows_warped).
    ``scores`` (contiguous fp32 [T, R, V], optional): row r's warped row goes to scores[step + step_offset, r]."""
    _need(params, torch.float32, "sample_rows.params"); _need(seeds, torch.int64, "sample_rows.seeds")
    _need(step, torch.int32, "sample_rows.step"); _need(ids, torch.int64, "sample_rows.ids")
    if not logits.is_cuda:
        raise SrgptError("sample_rows.logits: expected a CUDA tensor (the sm_90a kernels have no CPU fallback)")
    f32 = logits.dtype == torch.float32
    _need(logits, torch.float32 if f32 else ELEM(), "sample_rows.logits")
    if logits.dim() != 2:
        raise SrgptError(f"sample_rows: logits must be [R, V], got shape {tuple(logits.shape)}")
    ld = _rowmajor2d(logits, "sample_rows.logits")
    R, V = logits.shape
    if params.numel() < 3 or step.numel() < 1:
        raise SrgptError("sample_rows: params must be [temperature, top_p, top_k] and step a device int32 [1]")
    if seeds.dim() != 1 or seeds.numel() != R or not seeds.is_contiguous():
        raise SrgptError(f"sample_rows: seeds must be a contiguous int64 vector of {R} entries, got shape {tuple(seeds.shape)}")
    if ids.dim() != 1 or ids.numel() != R or not ids.is_contiguous():
        raise SrgptError(f"sample_rows: ids must be a contiguous int64 vector of {R} entries, got shape {tuple(ids.shape)}")
    if scores is not None:
        _need(scores, torch.float32, "sample_rows.scores")
        if scores.dim() != 3 or scores.shape[1:] != (R, V) or not scores.is_contiguous():
            raise SrgptError(f"sample_rows: scores must be contiguous fp32 [T, {R}, {V}], got shape {tuple(scores.shape)}")
        name = "srgpt_sample_rows_warped_scores" if params.numel() == 6 else "srgpt_sample_rows_scores"
        check(getattr(_lib.load(), name)(_p(logits), int(f32), ld, R, V, _p(params), _p(seeds), _p(step), step_offset, _p(ids), _p(scores),
                                         R * V, _stream()), name)
        return
    name = "srgpt_sample_rows_warped" if params.numel() == 6 else "srgpt_sample_rows"
    check(getattr(_lib.load(), name)(_p(logits), int(f32), ld, R, V, _p(params), _p(seeds), _p(step), step_offset, _p(ids), _stream()), name)


def step_scores(rows: torch.Tensor, step: torch.Tensor, step_offset: int, scores: torch.Tensor) -> None:
    """A decode step's score rows: rows ([R, V] fp32 or the element type, unit inner stride; a 1-D row counts as one) widened to fp32
    -> scores[step + step_offset] (``scores`` a [T, R, V] fp32 view whose last dimension is contiguous, e.g. a column of a wider
    [T, B, V] buffer; ``step`` = device int32 [1], read at run time)."""
    x = rows if rows.dim() == 2 else rows.view(1, -1)
    R, V = x.shape
    f32 = x.dtype == torch.float32
    _need(x, torch.float32 if f32 else ELEM(), "step_scores.rows"); _need(step, torch.int32, "step_scores.step")
    _need(scores, torch.float32, "step_scores.scores")
    if scores.dim() != 3 or scores.shape[1:] != (R, V) or scores.stride(2) != 1:
        raise SrgptError(f"step_scores: scores must be fp32 [T, {R}, {V}] with a unit inner stride, got shape {tuple(scores.shape)}")
    check(_lib.load().srgpt_step_scores(_p(x), int(f32), _rowmajor2d(x, "step_scores.rows"), R, V, _p(step), step_offset, _p(scores),
                                        scores.stride(0), scores.stride(1), _stream()), "srgpt_step_scores")


def token_logprobs(logits: torch.Tensor, rows, targets, loss: bool = False):
    """Log-softmax of each row of ``logits`` ([R, V] in the element type, unit inner stride, e.g. the lm_head GEMM's padded rows) at
    target tokens, without an fp32 copy of the logits.  ``rows`` / ``targets``: host int sequences or CPU tensors of n pairs; target -100
    is ignored.  Returns (lse fp32 [R], logprob fp32 [n], loss): logprob[i] = float(logits[rows[i], targets[i]]) - lse[rows[i]] (0 when
    ignored); loss (a 0-dim fp32 tensor when ``loss``, else None) = the mean of -logprob over the pairs not ignored (NaN when none is).
    Out-of-range pairs raise before anything is launched."""
    _need(logits, ELEM(), "token_logprobs.logits")
    if logits.dim() != 2:
        raise SrgptError(f"token_logprobs: logits must be [rows, V], got shape {tuple(logits.shape)}")
    ld = _rowmajor2d(logits, "token_logprobs.logits")
    R, V = logits.shape
    r = torch.as_tensor(rows, dtype=torch.int32).reshape(-1).contiguous()
    t = torch.as_tensor(targets, dtype=torch.int64).reshape(-1).contiguous()
    if r.device.type != "cpu" or t.device.type != "cpu" or r.numel() != t.numel():
        raise SrgptError("token_logprobs: rows and targets must be host sequences of the same length")
    n = r.numel()
    dev = logits.device
    lse = torch.empty(R, dtype=torch.float32, device=dev)
    lp = torch.empty(n, dtype=torch.float32, device=dev)
    out = torch.empty((), dtype=torch.float32, device=dev) if loss else None
    ws = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    check(_lib.load().srgpt_token_logprobs(_p(logits), ld, R, V, _p(r) if n else None, _p(t) if n else None, n, _p(ws), ws.numel() * 8,
                                           _p(lse), _p(lp) if n else None, _p(out), _stream()), "srgpt_token_logprobs")
    if n or loss:
        _count(1)
    return lse, lp, out


def logits_process(logits: torch.Tensor, hist: Optional[torch.Tensor], hist_row_stride: int, hist_tok_stride: int, step: Optional[torch.Tensor],
                   step_offset: int, fparams: torch.Tensor, spec: torch.Tensor, out: Optional[torch.Tensor] = None,
                   ids: Optional[torch.Tensor] = None) -> None:
    """HF's repetition penalty / no-repeat n-gram / bad words / minimum length processors over the rows of ``logits`` ([rows, V] fp32 or
    the element type, unit inner stride; a 1-D fp32 row counts as one row), then the greedy choice.  Row r's history is
    ``hist.view(-1)[r * hist_row_stride + t * hist_tok_stride]`` for t < step + step_offset (``step`` = device int32 [1], or None:
    step_offset tokens).  ``fparams`` = device float32 [penalty, 1 / penalty], ``spec`` = device int32 (layout: include/srgpt_b200.h).
    Writes the processed fp32 rows to ``out`` [rows, V] and / or the arg max of each processed row to ``ids`` int64 [rows]."""
    x = logits if logits.dim() == 2 else logits.view(1, -1)
    rows, V = x.shape
    f32 = x.dtype == torch.float32
    _need(x, torch.float32 if f32 else ELEM(), "logits_process.logits")
    _need(fparams, torch.float32, "logits_process.fparams"); _need(spec, torch.int32, "logits_process.spec")
    if out is not None:
        out = out if out.dim() == 2 else out.view(1, -1)
        _need(out, torch.float32, "logits_process.out")
        if out.shape != x.shape:
            raise SrgptError(f"logits_process: out {tuple(out.shape)} does not match logits {tuple(x.shape)}")
    if ids is not None:
        _need(ids, torch.int64, "logits_process.ids")
        if ids.numel() < rows or not ids.is_contiguous():
            raise SrgptError("logits_process: ids must be a contiguous int64 vector of at least `rows` entries")
    cap = 0
    if hist is not None:
        _need(hist, torch.int64, "logits_process.hist")
        if not hist.is_contiguous():
            raise SrgptError("logits_process: hist must be contiguous")
        last = (rows - 1) * hist_row_stride  # the history of every row must lie inside hist
        cap = max(0, (hist.numel() - 1 - last) // max(hist_tok_stride, 1) + 1) if hist.numel() > last else 0
    if step is not None:
        _need(step, torch.int32, "logits_process.step")
    check(_lib.load().srgpt_logits_process(_p(x), int(f32), _rowmajor2d(x, "logits_process.logits"), rows, V, _p(hist), hist_row_stride,
                                           hist_tok_stride, cap, _p(step), step_offset, _p(fparams), _p(spec), spec.numel(), _p(out),
                                           0 if out is None else _rowmajor2d(out, "logits_process.out"), _p(ids), _stream()),
          "srgpt_logits_process")
    if ids is not None:
        _count(2)  # the processing kernel and the key unpack


def logits_pick_token(ids: torch.Tensor, step: torch.Tensor, step_offset: int, out_ids: torch.Tensor, embed_table: Optional[torch.Tensor] = None,
                      next_x: Optional[torch.Tensor] = None) -> None:
    """out_ids[step + step_offset] = ids[0] (and next_x = embed_table[ids[0]]): the processed greedy choice of a one-token step."""
    _need(ids, torch.int64, "logits_pick_token.ids"); _need(step, torch.int32, "logits_pick_token.step")
    _need(out_ids, torch.int64, "logits_pick_token.out_ids")
    K = 0 if embed_table is None else embed_table.shape[1]
    check(_lib.load().srgpt_logits_pick_token(_p(ids), _p(step), step_offset, _p(out_ids), _p(embed_table), _p(next_x), K, _stream()),
          "srgpt_logits_pick_token")


def beam_candidates(logits: torch.Tensor, beam_scores: torch.Tensor, cand_scores: torch.Tensor, cand_tokens: torch.Tensor,
                    logprobs: Optional[torch.Tensor] = None) -> None:
    """Per beam row: the n_cand best (log_softmax(logits)[token] + beam_scores[row], token) -> cand_scores / cand_tokens [k, n_cand].
    ``logprobs`` (fp32 [k, V], unit inner stride, optional): every row's whole log_softmax."""
    _need(logits, ELEM(), "beam_candidates.logits"); _need(beam_scores, torch.float32, "beam_candidates.beam_scores")
    _need(cand_scores, torch.float32, "beam_candidates.cand_scores"); _need(cand_tokens, torch.int32, "beam_candidates.cand_tokens")
    k, V = logits.shape
    if cand_scores.shape != cand_tokens.shape or cand_scores.shape[0] != k or not cand_scores.is_contiguous() or not cand_tokens.is_contiguous():
        raise SrgptError("beam_candidates: cand_scores / cand_tokens must be contiguous [n_beams, n_cand]")
    if logprobs is not None:
        _need(logprobs, torch.float32, "beam_candidates.logprobs")
        if logprobs.shape != (k, V):
            raise SrgptError(f"beam_candidates: logprobs must be fp32 [{k}, {V}], got shape {tuple(logprobs.shape)}")
        check(_lib.load().srgpt_beam_candidates_scores_bf16(_p(logits), _rowmajor2d(logits, "beam_candidates.logits"), k, V, _p(beam_scores),
                                                            cand_scores.shape[1], _p(cand_scores), _p(cand_tokens), _p(logprobs),
                                                            _rowmajor2d(logprobs, "beam_candidates.logprobs"), _stream()),
              "srgpt_beam_candidates_scores_bf16")
        return
    check(_lib.load().srgpt_beam_candidates_bf16(_p(logits), _rowmajor2d(logits, "beam_candidates.logits"), k, V, _p(beam_scores), cand_scores.shape[1],
                                                 _p(cand_scores), _p(cand_tokens), _stream()), "srgpt_beam_candidates_bf16")


def beam_candidates_scored(logits: torch.Tensor, beam_scores: torch.Tensor, cand_scores: torch.Tensor, cand_tokens: torch.Tensor,
                           stats: torch.Tensor) -> None:
    """Per beam row: the n_cand best (log_softmax(logits)[token] + beam_scores[row], token) in (score desc, token asc) order of the fp32
    score -> cand_scores / cand_tokens [k, n_cand], and the row's (max, log-sum-exp) -> stats fp32 [k, 2] (diverse beam search)."""
    _need(logits, ELEM(), "beam_candidates_scored.logits"); _need(beam_scores, torch.float32, "beam_candidates_scored.beam_scores")
    _need(cand_scores, torch.float32, "beam_candidates_scored.cand_scores"); _need(cand_tokens, torch.int32, "beam_candidates_scored.cand_tokens")
    _need(stats, torch.float32, "beam_candidates_scored.stats")
    k, V = logits.shape
    if cand_scores.shape != cand_tokens.shape or cand_scores.shape[0] != k or not cand_scores.is_contiguous() or not cand_tokens.is_contiguous():
        raise SrgptError("beam_candidates_scored: cand_scores / cand_tokens must be contiguous [n_beams, n_cand]")
    if tuple(stats.shape) != (k, 2) or not stats.is_contiguous():
        raise SrgptError(f"beam_candidates_scored: stats must be contiguous fp32 [{k}, 2]")
    check(_lib.load().srgpt_beam_candidates_scored_bf16(_p(logits), _rowmajor2d(logits, "beam_candidates_scored.logits"), k, V, _p(beam_scores),
                                                        cand_scores.shape[1], _p(cand_scores), _p(cand_tokens), _p(stats), _stream()),
          "srgpt_beam_candidates_scored_bf16")


def beam_group_select(logits: torch.Tensor, stats: torch.Tensor, beam_scores: torch.Tensor, cand_tokens: torch.Tensor, k: int, n_groups: int,
                      eos: torch.Tensor, pad_id: int, diversity_penalty: float, done: torch.Tensor, out_scores: torch.Tensor,
                      out_beams: torch.Tensor, out_tokens: torch.Tensor, next_beams: torch.Tensor, next_tokens: torch.Tensor) -> None:
    """Diverse beam search's choice for the P = rows / k prompts of the [P * k, V] logits, group by group (srgpt_beam_group_select):
    stats / cand_tokens [P * k, L] from beam_candidates_scored over the same logits and beam_scores; eos int32 [n_eos]; done int32
    [P, n_groups].  -> out_scores / out_beams / out_tokens [P, n_groups, n_cand] (each group's ranked candidates, beams within the group)
    and next_beams / next_tokens int32 [P * k] (each beam's parent within its prompt, and its token)."""
    _need(logits, ELEM(), "beam_group_select.logits"); _need(stats, torch.float32, "beam_group_select.stats")
    _need(beam_scores, torch.float32, "beam_group_select.beam_scores"); _need(cand_tokens, torch.int32, "beam_group_select.cand_tokens")
    _need(eos, torch.int32, "beam_group_select.eos"); _need(done, torch.int32, "beam_group_select.done")
    _need(out_scores, torch.float32, "beam_group_select.out_scores")
    for t, name in ((out_beams, "out_beams"), (out_tokens, "out_tokens"), (next_beams, "next_beams"), (next_tokens, "next_tokens")):
        _need(t, torch.int32, f"beam_group_select.{name}")
    R, V = logits.shape
    if k < 1 or n_groups < 1 or R % k:
        raise SrgptError(f"beam_group_select: {R} rows are not prompts of k = {k} beams")
    P, L, n_cand = R // k, cand_tokens.shape[1], out_scores.shape[-1]
    if cand_tokens.shape[0] != R or not cand_tokens.is_contiguous() or tuple(stats.shape) != (R, 2) or not stats.is_contiguous():
        raise SrgptError(f"beam_group_select: cand_tokens must be contiguous [{R}, L] and stats [{R}, 2]")
    if beam_scores.numel() != R or tuple(done.shape) != (P, n_groups) or not done.is_contiguous() or not eos.is_contiguous():
        raise SrgptError(f"beam_group_select: beam_scores must hold {R} scores and done be [{P}, {n_groups}]")
    for o in (out_scores, out_beams, out_tokens):
        if tuple(o.shape) != (P, n_groups, n_cand) or not o.is_contiguous():
            raise SrgptError(f"beam_group_select: ranked outputs must be contiguous [{P}, {n_groups}, {n_cand}]")
    for o in (next_beams, next_tokens):
        if o.numel() != R or not o.is_contiguous():
            raise SrgptError(f"beam_group_select: next_beams / next_tokens must hold {R} entries")
    check(_lib.load().srgpt_beam_group_select(_p(logits), _rowmajor2d(logits, "beam_group_select.logits"), V, _p(stats), _p(beam_scores),
                                              _p(cand_tokens), L, P, k, n_groups, n_cand, _p(eos) if eos.numel() else None, eos.numel(),
                                              int(pad_id), float(diversity_penalty), _p(done), _p(out_scores), _p(out_beams), _p(out_tokens),
                                              _p(next_beams), _p(next_tokens), _stream()),
          "srgpt_beam_group_select")


def beam_select(cand_scores: torch.Tensor, cand_tokens: torch.Tensor, k: int, out_scores: torch.Tensor, out_beams: torch.Tensor,
                out_tokens: torch.Tensor) -> None:
    """Per prompt (k consecutive rows of the [G * k, n_cand] candidates of beam_candidates): its n_cand best (score, beam in the prompt,
    token) in (score desc, beam asc, token asc) order, token < 0 dropped -> out_* [G, n_cand] (-inf / -1 / -1 past the valid ones)."""
    _need(cand_scores, torch.float32, "beam_select.cand_scores"); _need(cand_tokens, torch.int32, "beam_select.cand_tokens")
    _need(out_scores, torch.float32, "beam_select.out_scores"); _need(out_beams, torch.int32, "beam_select.out_beams")
    _need(out_tokens, torch.int32, "beam_select.out_tokens")
    rows, n_cand = cand_scores.shape
    if k < 1 or rows % k or cand_tokens.shape != cand_scores.shape or not cand_scores.is_contiguous() or not cand_tokens.is_contiguous():
        raise SrgptError("beam_select: candidates must be contiguous [n_groups * k, n_cand] scores and tokens")
    G = rows // k
    for o in (out_scores, out_beams, out_tokens):
        if tuple(o.shape) != (G, n_cand) or not o.is_contiguous():
            raise SrgptError(f"beam_select: outputs must be contiguous [{G}, {n_cand}]")
    check(_lib.load().srgpt_beam_select(_p(cand_scores), _p(cand_tokens), G, k, n_cand, _p(out_scores), _p(out_beams), _p(out_tokens), _stream()),
          "srgpt_beam_select")


_KV_COPY_WS = {}  # device -> staging buffer of kv_copy_pages, grown on demand


def kv_copy_pages(pages: torch.Tensor, pairs, n_staged: int = 0) -> None:
    """Copies KV rows between pages of the paged cache pages [L, n_pages, 2, page_rows, n_kv_heads, head_dim] for K and V of every layer.
    pairs: a host int list / tensor [n, 4] of (src page, dst page, first row, rows).  The first n_staged pairs go through a workspace, so
    a pair whose destination is another pair's source must be among them (llama_decoder.beam_page_pairs orders them so)."""
    if not pages.is_cuda or pages.dim() != 6 or not pages.is_contiguous():
        raise SrgptError("kv_copy_pages: expected the contiguous CUDA KV cache [L, n_pages, 2, page_rows, n_kv_heads, head_dim]")
    L, n_pages, _, page_rows = pages.shape[:4]
    row_bytes = pages.shape[4] * pages.shape[5] * pages.element_size()
    host = torch.as_tensor(pairs, dtype=torch.int32).reshape(-1, 4)
    n = host.shape[0]
    if n == 0:
        return
    if not 0 <= n_staged <= n:
        raise SrgptError(f"kv_copy_pages: n_staged {n_staged} outside [0, {n}]")
    src, dst, lo, cnt = host.unbind(1)
    if bool(((src < 0) | (src >= n_pages) | (dst < 0) | (dst >= n_pages) | (lo < 0) | (cnt < 0) | (lo + cnt > page_rows)).any()):
        raise SrgptError(f"kv_copy_pages: a pair lies outside the {n_pages} pages of {page_rows} rows")
    lib = _lib.load()
    ws_bytes = int(lib.srgpt_kv_copy_workspace_bytes(n_staged, L, page_rows, row_bytes))
    ws = _KV_COPY_WS.get(pages.device)
    if n_staged and (ws is None or ws.numel() < ws_bytes):
        ws = _KV_COPY_WS[pages.device] = torch.empty(ws_bytes, dtype=torch.uint8, device=pages.device)
    d_pairs = host.to(pages.device, non_blocking=False)
    check(lib.srgpt_kv_copy_pages(_p(pages), L, n_pages, page_rows, row_bytes, _p(d_pairs), n, n_staged, _p(ws) if n_staged else None,
                                  ws_bytes if n_staged else 0, _stream()), "srgpt_kv_copy_pages")
    if n_staged:
        _count(1)


def kv_broadcast_rows(pages: torch.Tensor, page_tables: torch.Tensor, pos: torch.Tensor, pos_offset: int, sel: torch.Tensor, k: int) -> None:
    """Contrastive search's KV broadcast: for each prompt g (sel int32 [G]), the K / V of every layer at position pos[g * k + sel[g]] +
    pos_offset of row g * k + sel[g] -> the same position of rows g * k + i, i != sel[g].  page_tables: the cache's int32 [rows, cap]
    tables (row r = sequence r, G * k <= rows); pos: int32 [>= G * k]."""
    if not pages.is_cuda or pages.dim() != 6 or not pages.is_contiguous():
        raise SrgptError("kv_broadcast_rows: expected the contiguous CUDA KV cache [L, n_pages, 2, page_rows, n_kv_heads, head_dim]")
    _need(page_tables, torch.int32, "kv_broadcast_rows.page_tables"); _need(pos, torch.int32, "kv_broadcast_rows.pos")
    _need(sel, torch.int32, "kv_broadcast_rows.sel")
    G = sel.numel()
    if k < 1 or G < 1 or not sel.is_contiguous() or not pos.is_contiguous() or pos.numel() < G * k:
        raise SrgptError(f"kv_broadcast_rows: needs k >= 1, a contiguous sel [G >= 1] and pos of at least G * k entries")
    if page_tables.dim() != 2 or page_tables.shape[0] < G * k:
        raise SrgptError(f"kv_broadcast_rows: page_tables must be [>= {G * k}, cap], got shape {tuple(page_tables.shape)}")
    L, n_pages, _, page_rows = pages.shape[:4]
    row_bytes = pages.shape[4] * pages.shape[5] * pages.element_size()
    check(_lib.load().srgpt_kv_broadcast_rows(_p(pages), L, n_pages, page_rows, row_bytes, _p(page_tables),
                                              _rowmajor2d(page_tables, "kv_broadcast_rows.page_tables"), _p(pos), pos_offset, _p(sel), G, k,
                                              _stream()), "srgpt_kv_broadcast_rows")


def contrastive_partial(B: int, k: int, L_cap: int, device) -> torch.Tensor:
    """The fp32 buffer of contrastive_penalty's per-chunk maxima for B prompts of k candidates over contexts of at most L_cap rows."""
    n = int(_lib.load().srgpt_contrastive_partial_floats(B, k, L_cap))
    if n < 0:
        raise SrgptError(f"contrastive_partial: invalid B={B}, k={k}, L_cap={L_cap}")
    return torch.empty(n, dtype=torch.float32, device=device)


def contrastive_penalty(cand: torch.Tensor, ctx: torch.Tensor, pos: torch.Tensor, k: int, partial: torch.Tensor) -> None:
    """Degeneration penalty, first pass: the B * k rows of ``cand`` ([B * k, H], unit inner stride) against each prompt's context rows
    ctx[g, 0 .. pos[g * k]) (ctx contiguous [B, L_cap, H]) -> partial (contrastive_partial(B, k, L_cap)) = each 32-row chunk's largest
    cosine per candidate."""
    _need(cand, ELEM(), "contrastive_penalty.cand"); _need(ctx, ELEM(), "contrastive_penalty.ctx")
    _need(pos, torch.int32, "contrastive_penalty.pos"); _need(partial, torch.float32, "contrastive_penalty.partial")
    if ctx.dim() != 3 or not ctx.is_contiguous():
        raise SrgptError(f"contrastive_penalty: ctx must be contiguous [B, L_cap, H], got shape {tuple(ctx.shape)}")
    B, L_cap, H = ctx.shape
    if not 1 <= k <= 64 or tuple(cand.shape) != (B * k, H):
        raise SrgptError(f"contrastive_penalty: needs 1 <= k <= 64 and cand [{B} * k, {H}], got k={k}, shape {tuple(cand.shape)}")
    if pos.numel() < B * k or not pos.is_contiguous():
        raise SrgptError(f"contrastive_penalty: pos must be a contiguous int32 vector of at least {B * k} entries")
    if partial.numel() < _lib.load().srgpt_contrastive_partial_floats(B, k, L_cap) or not partial.is_contiguous():
        raise SrgptError("contrastive_penalty: partial is smaller than contrastive_partial(B, k, L_cap)")
    check(_lib.load().srgpt_contrastive_penalty_bf16(_p(cand), _rowmajor2d(cand, "contrastive_penalty.cand"), _p(ctx), L_cap, H, _p(pos), B, k,
                                                     _p(partial), _stream()), "srgpt_contrastive_penalty_bf16")


def contrastive_select(cand_scores: torch.Tensor, cand_tokens: torch.Tensor, partial: torch.Tensor, alpha: torch.Tensor, xn: torch.Tensor,
                       logits: torch.Tensor, ctx: torch.Tensor, next_logits: torch.Tensor, pos: torch.Tensor, out_ids: torch.Tensor,
                       step: torch.Tensor, ticket: torch.Tensor, sel: torch.Tensor, pen: torch.Tensor, score: torch.Tensor) -> None:
    """Contrastive search's choice for B prompts of k candidates (cand_scores fp32 / cand_tokens int32 [B, k], beam_candidates' log-probs
    over next_logits): pen = the penalty from ``partial``, score = (1 - a) * exp(log-prob) - a * pen with alpha = fp32 {1 - a, a}; the
    best candidate (lowest index on ties) -> sel [B], its token -> out_ids[step * B + g], its xn row appended to ctx[g] at pos[g * k],
    its logits row -> next_logits[g]; the k rows' positions and the step advance.  pen / score: fp32 [B, k]."""
    _need(cand_scores, torch.float32, "contrastive_select.cand_scores"); _need(cand_tokens, torch.int32, "contrastive_select.cand_tokens")
    _need(partial, torch.float32, "contrastive_select.partial"); _need(alpha, torch.float32, "contrastive_select.alpha")
    for t, n in ((xn, "xn"), (logits, "logits"), (ctx, "ctx"), (next_logits, "next_logits")):
        _need(t, ELEM(), "contrastive_select." + n)
    _need(pos, torch.int32, "contrastive_select.pos"); _need(out_ids, torch.int64, "contrastive_select.out_ids")
    _need(step, torch.int32, "contrastive_select.step"); _need(ticket, torch.int32, "contrastive_select.ticket")
    _need(sel, torch.int32, "contrastive_select.sel"); _need(pen, torch.float32, "contrastive_select.pen")
    _need(score, torch.float32, "contrastive_select.score")
    if cand_scores.dim() != 2 or cand_tokens.shape != cand_scores.shape or not cand_scores.is_contiguous() or not cand_tokens.is_contiguous():
        raise SrgptError("contrastive_select: candidates must be contiguous [B, k] scores and tokens")
    B, k = cand_scores.shape
    if not 1 <= k <= 64 or ctx.dim() != 3 or not ctx.is_contiguous() or ctx.shape[0] != B:
        raise SrgptError(f"contrastive_select: needs 1 <= k <= 64 and a contiguous ctx [{B}, L_cap, H]")
    _, L_cap, H = ctx.shape
    V = logits.shape[1]
    if tuple(xn.shape) != (B * k, H) or logits.shape[0] != B * k or tuple(next_logits.shape) != (B, V):
        raise SrgptError(f"contrastive_select: xn must be [{B * k}, {H}], logits [{B * k}, V] and next_logits [{B}, V]")
    if partial.numel() < _lib.load().srgpt_contrastive_partial_floats(B, k, L_cap) or alpha.numel() != 2:
        raise SrgptError("contrastive_select: partial is smaller than contrastive_partial(B, k, L_cap), or alpha is not {1 - a, a}")
    if pos.numel() < B * k or sel.numel() != B or pen.numel() != B * k or score.numel() != B * k or out_ids.numel() < B:
        raise SrgptError(f"contrastive_select: pos needs {B * k} entries, sel {B}, pen and score {B * k}, out_ids at least {B}")
    check(_lib.load().srgpt_contrastive_select_bf16(
        _p(cand_scores), _p(cand_tokens), _p(partial), _p(alpha), _p(xn), _rowmajor2d(xn, "contrastive_select.xn"), H, _p(logits),
        _rowmajor2d(logits, "contrastive_select.logits"), V, _p(ctx), L_cap, _p(next_logits), _rowmajor2d(next_logits, "contrastive_select.next_logits"),
        _p(pos), B, k, _p(out_ids), _p(step), _p(ticket), _p(sel), _p(pen), _p(score), _stream()), "srgpt_contrastive_select_bf16")


def argmax_f32(x: torch.Tensor) -> torch.Tensor:
    _need(x, torch.float32, "argmax_f32.x")
    rows, cols = x.shape
    out = torch.empty(rows, dtype=torch.int64, device=x.device)
    check(_lib.load().srgpt_argmax_f32(_p(x), rows, cols, _p(out), _stream()), "srgpt_argmax_f32")
    return out


def argmax_bf16(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need(x, ELEM(), "argmax_bf16.x")
    ldx = _rowmajor2d(x, "argmax_bf16.x")
    rows, cols = x.shape
    if out is None:
        out = torch.empty(rows, dtype=torch.int64, device=x.device)
    check(_lib.load().srgpt_argmax_bf16(_p(x), ldx, rows, cols, _p(out), _stream()), "srgpt_argmax_bf16")
    return out


# ------------------------------------------------------------------------------------------------ composite stacks
def _count(n: int) -> None:
    global LAUNCHES
    LAUNCHES += n - 1  # check() adds 1


def make_siglip_layer_array(layers):
    """ctypes array of srgpt_siglip_layer_weights over a list of VisionLayerW (keeps no tensor alive: the caller does)."""
    arr = (_lib.SiglipLayerWeights * len(layers))()
    for i, lw in enumerate(layers):
        for name in ("ln1_w", "ln1_b", "qkv_w", "qkv_b", "out_w", "out_b", "ln2_w", "ln2_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b"):
            setattr(arr[i], name, getattr(lw, name).data_ptr())
    return arr


_MATS = ("qkv", "o", "gateup", "down")


def _matrix_array(struct, desc, per_layer):
    """ctypes array of `struct` (srgpt_llama_layer_packed / _nf4) over per-layer dicts {"qkv", "o", "gateup", "down"} -> weight or None."""
    arr = (struct * len(per_layer))()
    for i, pl in enumerate(per_layer):
        for name in _MATS:
            setattr(arr[i], name, desc(pl[name]))
    return arr


class LlamaStack:
    """The Llama decoder's layers as the composite entry points (layers.cu) take them, and which family of those entry points each
    call uses.  Holds the layer array over the current KV pages (srgpt_llama_layer_fp8 when the layers' matrices are Fp8W, else
    srgpt_llama_layer_weights), the decode step's 12-bit packed matrices (``packed``: per-layer dicts of Packed12W or None) or NF4
    planes (``nf4``: from the layers' ``nf4`` dicts; ``planes_only``: the matrices keep no element-type copy, so prefill and the verify
    pass read the planes too), and lm_head's packing (``lm_packed``), with the tensors behind them."""

    def __init__(self, layers, kv_pages, packed=None, nf4: bool = False, planes_only: bool = False, lm_packed=None):
        self.src, self.n = layers, len(layers)
        self.quantizes_activations = any(isinstance(lw.qkv_w, Fp8W) for lw in layers)  # FP8: prefill / batched linears quantize x
        self.packed_layers, self.lm_packed = packed, lm_packed
        self.packed = None if packed is None else _matrix_array(_lib.LlamaLayerPacked, _packed_desc, packed)
        self.nf4 = _matrix_array(_lib.LlamaLayerNf4, _nf4_desc, [lw.nf4 for lw in layers]) if nf4 else None
        self.planes = self.nf4 if planes_only else None
        self._lm_desc = _packed_desc(lm_packed)
        # kernels per layer of the prefill stacks and the batched step (FP8: + 4 activation quantizers); of a decode step; of a verify pass
        self.kernels_per_layer = 12 if self.quantizes_activations else 8
        self.step_kernels = 5 * self.n + 2
        self.verify_kernels = 5 * self.n + 3
        self.rows_kernels = 5 * self.n + 2  # + 1 when the rows are sampled
        self.set_pages(kv_pages)

    def set_pages(self, kv_pages) -> None:
        """Rebuild the layer array over new per-layer KV pages (the packed and NF4 arrays point at no page).  A matrix held only as NF4
        planes (an Nf4W in its *_w field) gets NULL: the NF4 entry points take it from the planes."""
        if self.quantizes_activations:
            arr = (_lib.LlamaLayerFp8 * self.n)()
            for i, lw in enumerate(self.src):
                arr[i].in_norm, arr[i].post_norm = lw.in_norm.data_ptr(), lw.post_norm.data_ptr()
                for name in _MATS:
                    setattr(arr[i], name, _fp8_desc(getattr(lw, name + "_w")))
                arr[i].kv_pages = kv_pages[i].data_ptr()
        else:
            arr = (_lib.LlamaLayerWeights * self.n)()
            for i, lw in enumerate(self.src):
                for name in ("in_norm", "qkv_w", "o_w", "post_norm", "gateup_w", "down_w"):
                    t = getattr(lw, name)
                    setattr(arr[i], name, t.data_ptr() if isinstance(t, torch.Tensor) else None)
                arr[i].kv_pages = kv_pages[i].data_ptr()
        self.layers = arr

    def entry(self, op: str):
        """(symbol, layer array arguments, lm_head packing arguments) of srgpt_llama_<op>_*, op = "prefill_layers",
        "prefill_chunk_layers", "decode_step", "verify_step" or "decode_rows".  Prefill takes the FP8 or, planes-only, the NF4 stack; the
        decode step and the rows step stream FP8 (the step only), NF4 or packed matrices when there are some; the verify pass NF4
        planes-only or packed ones."""
        fmt, arrays, lm = self.formats(op)
        return f"srgpt_llama_{op}_{fmt + '_' if fmt else ''}bf16", arrays, lm

    def formats(self, op: str):
        """The weight format entry() picks for `op` ("" for the element-type matrices, "packed", "nf4" or "fp8"), the layer array
        arguments of that format and its lm_head packing arguments."""
        step = op in ("decode_step", "verify_step", "decode_rows")
        nf4 = self.nf4 if op in ("decode_step", "decode_rows") else self.planes
        if self.quantizes_activations:
            if op == "verify_step":
                raise SrgptError("the verify pass of prompt-lookup decoding has no FP8 form")
            if op == "decode_rows":
                raise SrgptError("the batch-invariant decode step has no FP8 form")
            fmt, arrays = "fp8", (self.layers,)
        elif nf4 is not None:
            fmt, arrays = "nf4", (self.layers, nf4)
        elif step and self.packed is not None:
            fmt, arrays = "packed", (self.layers, self.packed)
        else:
            fmt, arrays = "", (self.layers,)
        lm = (C.byref(self._lm_desc),) if step and fmt else ()
        return fmt, tuple(C.cast(a, C.c_void_p) for a in arrays), lm


def clip_embed(patch_embeds: torch.Tensor, class_embedding: torch.Tensor, position_embedding: torch.Tensor, n_img: int, T: int) -> torch.Tensor:
    """[n_img*T, D] patch embeddings -> [n_img*(T+1), D]: class token prepended, position embedding added (CLIPVisionEmbeddings)."""
    _need(patch_embeds, ELEM(), "clip_embed.patch_embeds")
    D = patch_embeds.shape[1]
    if patch_embeds.shape[0] != n_img * T or not patch_embeds.is_contiguous() or tuple(position_embedding.shape) != (T + 1, D):
        raise SrgptError(f"clip_embed: patch embeds {tuple(patch_embeds.shape)}, position embedding {tuple(position_embedding.shape)}, n_img {n_img}, T {T}")
    out = torch.empty((n_img * (T + 1), D), dtype=ELEM(), device=patch_embeds.device)
    check(_lib.load().srgpt_clip_embed_bf16(_p(patch_embeds), _p(class_embedding), _p(position_embedding), _p(out), n_img, T, D, _stream()),
          "srgpt_clip_embed_bf16")
    return out


def siglip_layers(x: torch.Tensor, layer_array, n_layers: int, n_img: int, T: int, D: int, heads: int, I: int, eps: float,
                  fc1_epilogue: int = EPI_BIAS_GELU_TANH) -> torch.Tensor:
    """n_layers pre-LN ViT encoder layers (SigLIP; CLIP with fc1_epilogue=EPI_BIAS_QUICK_GELU) in place on x [n_img*T, D]."""
    _need(x, ELEM(), "siglip_layers.x")
    _ensure_gemm_workspace(x.device)
    M = n_img * T
    dev = x.device
    ws_h = torch.empty((M, D), dtype=ELEM(), device=dev)
    ws_qkv = torch.empty((M, 3 * D), dtype=ELEM(), device=dev)
    ws_attn = torch.empty((M, D), dtype=ELEM(), device=dev)
    ws_mlp = torch.empty((M, I), dtype=ELEM(), device=dev)
    import ctypes
    check(_lib.load().srgpt_vit_layers_bf16(_p(x), ctypes.cast(layer_array, ctypes.c_void_p), n_layers, _p(ws_h), _p(ws_qkv),
                                            _p(ws_attn), _p(ws_mlp), n_img, T, D, heads, I, eps, fc1_epilogue, _stream()), "srgpt_vit_layers_bf16")
    _count(7 * n_layers)
    return x


def _fp8_workspaces(S: int, dims, dev):
    """The activation quantizer's codes [S, max(H, nh hd, I)] and scales [S] of the FP8 layer stacks."""
    K = max(dims.hidden_size, dims.num_attention_heads * dims.head_dim, dims.intermediate_size)
    return torch.empty(S * K, dtype=torch.uint8, device=dev), torch.empty(S, dtype=torch.float32, device=dev)


def _prefill(op: str, x: torch.Tensor, stack: LlamaStack, dims, cos, sin, start_pos, rows) -> torch.Tensor:
    """srgpt_llama_<op>_* of the stack over x [S, H] in place; ``rows`` = the entry point's arguments between sin and the stream."""
    _ensure_gemm_workspace(x.device)
    S, H = x.shape
    nh, nkv, hd, I = dims.num_attention_heads, dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
    dev = x.device
    ws = (torch.empty((S, H), dtype=ELEM(), device=dev), torch.empty((S, (nh + 2 * nkv) * hd), dtype=ELEM(), device=dev),
          torch.empty((S, nh * hd), dtype=ELEM(), device=dev), torch.empty((S, I), dtype=ELEM(), device=dev))
    if stack.quantizes_activations:
        ws += _fp8_workspaces(S, dims, dev)
    name, arrays, _ = stack.entry(op)
    check(getattr(_lib.load(), name)(_p(x), *arrays, stack.n, *(_p(t) for t in ws), S, H, nh, nkv, hd, I, dims.rms_norm_eps, _p(cos), _p(sin),
                                     _p(start_pos), *rows, _stream()), name)
    _count(stack.kernels_per_layer * stack.n)
    return x


def llama_prefill_layers(x: torch.Tensor, stack: LlamaStack, dims, cos, sin, start_pos, page_table, page_size: int,
                         cu_seqlens: Optional[torch.Tensor] = None, max_seqlen: int = 0) -> torch.Tensor:
    """All decoder layers over the prompt rows x [S, H] in place (K/V appended to the paged cache).  One prompt
    (page_table [cap], start_pos [1]) or, with cu_seqlens [n_seqs+1], n_seqs prompts packed back to back
    (page_table [n_seqs, cap], start_pos [n_seqs])."""
    _need(x, ELEM(), "llama_prefill_layers.x")
    n_seqs, pt_stride = 1, 0
    if cu_seqlens is not None:
        _need(cu_seqlens, torch.int32, "llama_prefill_layers.cu_seqlens")
        n_seqs = cu_seqlens.numel() - 1
        if page_table.dim() != 2 or page_table.shape[0] < n_seqs or start_pos.numel() < n_seqs or page_table.stride(1) != 1:
            raise SrgptError("llama_prefill_layers: packed prompts need page_table [n_seqs, cap] and start_pos [n_seqs]")
        pt_stride = page_table.stride(0)
    return _prefill("prefill_layers", x, stack, dims, cos, sin, start_pos,
                    (_p(page_table), page_size, n_seqs, _p(cu_seqlens), max_seqlen, pt_stride))


def llama_prefill_layers_probe(x: torch.Tensor, stack: LlamaStack, dims, cos, sin, start_pos, page_table, page_size: int, row_off: torch.Tensor,
                               hidden: Optional[torch.Tensor] = None, attn: Optional[torch.Tensor] = None,
                               cu_seqlens: Optional[torch.Tensor] = None, max_seqlen: int = 0) -> torch.Tensor:
    """llama_prefill_layers with the probes recorded: ``hidden`` [n_layers, n_seqs, R, H] gets the rows each layer reads (the
    embeddings, then the residual stream after every layer but the last), ``attn`` [n_layers, n_seqs, n_heads, R, R] every layer's
    attention probabilities; sequence b's rows start at output row row_off[b] (device int32 [n_seqs]).  Either may be None.  x, the KV
    cache and every bit of the arithmetic are those of llama_prefill_layers."""
    _need(x, ELEM(), "llama_prefill_layers_probe.x")
    _need(row_off, torch.int32, "llama_prefill_layers_probe.row_off")
    S, H = x.shape
    L, nh = stack.n, dims.num_attention_heads
    n_seqs, pt_stride = 1, 0
    if cu_seqlens is not None:
        _need(cu_seqlens, torch.int32, "llama_prefill_layers_probe.cu_seqlens")
        n_seqs = cu_seqlens.numel() - 1
        if page_table.dim() != 2 or page_table.shape[0] < n_seqs or start_pos.numel() < n_seqs or page_table.stride(1) != 1:
            raise SrgptError("llama_prefill_layers_probe: packed prompts need page_table [n_seqs, cap] and start_pos [n_seqs]")
        pt_stride = page_table.stride(0)
    if row_off.numel() < n_seqs:
        raise SrgptError("llama_prefill_layers_probe: row_off needs one offset per sequence")
    probe = _lib.PrefillProbe()
    R = None
    if hidden is not None:
        _need(hidden, ELEM(), "llama_prefill_layers_probe.hidden")
        if hidden.dim() != 4 or tuple(hidden.shape[:2]) != (L, n_seqs) or hidden.shape[3] != H or hidden.stride(3) != 1:
            raise SrgptError(f"llama_prefill_layers_probe: hidden must be [{L}, {n_seqs}, R, {H}] with unit inner stride, got {tuple(hidden.shape)}")
        R = hidden.shape[2]
        probe.hidden, probe.hidden_layer_stride, probe.hidden_seq_stride, probe.hidden_ld = hidden.data_ptr(), *hidden.stride()[:3]
    if attn is not None:
        _need(attn, ELEM(), "llama_prefill_layers_probe.attn")
        if attn.dim() != 5 or tuple(attn.shape[:3]) != (L, n_seqs, nh) or attn.shape[3] != attn.shape[4] or attn.stride(4) != 1:
            raise SrgptError(f"llama_prefill_layers_probe: attn must be [{L}, {n_seqs}, {nh}, R, R] with unit inner stride, got {tuple(attn.shape)}")
        if R is not None and attn.shape[3] != R:
            raise SrgptError("llama_prefill_layers_probe: hidden and attn must have the same rows per sequence")
        R = attn.shape[3]
        probe.attn, probe.attn_layer_stride, probe.attn_seq_stride, probe.attn_head_stride, probe.attn_ld = attn.data_ptr(), *attn.stride()[:4]
    if R is None:
        raise SrgptError("llama_prefill_layers_probe: nothing to record (hidden and attn are both None)")
    probe.out_rows, probe.row_off = R, row_off.data_ptr()
    _ensure_gemm_workspace(x.device)
    nkv, hd, I = dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
    dev = x.device
    ws = (torch.empty((S, H), dtype=ELEM(), device=dev), torch.empty((S, (nh + 2 * nkv) * hd), dtype=ELEM(), device=dev),
          torch.empty((S, nh * hd), dtype=ELEM(), device=dev), torch.empty((S, I), dtype=ELEM(), device=dev))
    ws += _fp8_workspaces(S, dims, dev) if stack.quantizes_activations else (None, None)
    fmt, arrays, _ = stack.formats("prefill_layers")
    layers, nf4, fp8 = (None, None, arrays[0]) if fmt == "fp8" else (arrays[0], arrays[1] if fmt == "nf4" else None, None)
    check(_lib.load().srgpt_llama_prefill_layers_probe_bf16(_p(x), layers, nf4, fp8, L, *(_p(t) for t in ws), S, H, nh, nkv, hd, I,
                                                            dims.rms_norm_eps, _p(cos), _p(sin), _p(start_pos), _p(page_table), page_size, n_seqs,
                                                            _p(cu_seqlens), max_seqlen, pt_stride, C.byref(probe), _stream()),
          "srgpt_llama_prefill_layers_probe_bf16")
    _count((stack.kernels_per_layer + (hidden is not None) + (attn is not None)) * L)
    return x


def attention_probs(q: torch.Tensor, k: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, scale: float, out: torch.Tensor,
                    cu_seqlens: Optional[torch.Tensor] = None, max_seqlen: int = 0, row_off: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Causal attention probabilities in the element type into out [n_seqs, n_heads, R, R] (any strides, unit inner one): q / k are
    row-major views [rows, heads * head_dim] (e.g. the rotated columns of a fused qkv buffer) of one sequence (cu_seqlens None) or of
    sequences packed by cu_seqlens [n_seqs + 1] (max_seqlen = the longest); sequence b's block starts at row / column row_off[b].
    Every entry of ``out`` is written."""
    _need(q, ELEM(), "attention_probs.q"); _need(k, ELEM(), "attention_probs.k"); _need(out, ELEM(), "attention_probs.out")
    n_seqs = 1 if cu_seqlens is None else cu_seqlens.numel() - 1
    if cu_seqlens is None:
        max_seqlen = q.shape[0]
    else:
        _need(cu_seqlens, torch.int32, "attention_probs.cu_seqlens")
    if row_off is not None:
        _need(row_off, torch.int32, "attention_probs.row_off")
    if out.dim() != 4 or tuple(out.shape[:2]) != (n_seqs, n_heads) or out.shape[2] != out.shape[3] or out.stride(3) != 1:
        raise SrgptError(f"attention_probs: out must be [{n_seqs}, {n_heads}, R, R] with unit inner stride, got {tuple(out.shape)}")
    check(_lib.load().srgpt_attention_probs_bf16(_p(q), _rowmajor2d(q, "attention_probs.q"), _p(k), _rowmajor2d(k, "attention_probs.k"), n_seqs,
                                                 _p(cu_seqlens), max_seqlen, n_heads, n_kv_heads, head_dim, scale, _p(out), out.stride(0),
                                                 out.stride(1), out.stride(2), out.shape[2], _p(row_off), _stream()), "srgpt_attention_probs_bf16")
    return out


DECODE_PROBS_CHUNK = 128  # output columns per CTA of srgpt_attention_probs_decode_bf16; its workspace holds a (max, sum) per chunk


def attention_probs_decode_ws(rows: int, n_heads: int, n_cols: int, device) -> torch.Tensor:
    """The fp32 workspace srgpt_attention_probs_decode_bf16 needs for `rows` rows of n_heads heads and n_cols output columns."""
    return torch.empty(rows * n_heads * ((n_cols + DECODE_PROBS_CHUNK - 1) // DECODE_PROBS_CHUNK) * 2, dtype=torch.float32, device=device)


def _check_decode_probs_out(out: torch.Tensor, R: int, n_heads: int, T: int, what: str) -> None:
    _need(out, ELEM(), what)
    if out.dim() != 4 or tuple(out.shape[1:3]) != (R, n_heads) or out.shape[3] < T or out.stride(3) != 1:
        raise SrgptError(f"{what} must be [steps, {R}, {n_heads}, n_cols >= {T}] with unit inner stride, got {tuple(out.shape)}")


def attention_probs_decode(q: torch.Tensor, kv_pages: torch.Tensor, page_tables: torch.Tensor, page_size: int, pos: torch.Tensor, n_heads: int,
                           n_kv_heads: int, head_dim: int, scale: float, off: torch.Tensor, n_prompt: torch.Tensor, T: int, step: torch.Tensor,
                           step_offset: int, out: torch.Tensor, ws: torch.Tensor) -> torch.Tensor:
    """The attention probabilities of a one-token decode step of R rows over one layer's paged cache, in the element type: q [R, >=
    n_heads * head_dim] (row-strided, e.g. the q columns of a fused qkv buffer; rotated), page_tables [>= R, cap] (or the one table of a
    single row), pos int32 [R] each row's newest position.  Row r, head h goes to out[step + step_offset, r, h] (``out`` a [steps, R,
    n_heads, n_cols] view with unit inner stride; ``step`` device int32 [1], read at run time) with prompt key p at column off[r] + p
    (p < n_prompt[r]) and generated key n_prompt[r] + j at column T + j; every column of the row's [0, T + pos[r] + 1 - n_prompt[r]) is
    written and nothing past it.  ``ws``: attention_probs_decode_ws(R, n_heads, n_cols)."""
    _need(q, ELEM(), "attention_probs_decode.q")
    for t, what in ((pos, "pos"), (off, "off"), (n_prompt, "n_prompt"), (step, "step"), (page_tables, "page_tables")):
        _need(t, torch.int32, "attention_probs_decode." + what)
    _need(ws, torch.float32, "attention_probs_decode.ws")
    R = q.shape[0]
    _check_decode_probs_out(out, R, n_heads, T, "attention_probs_decode.out")
    n_cols = out.shape[3]
    if pos.numel() < R or off.numel() < R or n_prompt.numel() < R or ws.numel() < attention_probs_decode_ws(R, n_heads, n_cols, "meta").numel():
        raise SrgptError("attention_probs_decode: pos / off / n_prompt need one entry per row and ws attention_probs_decode_ws's size")
    pt_stride = page_tables.stride(0) if page_tables.dim() == 2 else 0
    if R > 1 and (page_tables.dim() != 2 or page_tables.shape[0] < R or page_tables.stride(1) != 1):
        raise SrgptError("attention_probs_decode: R > 1 rows need page_tables [R, cap] with unit inner stride")
    check(_lib.load().srgpt_attention_probs_decode_bf16(_p(q), _rowmajor2d(q, "attention_probs_decode.q"), _p(kv_pages), _p(page_tables), pt_stride,
                                                        page_size, _p(pos), R, n_heads, n_kv_heads, head_dim, scale, _p(off), _p(n_prompt), T,
                                                        n_cols, _p(step), step_offset, _p(out), out.stride(0), out.stride(1), out.stride(2),
                                                        _p(ws), _stream()), "srgpt_attention_probs_decode_bf16")
    _count(2)
    return out


def store_step_rows(x: torch.Tensor, step: torch.Tensor, step_offset: int, dst: torch.Tensor) -> None:
    """Rows x [R, H] (contiguous, the element type) -> dst[step + step_offset] (``dst`` a [steps, R, H] view with unit inner stride;
    ``step`` device int32 [1], read at run time)."""
    _need(x, ELEM(), "store_step_rows.x"); _need(dst, ELEM(), "store_step_rows.dst"); _need(step, torch.int32, "store_step_rows.step")
    x2 = x.view(1, -1) if x.dim() == 1 else x
    if not x2.is_contiguous() or dst.dim() != 3 or tuple(dst.shape[1:]) != tuple(x2.shape) or dst.stride(2) != 1:
        raise SrgptError(f"store_step_rows: dst must be [steps, {x2.shape[0]}, {x2.shape[1]}] with unit inner stride over contiguous rows")
    check(_lib.load().srgpt_store_step_rows_bf16(_p(x2), x2.shape[0], x2.shape[1], _p(step), step_offset, _p(dst), dst.stride(0), dst.stride(1),
                                                 _stream()), "srgpt_store_step_rows_bf16")
    _count(1)


class StepProbe:
    """What the probed decode steps record (generate(output_hidden_states=, output_attentions=)): ``hidden`` [steps, L + 1, R, H] (slot l
    the row layer l reads, slot L the final norm of the last layer's row) and ``attn`` [steps, L, R, n_heads, n_cols] (each layer's
    probabilities in generate()'s padded columns: T prompt columns, row r's prompt at off[r], then the generated keys), either may be
    None; a step writes slot step + step_offset.  off / n_prompt: device int32 [R]; ws: attention_probs_decode_ws(R, n_heads, n_cols)."""

    def __init__(self, off: torch.Tensor, n_prompt: torch.Tensor, T: int, hidden: Optional[torch.Tensor] = None, attn: Optional[torch.Tensor] = None,
                 step_offset: int = -1):
        if hidden is None and attn is None:
            raise SrgptError("StepProbe: nothing to record (hidden and attn are both None)")
        for t, what in ((hidden, "hidden"), (attn, "attn")):
            if t is not None and (t.stride(-1) != 1 or t.dtype != ELEM()):
                raise SrgptError(f"StepProbe.{what} must be element-type with unit inner stride")
        self.off, self.n_prompt, self.T, self.hidden, self.attn, self.step_offset = off, n_prompt, int(T), hidden, attn, int(step_offset)
        self.ws = None if attn is None else attention_probs_decode_ws(attn.shape[2], attn.shape[3], attn.shape[4], attn.device)

    def kernels(self, n_layers: int, final_norm: bool) -> int:
        """Launches the probes add to a step of n_layers layers (the one-row step computes the final norm row itself)."""
        return n_layers * ((self.hidden is not None) + 2 * (self.attn is not None)) + (self.hidden is not None) * (2 if final_norm else 1)

    def key(self) -> tuple:
        """GraphKey.probe: the addresses and strides a captured graph holds."""
        return tuple((t.data_ptr(), tuple(t.shape), t.stride()) if t is not None else None
                     for t in (self.hidden, self.attn, self.off, self.n_prompt, self.ws)) + (self.T, self.step_offset)

    def desc(self, n_layers: int, n_heads: int):
        """The srgpt_decode_probe of a one-row step."""
        d = _lib.DecodeProbe()
        if self.hidden is not None:
            if self.hidden.dim() != 4 or self.hidden.shape[1] != n_layers + 1 or self.hidden.shape[2] != 1:
                raise SrgptError(f"StepProbe.hidden must be [steps, {n_layers + 1}, 1, H], got {tuple(self.hidden.shape)}")
            d.hidden, d.hidden_step_stride, d.hidden_layer_stride, d.hidden_row_stride = self.hidden.data_ptr(), *self.hidden.stride()[:3]
        if self.attn is not None:
            _check_decode_probs_out(self.attn[:, 0], 1, n_heads, self.T, "StepProbe.attn")
            if self.attn.shape[1] != n_layers:
                raise SrgptError(f"StepProbe.attn must hold {n_layers} layers, got {tuple(self.attn.shape)}")
            a = self.attn.stride()
            d.attn, d.attn_step_stride, d.attn_layer_stride, d.attn_row_stride, d.attn_head_stride = self.attn.data_ptr(), a[0], a[1], a[2], a[3]
            d.n_cols = self.attn.shape[4]
        d.step_offset, d.T, d.off, d.n_prompt, d.ws = self.step_offset, self.T, _p(self.off), _p(self.n_prompt), _p(self.ws)
        return d


def llama_prefill_chunk_layers(x: torch.Tensor, stack: LlamaStack, dims, cos, sin, start_pos, page_tables, page_size: int, n_pages: int,
                               cu_seqlens: torch.Tensor, max_rows: int) -> torch.Tensor:
    """All decoder layers over x [S, H] in place: n_seqs chunks packed by cu_seqlens [n_seqs+1] that continue their sequences at
    start_pos [n_seqs] (page_tables [n_seqs, cap]); attention reads every earlier position from the paged cache."""
    _need(x, ELEM(), "llama_prefill_chunk_layers.x")
    _need(cu_seqlens, torch.int32, "llama_prefill_chunk_layers.cu_seqlens")
    n_seqs = cu_seqlens.numel() - 1
    if page_tables.dim() != 2 or page_tables.shape[0] < n_seqs or start_pos.numel() < n_seqs or page_tables.stride(1) != 1:
        raise SrgptError("llama_prefill_chunk_layers: page_tables [n_seqs, cap] and start_pos [n_seqs] expected")
    return _prefill("prefill_chunk_layers", x, stack, dims, cos, sin, start_pos,
                    (_p(page_tables), page_tables.stride(0), page_size, n_pages, n_seqs, _p(cu_seqlens), max_rows))


def llama_decode_step(h, stack: LlamaStack, q_buf, attn_buf, act_buf, dims, cos, sin, pos, page_table, page_size: int,
                      final_norm, lm_head, embed, lm_ws, out_ids, step, logits_out=None, probe: Optional["StepProbe"] = None) -> None:
    """One whole decode step (5 kernels per layer, lm_head + arg max) streaming the stack's decode weights.  ``probe`` (a StepProbe of
    one row): the step also records its hidden rows and attention probabilities (srgpt_llama_decode_step_probe_bf16); every other
    output is bit-identical."""
    nh, nkv, hd, I = dims.num_attention_heads, dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
    if probe is not None:
        fmt, arrays, lm = stack.formats("decode_step")
        by = dict(zip({"": ("layers",), "fp8": ("fp8",)}.get(fmt, ("layers", fmt)), arrays))
        desc = probe.desc(stack.n, nh)
        check(_lib.load().srgpt_llama_decode_step_probe_bf16(
            _p(h), by.get("layers"), by.get("packed"), by.get("nf4"), by.get("fp8"), stack.n, _p(q_buf), _p(attn_buf), _p(act_buf),
            dims.hidden_size, nh, nkv, hd, I, dims.rms_norm_eps, _p(cos), _p(sin), _p(pos), _p(page_table), page_size, _p(final_norm),
            _p(lm_head), lm[0] if lm else None, dims.vocab_size, _p(embed), _p(lm_ws), _p(logits_out), _p(out_ids), _p(step), C.byref(desc),
            _stream()), "srgpt_llama_decode_step_probe_bf16")
        _count(stack.step_kernels + probe.kernels(stack.n, final_norm=True))
        return
    name, arrays, lm = stack.entry("decode_step")
    check(getattr(_lib.load(), name)(_p(h), *arrays, stack.n, _p(q_buf), _p(attn_buf), _p(act_buf), dims.hidden_size, nh, nkv, hd, I,
                                     dims.rms_norm_eps, _p(cos), _p(sin), _p(pos), _p(page_table), page_size, _p(final_norm), _p(lm_head), *lm,
                                     dims.vocab_size, _p(embed), _p(lm_ws), _p(logits_out), _p(out_ids), _p(step), _stream()), name)
    _count(stack.step_kernels)


def linear(x: torch.Tensor, w, q8: Optional[torch.Tensor] = None, s8: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
    """x · w^T (kw: gemm's residual / epilogue / out) by the kernel of w's format: gemm over an element-type matrix, gemm_nf4 over an
    Nf4W, the activation quantizer into q8 [M, >= K] / s8 [M] + gemm_fp8 over an Fp8W."""
    if isinstance(w, Nf4W):
        return gemm_nf4(x, w, **kw)
    if isinstance(w, Fp8W):
        return linear_fp8(x, w, q=q8[:, :x.shape[1]], scale=s8, **kw)
    return gemm(x, w, **kw)


# ------------------------------------------------------------------------------------------------ prompt-lookup speculative decoding
SPEC_T_MAX = _lib.SPEC_T_MAX


def gemv_multi(x: torch.Tensor, w: torch.Tensor, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
               residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0, head_dim: int = 0,
               cos=None, sin=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0, packed=None) -> torch.Tensor:
    """gemv() over the T rows of x [T, K] -> y [T, ldy] with every weight streamed once; each row is bit-identical to a one-token gemv()
    call (QKV_ROPE: row t at position pos + t).  ``packed`` = a Packed12W of ``w`` streams the 12-bit packing instead."""
    _need(x, ELEM(), "gemv_multi.x")
    T, K = x.shape
    N = w.shape[0] if packed is None else packed.sm.shape[0]
    ldx, ldy = _rowmajor2d(x, "gemv_multi.x"), _rowmajor2d(y, "gemv_multi.y")
    tail = (_p(norm_weight), eps, _p(residual), mode, n_heads, n_kv_heads, head_dim, _p(cos), _p(sin), _p(pos), _p(kv_pages), _p(page_table),
            page_size, _stream())
    if packed is None:
        check(_lib.load().srgpt_gemv_multi_bf16(_p(x), ldx, _p(w), w.stride(0), _p(y), ldy, T, N, K, *tail), "srgpt_gemv_multi_bf16")
    else:
        d = _packed_desc(packed)
        check(_lib.load().srgpt_gemv_multi_packed_bf16(_p(x), ldx, C.byref(d), _p(y), ldy, T, N, K, *tail), "srgpt_gemv_multi_packed_bf16")
    return y


def gemv_multi_nf4(x: torch.Tensor, p, y: torch.Tensor, norm_weight: Optional[torch.Tensor] = None, eps: float = 0.0,
                   residual: Optional[torch.Tensor] = None, mode: int = GEMV_PLAIN, n_heads: int = 0, n_kv_heads: int = 0, head_dim: int = 0,
                   cos=None, sin=None, pos=None, kv_pages=None, page_table=None, page_size: int = 0) -> torch.Tensor:
    """gemv_multi() streaming an Nf4W's planes: bit-identical to gemv_multi() over the dequantized matrix."""
    _need(x, ELEM(), "gemv_multi_nf4.x")
    T, K = x.shape
    N = p.q.shape[0]
    d = _nf4_desc(p)
    check(_lib.load().srgpt_gemv_multi_nf4_bf16(_p(x), _rowmajor2d(x, "gemv_multi_nf4.x"), C.byref(d), _p(y), _rowmajor2d(y, "gemv_multi_nf4.y"), T, N, K,
                                                _p(norm_weight), eps, _p(residual), mode, n_heads, n_kv_heads, head_dim, _p(cos), _p(sin), _p(pos),
                                                _p(kv_pages), _p(page_table), page_size, _stream()), "srgpt_gemv_multi_nf4_bf16")
    return y


def lm_head_multi(x: torch.Tensor, w: torch.Tensor, norm_weight: Optional[torch.Tensor], eps: float, workspace: torch.Tensor,
                  logits_out: Optional[torch.Tensor] = None, packed=None) -> None:
    """Final norm + lm_head over the T rows of x [T, H]: fp32 logits [T, V] (optional) and the per-token arg max partials in
    ``workspace`` (T * lm_head_workspace bytes), which spec_accept() reduces."""
    T, K = x.shape
    ldx = _rowmajor2d(x, "lm_head_multi.x")
    if packed is None:
        V = w.shape[0]
        check(_lib.load().srgpt_lm_head_multi_bf16(_p(x), ldx, _p(w), w.stride(0), T, V, K, _p(norm_weight), eps, _p(logits_out), _p(workspace),
                                                   _stream()), "srgpt_lm_head_multi_bf16")
    else:
        V = packed.sm.shape[0]
        d = _packed_desc(packed)
        check(_lib.load().srgpt_lm_head_multi_packed_bf16(_p(x), ldx, C.byref(d), T, V, K, _p(norm_weight), eps, _p(logits_out), _p(workspace),
                                                          _stream()), "srgpt_lm_head_multi_packed_bf16")


def attention_decode_multi(q: torch.Tensor, out: torch.Tensor, kv_pages: torch.Tensor, page_table: torch.Tensor, page_size: int,
                           pos_rows: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, scale: float) -> torch.Tensor:
    """Decode attention of T consecutive tokens: row t of q [T, >= nh*hd] attends over kv rows 0 .. pos_rows[t] -> out row t."""
    _need(pos_rows, torch.int32, "attention_decode_multi.pos_rows")
    T = q.shape[0]
    check(_lib.load().srgpt_attention_decode_multi_bf16(_p(q), _rowmajor2d(q, "attention_decode_multi.q"), _p(out),
                                                        _rowmajor2d(out, "attention_decode_multi.out"), _p(kv_pages), _p(page_table), page_size,
                                                        _p(pos_rows), T, n_heads, n_kv_heads, head_dim, scale, _stream()),
          "srgpt_attention_decode_multi_bf16")
    return out


def spec_draft(prompt_ids: Optional[torch.Tensor], prompt_len: Optional[torch.Tensor], out_ids: torch.Tensor, step: torch.Tensor, pos: torch.Tensor, pos_rows: torch.Tensor, T: int,
               ngram: int, embed_table: torch.Tensor, x: torch.Tensor, draft_ids: torch.Tensor, state: torch.Tensor) -> None:
    """prompt_ids: device int32 history buffer, prompt_len: device int32 [1] = its length (read at run time)."""
    check(_lib.load().srgpt_spec_draft(_p(prompt_ids), _p(prompt_len), _p(out_ids), _p(step), _p(pos), _p(pos_rows), T, ngram, _p(embed_table), _p(x),
                                       embed_table.shape[1], _p(draft_ids), _p(state), _stream()), "srgpt_spec_draft")


def spec_accept(workspace: torch.Tensor, V: int, T: int, draft_ids: torch.Tensor, out_ids: torch.Tensor, step: torch.Tensor, pos: torch.Tensor,
                state: torch.Tensor, logits_rows: Optional[torch.Tensor] = None, logits_all: Optional[torch.Tensor] = None) -> None:
    check(_lib.load().srgpt_spec_accept(_p(workspace), V, T, _p(draft_ids), _p(out_ids), out_ids.numel(), _p(step), _p(pos), _p(state),
                                        _p(logits_rows), _p(logits_all), _stream()), "srgpt_spec_accept")


def llama_verify_step(h, stack: LlamaStack, q_buf, attn_buf, act_buf, T: int, dims, cos, sin, pos, pos_rows, page_table, page_size: int,
                      final_norm, lm_head, embed, lm_ws, logits_rows, logits_all, prompt_ids, prompt_len, ngram: int, draft_ids, out_ids, step,
                      state) -> None:
    """One verify pass of T tokens (draft, layers, lm_head, accept) streaming the stack's verify weights."""
    nh, nkv, hd, I = dims.num_attention_heads, dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
    name, arrays, lm = stack.entry("verify_step")
    check(getattr(_lib.load(), name)(_p(h), *arrays, stack.n, _p(q_buf), _p(attn_buf), _p(act_buf), T, dims.hidden_size, nh, nkv, hd, I,
                                     dims.rms_norm_eps, _p(cos), _p(sin), _p(pos), _p(pos_rows), _p(page_table), page_size, _p(final_norm),
                                     _p(lm_head), *lm, dims.vocab_size, _p(embed), _p(lm_ws), _p(logits_rows), _p(logits_all), _p(prompt_ids),
                                     _p(prompt_len), ngram, _p(draft_ids), _p(out_ids), out_ids.numel(), _p(step), _p(state), _stream()), name)
    _count(stack.verify_kernels + (1 if logits_all is not None else 0))


# ------------------------------------------------------------------------------------------------ batch-invariant decoding
def gemv_rows(x: torch.Tensor, w, y: torch.Tensor, norm_weight: Optional[torch.Tensor], eps: float, n_heads: int, n_kv_heads: int,
              head_dim: int, cos, sin, pos_rows: torch.Tensor, kv_pages, page_tables: torch.Tensor, page_size: int, packed=None) -> torch.Tensor:
    """The QKV + RoPE + KV-append gemv of T rows of different sequences, x [T, K] -> y [T, >= nh*hd], every weight streamed once: row t
    at position pos_rows[t] (int32 [T]) with the page table page_tables[t] (row t of a [T, cap] view).  ``w`` is the element-type matrix
    or an Nf4W (its planes); ``packed`` = a Packed12W of ``w`` streams the 12-bit packing.  Row t equals a one-token gemv() there."""
    _need(x, ELEM(), "gemv_rows.x")
    _need(pos_rows, torch.int32, "gemv_rows.pos_rows")
    T, K = x.shape
    ldx, ldy, pt_ld = _rowmajor2d(x, "gemv_rows.x"), _rowmajor2d(y, "gemv_rows.y"), _rowmajor2d(page_tables, "gemv_rows.page_tables")
    tail = (_p(norm_weight), eps, n_heads, n_kv_heads, head_dim, _p(cos), _p(sin), _p(pos_rows), _p(kv_pages), _p(page_tables), pt_ld, page_size,
            _stream())
    lib = _lib.load()
    if isinstance(w, Nf4W):
        check(lib.srgpt_gemv_rows_nf4_bf16(_p(x), ldx, C.byref(_nf4_desc(w)), _p(y), ldy, T, w.q.shape[0], K, *tail), "srgpt_gemv_rows_nf4_bf16")
    elif packed is not None:
        check(lib.srgpt_gemv_rows_packed_bf16(_p(x), ldx, C.byref(_packed_desc(packed)), _p(y), ldy, T, packed.sm.shape[0], K, *tail),
              "srgpt_gemv_rows_packed_bf16")
    else:
        check(lib.srgpt_gemv_rows_bf16(_p(x), ldx, _p(w), w.stride(0), _p(y), ldy, T, w.shape[0], K, *tail), "srgpt_gemv_rows_bf16")
    return y


def attention_decode_rows(q: torch.Tensor, out: torch.Tensor, kv_pages: torch.Tensor, page_tables: torch.Tensor, page_size: int,
                          pos_rows: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int, scale: float) -> torch.Tensor:
    """Decode attention of T rows of different sequences: row t of q [T, >= nh*hd] attends over kv rows 0 .. pos_rows[t] of the page table
    page_tables[t] -> out row t, each row as attention_decode() computes it."""
    _need(pos_rows, torch.int32, "attention_decode_rows.pos_rows")
    T = q.shape[0]
    check(_lib.load().srgpt_attention_decode_rows_bf16(_p(q), _rowmajor2d(q, "attention_decode_rows.q"), _p(out),
                                                       _rowmajor2d(out, "attention_decode_rows.out"), _p(kv_pages), _p(page_tables),
                                                       _rowmajor2d(page_tables, "attention_decode_rows.page_tables"), page_size, _p(pos_rows), T,
                                                       n_heads, n_kv_heads, head_dim, scale, _stream()), "srgpt_attention_decode_rows_bf16")
    return out


def rows_advance(workspace: Optional[torch.Tensor], V: int, ids: Optional[torch.Tensor], B: int, embed_table: torch.Tensor, x: torch.Tensor,
                 out_ids: torch.Tensor, step: torch.Tensor, pos_rows: torch.Tensor) -> None:
    """The end of a step of B rows: each row's arg max from lm_head_multi's partials in ``workspace`` (or the ids [B] given) goes to
    out_ids[step * B + b], x row b becomes its embedding, pos_rows[b] and then step advance."""
    check(_lib.load().srgpt_rows_advance(_p(workspace), V, _p(ids), B, _p(embed_table), _p(x), embed_table.shape[1], _p(out_ids), _p(step),
                                         _p(pos_rows), _stream()), "srgpt_rows_advance")


def guidance_rows(logits: torch.Tensor, scale: torch.Tensor, guided: torch.Tensor, lse: Optional[torch.Tensor] = None,
                  ids: Optional[torch.Tensor] = None) -> None:
    """Classifier-free guidance over the fp32 rows logits [2P, V]: guided [P, V] row b = g * (log_softmax(row b) - log_softmax(row P + b))
    + log_softmax(row P + b) with g = scale[0] (device fp32), three separately rounded fp32 operations.  ``lse`` (fp32 [2P, 2]): each row's
    {max, log sum exp(x - max)}.  ``ids`` (int64 [2P]): ids[b] = ids[P + b] = the arg max of guided row b (lowest index on ties, NaN never
    wins)."""
    _need(logits, torch.float32, "guidance_rows.logits"); _need(scale, torch.float32, "guidance_rows.scale")
    _need(guided, torch.float32, "guidance_rows.guided")
    if logits.dim() != 2 or logits.shape[0] % 2 or not logits.is_contiguous():
        raise SrgptError(f"guidance_rows: logits must be contiguous fp32 [2P, V], got shape {tuple(logits.shape)}")
    P, V = logits.shape[0] // 2, logits.shape[1]
    if tuple(guided.shape) != (P, V) or not guided.is_contiguous():
        raise SrgptError(f"guidance_rows: guided must be contiguous fp32 [{P}, {V}], got shape {tuple(guided.shape)}")
    if lse is not None and (lse.dtype != torch.float32 or lse.numel() != 4 * P or not lse.is_contiguous()):
        raise SrgptError(f"guidance_rows: lse must be contiguous fp32 [{2 * P}, 2]")
    if ids is not None and (ids.dtype != torch.int64 or ids.numel() != 2 * P or not ids.is_contiguous()):
        raise SrgptError(f"guidance_rows: ids must be a contiguous int64 vector of {2 * P} entries")
    check(_lib.load().srgpt_guidance_rows(_p(logits), V, P, _p(scale), _p(guided), _p(lse), _p(ids), _stream()), "srgpt_guidance_rows")
    _count(1)


def guidance_pair_ids(ids: torch.Tensor, P: int) -> None:
    """ids[P + b] = ids[b] for b < P (int64 [2P])."""
    _need(ids, torch.int64, "guidance_pair_ids.ids")
    if ids.numel() < 2 * P:
        raise SrgptError(f"guidance_pair_ids: ids holds {ids.numel()} entries, needs {2 * P}")
    check(_lib.load().srgpt_guidance_pair_ids(_p(ids), P, _stream()), "srgpt_guidance_pair_ids")
    _count(1)


def llama_decode_rows(h, stack: LlamaStack, q_buf, attn_buf, act_buf, B: int, dims, cos, sin, pos_rows, page_tables, page_size: int, final_norm,
                      lm_head, embed, lm_ws, out_ids, step, logits_rows=None, sample_params=None, seeds=None, ids=None, guidance=None) -> None:
    """One decode step of B sequences, each row bit-identical to that sequence's one-token step (llama_decode_step): the rows layers,
    lm_head over the B rows, then the arg max (or, with ``seeds``, the draw from logits_rows) and the advance.  page_tables is a
    [>= B, cap] row-major view; row b of h / pos_rows / page_tables is sequence b.
    ``guidance`` = (scale, guided): classifier-free guidance over B = 2P rows, row P + b the unconditional branch of row b
    (srgpt_llama_decode_rows_guided_bf16): both rows of a pair take the arg max of guided row b, or with ``seeds`` ([P]) the draw from
    it.  scale is the device fp32 g, guided the fp32 [P, V] rows; ids [B] and logits_rows are needed.
    ``sample_params`` of 6 floats (with ``seeds``): the draws run HF's typical / epsilon / eta warpers after top-p
    (srgpt_llama_decode_rows_warped_bf16, guided or not; sample_top_p's params)."""
    nh, nkv, hd, I = dims.num_attention_heads, dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
    warped = seeds is not None and sample_params is not None and sample_params.numel() == 6
    if guidance is not None or warped:  # one entry point for every format of the rows step: the format's array goes to its own argument
        fmt, arrays, lm = stack.formats("decode_rows")
        desc = None if guidance is None else _lib.Guidance(_p(guidance[0]), _p(guidance[1]))
        layers = arrays[0]
        packed = arrays[1] if fmt == "packed" else None
        nf4 = arrays[1] if fmt == "nf4" else None
        name = "srgpt_llama_decode_rows_warped_bf16" if warped else "srgpt_llama_decode_rows_guided_bf16"
        check(getattr(_lib.load(), name)(
            _p(h), layers, packed, nf4, stack.n, _p(q_buf), _p(attn_buf), _p(act_buf), B, dims.hidden_size, nh, nkv, hd, I, dims.rms_norm_eps,
            _p(cos), _p(sin), _p(pos_rows), _p(page_tables), _rowmajor2d(page_tables, "llama_decode_rows.page_tables"), page_size, _p(final_norm),
            _p(lm_head), lm[0] if lm else None, dims.vocab_size, _p(embed), _p(lm_ws), _p(logits_rows), _p(sample_params), _p(seeds), _p(ids),
            _p(out_ids), _p(step), None if desc is None else C.byref(desc), _stream()), name)
        _count(stack.rows_kernels + ((3 if seeds is not None else 1) if guidance is not None else 1))
        return
    name, arrays, lm = stack.entry("decode_rows")
    check(getattr(_lib.load(), name)(_p(h), *arrays, stack.n, _p(q_buf), _p(attn_buf), _p(act_buf), B, dims.hidden_size, nh, nkv, hd, I,
                                     dims.rms_norm_eps, _p(cos), _p(sin), _p(pos_rows), _p(page_tables),
                                     _rowmajor2d(page_tables, "llama_decode_rows.page_tables"), page_size, _p(final_norm), _p(lm_head), *lm,
                                     dims.vocab_size, _p(embed), _p(lm_ws), _p(logits_rows), _p(sample_params), _p(seeds), _p(ids), _p(out_ids),
                                     _p(step), _stream()), name)
    _count(stack.rows_kernels + (1 if seeds is not None else 0))
