"""CPU restatement of the FP8 (E4M3) W8A8 definition the kernels implement (include/srgpt_b200.h srgpt_fp8, DESIGN.md §3).

Every row r of a weight W [N, K] or an activation x [M, K] is quantized alike:
  a = max_k |x[r, k]| in fp32; inv = fl32(448 / a), s[r] = fl32(a / 448) (both 1 when a == 0);
  q[r, k] = e4m3(fl32(x[r, k] * inv)), round to nearest even, saturated to +-448.
A linear is y[m, n] = acc[m, n] * fl32(s_x[m] * s_w[n]), acc the sum of the exact products float(q_x) * float(q_w).  The order of the sum
is not part of the definition, nor quite its precision: the H100's FP8 tensor cores add the 32 products of one wgmma with fewer bits than
fp32 before they reach the fp32 accumulators.  ``linear`` below sums in fp64, where the sum is exact.
"""
import torch

E4M3_MAX = 448.0


def e4m3(v: torch.Tensor) -> torch.Tensor:
    """fp32 -> float8_e4m3fn codes as uint8, RNE with saturation.  The clamp is needed: .to(float8_e4m3fn) maps 470 to NaN."""
    return torch.clamp(v.float(), -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def decode(q: torch.Tensor) -> torch.Tensor:
    """uint8 E4M3 codes -> their fp32 values."""
    return q.view(torch.float8_e4m3fn).float()


def quantize_rows(x: torch.Tensor):
    """x [M, K] (any float dtype) -> (q [M, K] uint8, s [M] fp32)."""
    xf = x.float()
    a = xf.abs().amax(1)
    one = torch.ones_like(a)
    inv = torch.where(a > 0, torch.full_like(a, E4M3_MAX) / torch.where(a > 0, a, one), one)
    s = torch.where(a > 0, a / E4M3_MAX, one)
    return e4m3(xf * inv[:, None]), s


def linear_q(qx: torch.Tensor, sx: torch.Tensor, qw: torch.Tensor, sw: torch.Tensor):
    """The W8A8 linear over quantized operands (qx [M, K], sx [M]) and (qw [N, K], sw [N]), on qx's device -> (y [M, N] fp32, bound [M, N]).
    y = fp32(exact acc) * fl32(s_x s_w); bound = max(K 2^-21, 2^-12) sum |products|, scaled the same: what the tensor cores' summation may
    move acc by.  An fp32 sum stays within K 2^-24 sum |products|; the FP8 wgmma's was measured on H100 at up to 3.5 times that for
    K >= 4096, and at 2^-12.9 sum |products| for K = 256 (its error does not shrink with K as an fp32 sum's does)."""
    dev = qx.device
    dx, dw = decode(qx).double(), decode(qw.to(dev)).double()
    acc = dx @ dw.t()
    mag = dx.abs() @ dw.abs().t()
    sc = sx.to(dev).float()[:, None] * sw.to(dev).float()[None, :]
    return acc.float() * sc, (mag * max(qx.shape[1] * 2.0 ** -21, 2.0 ** -12)).float() * sc


def linear(x: torch.Tensor, qw: torch.Tensor, sw: torch.Tensor) -> torch.Tensor:
    """y [M, N] fp32 of the W8A8 linear of the activation x [M, K] (quantized here) over (qw, sw), acc summed in fp64."""
    qx, sx = quantize_rows(x)
    return linear_q(qx, sx, qw, sw)[0]
