"""Numpy restatement of the NF4 weight-only quantization (csrc/nf4.cu, DESIGN.md §3): the rules the device quantizer, the dequantize
kernel and the NF4 decode GEMV are checked against.

It restates bitsandbytes' quantize_4bit(quant_type="nf4", blocksize=64, compress_statistics=True), the setting the reference's
load_pretrained_model(load_4bit=True) loads the LLM with (llava/model/builder.py:51-60).  bitsandbytes is not available here, so
nothing is pinned to its bytes; every choice is stated below.

* Blocks: 64 consecutive weights of a row.  The input is the element-type (bf16 / fp16) weight as loaded, held exactly in fp32.
  absmax = the fp32 maximum of |w| over the block.
* Normalisation: x = w * fl32(1 / absmax) (a reciprocal, then a multiply, as bitsandbytes' blockwise kernel does).
* Code table: the 16 NF4 values of QLoRA / bitsandbytes (NF4_CODE).
* Rounding: q = the number of fp32 midpoints fl32(fl32(c_i + c_{i+1}) * 0.5) that x exceeds (compared with `>`), i.e. the nearest
  code with a tie going to the lower one.  bitsandbytes compares against hard-coded decimal midpoints, so a value within an ulp
  of a midpoint may get the neighbouring code there.
* Zero blocks: a NaN x (w = 0 against an infinite reciprocal: an all-zero block, or a zero beside subnormal weights whose
  reciprocal overflows) gets code 7, the value 0.  bitsandbytes computes 0 * inf there.
* Packing (natural order): two codes per byte, the even index in the high nibble.
* Double quantization, over the matrix's absmax vector in natural (row-major) order:
  - offset = its mean: summed in fp64 in index order and rounded to fp32.  This is deterministic; torch's fp32 mean, which
    bitsandbytes uses, is not, and can differ from it in the last bits.
  - blocks of 256 of v = fl32(absmax - offset): absmax2 = max |v|, y = v * fl32(1 / absmax2), clamped to [-1, 1] (a NaN y, from a
    block whose values all equal the offset, counts as 0), code = the nearest entry of the signed dynamic map by fp32 distance
    |fl32(y - map[k])|, the lowest index on a tie.
  - dynamic map = bitsandbytes' create_dynamic_map(signed=True): for i = 0..6, +-10^(i-6) times the midpoints of
    linspace(0.1, 1, 2^i + 1), plus 0 and 1, sorted: 256 values.  Here the linspace points are fl32(0.1 + 0.9 j / (n - 1))
    computed in fp64 and the midpoints and products in fp32 (torch's fp32 linspace may differ in the last bit).
  - resolved scale = fl32(map[c] * absmax2) + offset in fp32.  The NF4 codes were chosen with the exact absmax; the scale is the
    lossy one (bitsandbytes' order).
* Dequantized value: round_to_elem(fl32(NF4_CODE[q] * scale)), rounding to nearest even.  The element-type value is what
  Linear4bit multiplies with: it dequantizes to the compute dtype first.
* Lane order (the decode GEMV's q plane): chunk cc (weights 8 cc .. 8 cc + 7) of a row goes to byte offset
  (cc >> 7) * 512 + (cc & 31) * 16 + ((cc >> 5) & 3) * 4 as one 32-bit word, weight t in bits 4t .. 4t + 3.
"""
import numpy as np

NF4_CODE = np.array([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635, -0.18477343022823334,
                     -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725, 0.24611230194568634, 0.33791524171829224,
                     0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0], dtype=np.float32)
NF4_MID = ((NF4_CODE[:-1] + NF4_CODE[1:]) * np.float32(0.5)).astype(np.float32)
BLOCK, BLOCK2 = 64, 256


def dynamic_map() -> np.ndarray:
    vals = []
    for i in range(7):
        n = 2 ** i + 1
        b = np.array([0.1 + 0.9 * j / (n - 1) for j in range(n)], dtype=np.float32)
        means = (b[:-1] + b[1:]) * np.float32(0.5)
        s = np.float32(10.0 ** (i - 6))
        vals += list(s * means) + list(-(s * means))
    vals += [np.float32(0.0), np.float32(1.0)]
    return np.sort(np.array(vals, dtype=np.float32))


DYN_MAP = dynamic_map()


def quantize(w: np.ndarray):
    """w: fp32 [N, K] holding element-type values.  -> (codes uint8 [N, K] one per weight, absmax fp32 [N, K/64])."""
    n, K = w.shape
    blk = w.astype(np.float32).reshape(n, K // BLOCK, BLOCK)
    absmax = np.abs(blk).max(-1).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        rcp = (np.float32(1.0) / absmax).astype(np.float32)
        x = (blk * rcp[..., None]).astype(np.float32)
    q = np.zeros(x.shape, dtype=np.uint8)
    for m in NF4_MID:
        q += (x > m).astype(np.uint8)
    q[np.isnan(x)] = 7
    return q.reshape(n, K), absmax


def pack_natural(q: np.ndarray) -> np.ndarray:
    """codes [N, K] -> [N, K/2] bytes, weight 2j in the high nibble of byte j."""
    return ((q[:, 0::2] << 4) | q[:, 1::2]).astype(np.uint8)


def unpack_natural(b: np.ndarray) -> np.ndarray:
    q = np.empty((b.shape[0], b.shape[1] * 2), dtype=np.uint8)
    q[:, 0::2], q[:, 1::2] = b >> 4, b & 15
    return q


def double_quant(absmax: np.ndarray):
    """absmax (any shape, natural order) -> (resolved scales fp32 of the same shape, offset, codes2, absmax2)."""
    a = absmax.reshape(-1).astype(np.float32)
    offset = np.float32(np.cumsum(a.astype(np.float64))[-1] / a.size)
    v = (a - offset).astype(np.float32)
    nb = (a.size + BLOCK2 - 1) // BLOCK2
    pad = np.zeros(nb * BLOCK2, dtype=np.float32)
    pad[:a.size] = v
    m2 = np.abs(pad.reshape(nb, BLOCK2)).max(-1).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        y = (pad.reshape(nb, BLOCK2) * (np.float32(1.0) / m2).astype(np.float32)[:, None]).astype(np.float32).reshape(-1)[:a.size]
    y = np.where(np.isnan(y), np.float32(0.0), np.clip(y, np.float32(-1.0), np.float32(1.0))).astype(np.float32)
    codes2 = np.empty(a.size, dtype=np.int64)
    for s in range(0, a.size, 1 << 14):
        d = np.abs((y[s:s + (1 << 14), None] - DYN_MAP[None, :]).astype(np.float32))
        codes2[s:s + (1 << 14)] = d.argmin(-1)
    m2_of = np.repeat(m2, BLOCK2)[:a.size]
    scale = ((DYN_MAP[codes2] * m2_of).astype(np.float32) + offset).astype(np.float32)
    return scale.reshape(absmax.shape), offset, codes2, m2


def round_to_elem(x: np.ndarray, elem: str) -> np.ndarray:
    """fp32 -> the nearest bf16 / fp16 value (ties to even), returned as fp32."""
    x = np.asarray(x, dtype=np.float32)
    if elem == "f16":
        return x.astype(np.float16).astype(np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def dequantize(q: np.ndarray, scale: np.ndarray, elem: str) -> np.ndarray:
    """codes [N, K], scales [N, K/64] -> the element-type values as fp32 [N, K]."""
    s = np.repeat(scale.astype(np.float32), BLOCK, axis=1)
    return round_to_elem((NF4_CODE[q] * s).astype(np.float32), elem)


def quantize_all(w: np.ndarray, elem: str):
    """The whole pipeline of one matrix: (codes [N, K], resolved scales [N, K/64], dequantized fp32 [N, K])."""
    q, absmax = quantize(w)
    scale = double_quant(absmax)[0]
    return q, scale, dequantize(q, scale, elem)


def lane_offset(cc):
    return (cc >> 7) * 512 + (cc & 31) * 16 + ((cc >> 5) & 3) * 4


def lane_order(q: np.ndarray) -> np.ndarray:
    """codes [N, K] (K a multiple of 1024) -> the GEMV's q plane [N, K/2]."""
    n, K = q.shape
    words = np.zeros((n, K // 8), dtype=np.uint32)
    for t in range(8):
        words |= q[:, t::8].astype(np.uint32) << np.uint32(4 * t)
    out = np.zeros((n, K // 2), dtype=np.uint8)
    offs = lane_offset(np.arange(K // 8))
    for k in range(4):
        out[:, offs + k] = ((words >> np.uint32(8 * k)) & 0xFF).astype(np.uint8)
    return out
