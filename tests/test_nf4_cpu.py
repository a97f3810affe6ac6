"""NF4 weight-only quantization checked without a GPU: the numpy restatement's invariants (tests/nf4_ref.py), a replay of the NF4 decode
GEMV's lane-order addressing, scale shuffle and dequantization against the plain GEMV's fp32 sum order, the C-ABI's argument checks,
the exports of both builds and the NF4 kernels' resources in SASS."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from tests import nf4_ref as R
from tests.test_packed_ring_cpu import cuda_tool


def test_code_table_and_midpoints():
    c = R.NF4_CODE
    assert c.dtype == np.float32 and c.size == 16 and np.all(np.diff(c) > 0)
    assert (c[0], c[7], c[15]) == (-1.0, 0.0, 1.0)
    # the published QLoRA / bitsandbytes NF4 table, to the printed digits
    assert np.allclose(c[[1, 6, 8, 14]], [-0.6961928, -0.0910500, 0.0795803, 0.7229568], atol=1e-7)
    m = R.NF4_MID
    assert m.size == 15 and np.all(m > c[:-1]) and np.all(m < c[1:])
    assert np.array_equal(m, ((c[:-1] + c[1:]) * np.float32(0.5)).astype(np.float32))


def test_dynamic_map_invariants_and_the_product_map():
    d = R.DYN_MAP
    assert d.dtype == np.float32 and d.size == 256 and np.all(np.diff(d) > 0)
    assert 0.0 in d and 1.0 in d and -1.0 not in d
    neg, pos = d[d < 0], d[(d > 0) & (d < 1)]
    assert neg.size == pos.size == 127 and np.array_equal(-neg[::-1], pos)
    assert np.isclose(pos.min(), 0.55e-6) and pos.max() < 1.0  # 10^-6 * the one midpoint of linspace(0.1, 1, 2)
    from spatialrgpt_b200 import ops
    assert np.array_equal(ops.nf4_dynamic_map("cpu").numpy().view(np.uint32), d.view(np.uint32))


def test_exact_code_values_round_trip():
    rng = np.random.default_rng(0)
    q = rng.integers(0, 16, size=(8, 256)).astype(np.uint8)
    q[:, ::64] = 15  # every block holds +1 * a, so absmax = a exactly
    a = np.float32(2.0) ** rng.integers(-12, -2, size=(8, 4)).astype(np.float32)
    w = (R.NF4_CODE[q] * np.repeat(a, 64, axis=1)).astype(np.float32)
    q2, absmax = R.quantize(w)
    assert np.array_equal(absmax, a) and np.array_equal(q2, q)
    assert np.array_equal(R.unpack_natural(R.pack_natural(q)), q)
    assert R.pack_natural(np.array([[1, 2]], dtype=np.uint8))[0, 0] == 0x12


def test_zero_block_rule():
    w = np.zeros((2, 128), dtype=np.float32)
    w[1, 64:] = np.linspace(-0.5, 0.5, 64)
    q, absmax = R.quantize(w)
    assert np.all(q[0] == 7) and np.all(q[1, :64] == 7) and absmax[0, 0] == 0.0
    q, s, deq = R.quantize_all(w, "bf16")
    assert np.all(deq[0] == 0.0) and np.all(deq[1, :64] == 0.0)
    # a zero beside subnormal weights whose reciprocal overflows: NaN -> code 7, the subnormals keep their sign's end code
    sub = np.zeros((1, 64), dtype=np.float32)
    sub[0, 1], sub[0, 2] = np.float32(1e-39), np.float32(-1e-39)
    q, _ = R.quantize(sub)
    assert q[0, 0] == 7 and q[0, 1] == 15 and q[0, 2] == 0


def test_rounding_is_to_the_nearest_code():
    w = np.linspace(-1, 1, 4096, dtype=np.float32).reshape(64, 64)
    w[:, 0] = 1.0  # absmax 1: x = w
    q, _ = R.quantize(w)
    dist = np.abs(w[..., None].astype(np.float64) - R.NF4_CODE.astype(np.float64))
    clear = np.abs(w[..., None] - R.NF4_MID).min(-1) > 1e-6  # away from a midpoint, where the decimal tie rules may differ
    assert np.array_equal(q[clear], dist.argmin(-1)[clear])
    assert np.all(q[np.isin(w, R.NF4_MID)] == np.searchsorted(R.NF4_MID, w[np.isin(w, R.NF4_MID)]))  # a tie goes down


@pytest.mark.parametrize("seed", [0, 1])
def test_resolved_scale_error_within_half_a_map_gap(seed):
    rng = np.random.default_rng(seed)
    absmax = (np.abs(rng.standard_normal((96, 56))) * 0.05).astype(np.float32)
    absmax[3, :7] = 1.5  # outliers
    scale, offset, codes2, m2 = R.double_quant(absmax)
    a = absmax.reshape(-1)
    d = R.DYN_MAP
    gap = np.maximum(np.diff(d, prepend=d[0])[codes2], np.diff(d, append=d[-1])[codes2])
    bound = 0.5 * gap * np.repeat(m2, R.BLOCK2)[:a.size] * (1 + 1e-5) + 4 * np.spacing(np.float32(abs(offset) + a.max()))
    assert np.all(np.abs(scale.reshape(-1).astype(np.float64) - a) <= bound)
    assert offset == np.float32(a.astype(np.float64).sum() / a.size)


def _fma(a, b, c):
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def _warp_sum(v):
    v = list(v)
    for o in (16, 8, 4, 2, 1):
        v = [np.float32(v[l] + v[l ^ o]) for l in range(32)]
    return v[0]


def _plain_gemv_row(wrow, x):
    """decode_gemv_kernel's fp32 sum of one row: lane l runs dot8 over chunks l, l + 32, ... (a fresh fma chain per chunk, added to
    the lane's partial), then warp_sum."""
    parts = []
    for l in range(32):
        acc = np.float32(0)
        for c in range(l, wrow.size // 8, 32):
            d = np.float32(0)
            for t in range(8):
                d = _fma(wrow[8 * c + t], x[8 * c + t], d)
            acc = np.float32(acc + d)
        parts.append(acc)
    return _warp_sum(parts)


def _nf4_gemv_pair(plane, scale, r0, r1, x, elem):
    """decode_gemv_nf4_kernel's sums of rows r0 / r1 from the lane-ordered plane: per batch b lane l loads its 16 code bytes of each
    row at b * 512 + 16 l and the scale of block 16 b + (l & 15) of row r0 (l < 16) or r1; chunk i's scales come by shuffle from
    lanes 4 i + l / 8 and 16 + 4 i + l / 8."""
    K = plane.shape[1] * 2
    a = [[np.float32(0)] * 32 for _ in range(2)]
    for b in range(K // 1024):
        s_lane = [scale[r0 if l < 16 else r1, 16 * b + (l & 15)] for l in range(32)]
        for l in range(32):
            for i in range(4):
                c = b * 128 + l + 32 * i
                for ri, r in enumerate((r0, r1)):
                    s = s_lane[(16 if ri else 0) + 4 * i + (l >> 3)]
                    word = int.from_bytes(plane[r, b * 512 + 16 * l + 4 * i: b * 512 + 16 * l + 4 * i + 4].tobytes(), "little")
                    f = R.round_to_elem((R.NF4_CODE[[(word >> (4 * t)) & 15 for t in range(8)]] * np.float32(s)).astype(np.float32), elem)
                    d = np.float32(0)
                    for t in range(8):
                        d = _fma(f[t], x[8 * c + t], d)
                    a[ri][l] = np.float32(a[ri][l] + d)
    return _warp_sum(a[0]), _warp_sum(a[1])


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_gemv_replay_from_the_lane_order_reproduces_the_plain_sum(elem):
    rng = np.random.default_rng(5)
    N, K = 4, 2048
    w = R.round_to_elem((rng.standard_normal((N, K)) * 0.02).astype(np.float32), elem)
    q, scale, deq = R.quantize_all(w, elem)
    plane = R.lane_order(q)
    x = R.round_to_elem(rng.standard_normal(K).astype(np.float32), elem)
    for r0, r1 in ((0, 1), (2, 3)):
        got = _nf4_gemv_pair(plane, scale, r0, r1, x, elem)
        want = (_plain_gemv_row(deq[r0], x), _plain_gemv_row(deq[r1], x))
        assert np.float32(got[0]).view(np.uint32) == np.float32(want[0]).view(np.uint32)
        assert np.float32(got[1]).view(np.uint32) == np.float32(want[1]).view(np.uint32)


def test_lane_order_is_a_permutation_of_the_natural_bytes():
    rng = np.random.default_rng(9)
    q = rng.integers(0, 16, size=(3, 2048)).astype(np.uint8)
    plane = R.lane_order(q)
    offs = R.lane_offset(np.arange(2048 // 8))
    assert np.array_equal(np.sort(offs), np.arange(0, 1024, 4))
    # chunk 37 of row 1: word at its lane offset, weight t in nibble t
    word = int.from_bytes(plane[1, offs[37]: offs[37] + 4].tobytes(), "little")
    assert [(word >> (4 * t)) & 15 for t in range(8)] == q[1, 8 * 37: 8 * 37 + 8].tolist()


@pytest.fixture(scope="module", params=["bf16", "f16"])
def lib(request):
    from spatialrgpt_b200 import _lib
    return _lib.load(elem=request.param)


def test_c_abi_rejects_bad_arguments_without_a_gpu(lib):
    from spatialrgpt_b200 import _lib
    fake = 1 << 20  # aligned, never dereferenced: the checks run before any CUDA call
    d = _lib.Nf4(q=fake, scale=fake)
    args = lambda K, desc: (fake, C.byref(desc) if desc is not None else None, fake + 4096, 64, K, None, 0.0, None, 0, 0, 0, 0,  # noqa: E731
                            None, None, None, None, None, 0, None)
    assert lib.srgpt_gemv_nf4_bf16(*args(4096, None)) == -1
    assert lib.srgpt_gemv_nf4_bf16(*args(4096, _lib.Nf4(q=None, scale=fake))) == -1
    assert lib.srgpt_gemv_nf4_bf16(*args(4096, _lib.Nf4(q=fake, scale=None))) == -1
    assert lib.srgpt_gemv_nf4_bf16(*args(4100, d)) == -1  # K % 64
    assert b"BLOCK" in lib.srgpt_last_error()
    assert lib.srgpt_gemv_nf4_bf16(*args(640, d)) == -1  # K % 1024
    assert b"BATCH" in lib.srgpt_last_error()
    assert lib.srgpt_nf4_quantize_bf16(fake, 100, 4, 100, fake, fake, fake, None) == -1
    assert lib.srgpt_nf4_quantize_bf16(None, 128, 4, 128, fake, fake, fake, None) == -1
    assert lib.srgpt_nf4_lane_order(fake, 4, 640, fake + 4096, None) == -1
    assert lib.srgpt_nf4_unpack_bf16(C.byref(_lib.Nf4(q=fake, scale=fake)), 4, 640, fake, 640, None) == -1
    assert lib.srgpt_nf4_dequantize_bf16(None, fake, 4, 128, fake, 128, None) == -1
    assert lib.srgpt_nf4_double_quant(None, 10, fake, fake, fake, None) == -1
    assert lib.srgpt_llama_decode_step_nf4_bf16(*([None] * 3), 1, *([None] * 3), 64, 1, 1, 64, 64, 1e-5, *([None] * 4), 16, *([None] * 3), 8,
                                                *([None] * 6)) == -1


NF4_KERNELS = r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-2]ENS0_3Nf4EEEvNS0_6ParamsE"
NEW_SYMBOLS = ["srgpt_nf4_quantize_bf16", "srgpt_nf4_double_quant", "srgpt_nf4_dequantize_bf16", "srgpt_nf4_lane_order", "srgpt_nf4_unpack_bf16",
               "srgpt_gemv_nf4_bf16", "srgpt_llama_decode_step_nf4_bf16"]


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_builds_export_the_nf4_entries(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.lib_path(elem)], capture_output=True, text=True, check=True).stdout
    for s in NEW_SYMBOLS:
        assert re.search(rf"\sT\s+{s}$", out, flags=re.M), s


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_nf4_format_gemv_kernels_fit_three_ctas_per_sm_without_local_memory(elem):
    """The plain decode GEMV runs 3 CTAs of 256 threads per SM (80 registers); the NF4 kernels must allow the same."""
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    r = subprocess.run([cuda_tool("cuobjdump"), "--dump-resource-usage", _lib.lib_path(elem)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", r.stdout))
    nf4 = {k: v for k, v in usage.items() if re.match(NF4_KERNELS, k)}
    assert len(nf4) == 3, "one NF4 GEMV per mode (plain, SwiGLU, QKV + RoPE)"
    for name, u in nf4.items():
        reg, stack, local = (int(re.search(f"{k}:(\\d+)", u).group(1)) for k in ("REG", "STACK", "LOCAL"))
        assert reg <= 80 and stack == 0 and local == 0, (name, u)
    s = subprocess.run([cuda_tool("cuobjdump"), "-sass", _lib.lib_path(elem)], capture_output=True, text=True).stdout
    for f in re.split(r"\n\s*Function : ", s)[1:]:
        name, body = f.split("\n", 1)
        if re.match(NF4_KERNELS, name.strip()):
            body = body.split("\n\t\t..........")[0]
            assert "STL" not in body and "LDL" not in body and "LDGSTS" in body and "SHFL.IDX" in body
