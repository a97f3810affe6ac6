"""The 12-bit lossless packing of decode weights (DESIGN.md §3, csrc/pack12.cuh), checked without a GPU: a numpy reference of
the format, the GEMV's decode arithmetic replayed in numpy on it, and the C-ABI's argument checks and SASS."""
import re
import subprocess

import numpy as np
import pytest

MAX_EXC_PER_ROW, MAX_EXC_RATE = 32, 0.01


def bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit patterns (round to nearest even), uint16."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def sm_offset(cc):
    return (cc >> 7) * 1024 + ((cc >> 6) & 1) * 512 + (cc & 31) * 16 + ((cc >> 5) & 1) * 8


def ex_offset(cc):
    return (cc >> 7) * 512 + (cc & 31) * 16 + ((cc >> 5) & 3) * 4


def nibble_of(t):
    return ((t & 1) << 2) | (t & 2) | (t >> 2)


def pack12_np(w16: np.ndarray):
    """bf16 bits [N, K] -> dict(sm, ex, base, row_ptr, exc), or (None, reason) for a matrix that stays plain."""
    N, K = w16.shape
    if K % 1024:
        return None, "K"
    e = ((w16 >> 7) & 0xFF).astype(np.int32)
    if (e == 255).any():
        return None, "inf/nan"
    base = np.maximum(1, e.max(axis=1) - 14)
    is_exc = (e != 0) & (e < base[:, None])
    n_exc = is_exc.sum(axis=1)
    if n_exc.sum() > MAX_EXC_RATE * N * K:
        return None, "rate"
    if n_exc.max(initial=0) > MAX_EXC_PER_ROW:
        return None, "row"
    code = np.where((e != 0) & ~is_exc, e - base[:, None] + 1, 0).astype(np.uint32)
    smb = (((w16 >> 8) & 0x80) | (w16 & 0x7F)).astype(np.uint8)
    cc = np.arange(K // 8)
    sm = np.zeros((N, K), np.uint8)
    ex = np.zeros((N, K // 2), np.uint8)
    for t in range(8):
        sm[:, sm_offset(cc) + t] = smb[:, t::8]
    words = np.zeros((N, K // 8), np.uint32)
    for t in range(8):
        words |= code[:, t::8] << (4 * nibble_of(t))
    for k in range(4):
        ex[:, ex_offset(cc)[None, :].repeat(1, 0)[0] + k] = ((words >> (8 * k)) & 0xFF).astype(np.uint8)
    rows, cols = np.nonzero(is_exc)  # row-major: sorted by column within a row
    exc = (cols.astype(np.int64) << 8 | e[rows, cols]).astype(np.int32)
    row_ptr = np.concatenate([[0], np.cumsum(n_exc)]).astype(np.int32)
    return dict(sm=sm, ex=ex, base=base.astype(np.uint8), row_ptr=row_ptr, exc=exc), None


def _prmt_signrep(s: np.ndarray, sel: int) -> np.ndarray:
    """prmt.b32 d, s, 0, sel (default mode: selector bit 3 replicates the byte's sign) over uint32 arrays."""
    out = np.zeros_like(s)
    for k in range(4):
        nib = (sel >> (4 * k)) & 0xF
        byte = (s >> np.uint32(8 * (nib & 3))) & np.uint32(0xFF) if (nib & 7) < 4 else np.zeros_like(s)
        if nib & 8:
            byte = np.where(byte & np.uint32(0x80), np.uint32(0xFF), np.uint32(0))
        out |= byte << np.uint32(8 * k)
    return out


def decode_chunk_np(s_lo, s_hi, e, bp):
    """pack12::decode_chunk, operation for operation, on uint32 arrays -> the 4 words of bf16 pairs."""
    u = np.uint32
    x0 = e & u(0x0F0F0F0F)
    x1 = (e >> u(4)) & u(0x0F0F0F0F)
    x0 = x0 + (((x0 + u(0x7F7F7F7F)) >> u(7)) & u(0x01010101)) * bp
    x1 = x1 + (((x1 + u(0x7F7F7F7F)) >> u(7)) & u(0x01010101)) * bp
    merge = lambda a, b: (a & u(0x807F807F)) | (b & u(0x7F807F80))  # noqa: E731
    return [merge(_prmt_signrep(s_lo, 0x9180), x0 << u(7)), merge(_prmt_signrep(s_lo, 0xB3A2), x0 >> u(1)),
            merge(_prmt_signrep(s_hi, 0x9180), x1 << u(7)), merge(_prmt_signrep(s_hi, 0xB3A2), x1 >> u(1))]


def unpack12_np(p) -> np.ndarray:
    """The inverse through decode_chunk_np, plus the exception patch: bf16 bits [N, K]."""
    sm, ex = p["sm"], p["ex"]
    N, K = sm.shape
    cc = np.arange(K // 8)
    smw = sm.reshape(N, -1).view(np.uint8)
    s_lo = np.zeros((N, K // 8), np.uint32)
    s_hi = np.zeros((N, K // 8), np.uint32)
    e = np.zeros((N, K // 8), np.uint32)
    for k in range(4):
        s_lo |= smw[:, sm_offset(cc) + k].astype(np.uint32) << np.uint32(8 * k)
        s_hi |= smw[:, sm_offset(cc) + 4 + k].astype(np.uint32) << np.uint32(8 * k)
        e |= ex[:, ex_offset(cc) + k].astype(np.uint32) << np.uint32(8 * k)
    bp = (p["base"].astype(np.uint32) - np.uint32(1))[:, None]
    words = decode_chunk_np(s_lo, s_hi, e, bp)
    out = np.zeros((N, K), np.uint16)
    for j, wd in enumerate(words):
        out[:, 8 * cc + 2 * j] = (wd & np.uint32(0xFFFF)).astype(np.uint16)
        out[:, 8 * cc + 2 * j + 1] = (wd >> np.uint32(16)).astype(np.uint16)
    for r in range(N):
        for v in p["exc"][p["row_ptr"][r]:p["row_ptr"][r + 1]]:
            out[r, v >> 8] |= np.uint16((v & 0xFF) << 7)
    return out


def _roundtrip(w16):
    p, why = pack12_np(w16)
    assert p is not None, why
    assert np.array_equal(unpack12_np(p), w16)
    return p


RNG = np.random.default_rng(0)


@pytest.mark.parametrize("kind", ["gauss", "lm_head", "student_t", "row_scaled"])
def test_roundtrip_is_bit_exact(kind):
    N, K = 16, 2048
    if kind == "gauss":
        x = RNG.normal(0, 0.02, (N, K))
    elif kind == "lm_head":
        x = RNG.normal(0, 0.08, (N, K))
    elif kind == "student_t":
        x = RNG.standard_t(3, (N, K)) * 0.02
    else:
        x = RNG.normal(0, 1, (N, K)) * np.exp(RNG.normal(0, 2, (N, 1)))
    w16 = bf16_bits(x)
    p = _roundtrip(w16)
    assert p["sm"].nbytes + p["ex"].nbytes == N * K * 3 // 2


def test_zeros_subnormals_and_signs_are_exact():
    w16 = bf16_bits(RNG.normal(0, 0.02, (4, 1024)))
    w16[0, :16] = [0x0000, 0x8000, 0x0001, 0x807F, 0x0040, 0x8001, 0x0000, 0x8000] * 2  # ±0 and subnormals: code 0, not listed
    w16[1, :] = 0x8000  # a row of -0
    p = _roundtrip(w16)
    assert all((v >> 8) >= 16 for v in p["exc"][p["row_ptr"][0]:p["row_ptr"][1]])
    assert p["row_ptr"][2] == p["row_ptr"][1]


def test_row_with_the_maximum_number_of_exceptions():
    w16 = bf16_bits(RNG.normal(0, 0.02, (3, 4096)))
    w16[1] = (120 << 7) | RNG.integers(0, 1 << 16, 4096, dtype=np.uint16) & 0x807F  # one exponent: no natural exceptions
    cols = RNG.choice(4096, MAX_EXC_PER_ROW, replace=False)
    w16[1, cols] = 0x0080 | (w16[1, cols] & 0x807F)  # exponent 1: far below the window
    p = _roundtrip(w16)
    assert p["row_ptr"][2] - p["row_ptr"][1] == MAX_EXC_PER_ROW
    w16[1, (cols[0] + 1) % 4096] = 0x0100  # one more exception than a row may hold
    assert pack12_np(w16) == (None, "row")


def test_exceptions_in_the_first_and_last_chunk_of_a_lane():
    w16 = bf16_bits(RNG.normal(0, 0.02, (2, 2048)))
    # lane 0: chunks 0 and 224 (its last, batch 1 step 3); lane 31: chunks 31 and 255 (weight 7)
    for col in (0, 8 * 224 + 3, 8 * 31 + 7, 8 * 255 + 7, 2047):
        w16[0, col] = 0x0100 | (w16[0, col] & 0x807F)
    _roundtrip(w16)


def test_matrices_that_stay_plain():
    w16 = bf16_bits(RNG.normal(0, 0.02, (8, 1024)))
    for bad in (0x7F80, 0xFF80, 0x7FC1):  # +Inf, -Inf, NaN
        v = w16.copy()
        v[3, 5] = bad
        assert pack12_np(v) == (None, "inf/nan")
    dense = bf16_bits(RNG.normal(0, 1, (8, 1024)) * np.exp(RNG.uniform(-30, 0, (8, 1024))))  # exponents spread far below the max
    assert pack12_np(dense)[0] is None
    assert pack12_np(w16[:, :1000])[1] == "K"


def test_layout_is_the_lanes_batches():
    """Chunk c of a row belongs to lane c % 32 and batch c // 128; inside a batch a lane's 4 chunks are 2 sm vectors + 1 ex vector."""
    assert [sm_offset(c) for c in (0, 32, 64, 96, 1, 128)] == [0, 8, 512, 520, 16, 1024]
    assert [ex_offset(c) for c in (0, 32, 64, 96, 1, 128)] == [0, 4, 8, 12, 16, 512]
    assert sorted(nibble_of(t) for t in range(8)) == list(range(8))


# ---- C-ABI without a GPU --------------------------------------------------------------------------------------------------
P = 1 << 20  # a 16-byte-aligned stand-in pointer: argument checks fail before anything touches it


def _desc(**over):
    from spatialrgpt_b200 import _lib
    d = _lib.Packed12()
    for k in ("sm", "ex", "base", "row_ptr", "exc"):
        setattr(d, k, over.get(k, P))
    return d


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_cabi_rejects_bad_arguments_without_a_gpu(elem):
    import ctypes as C

    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    ok = _desc()
    for d, K in ((_desc(sm=None), 4096), (_desc(exc=None), 4096), (_desc(ex=P + 8), 4096), (ok, 4000)):
        assert lib.srgpt_gemv_packed_bf16(P, C.byref(d), P, 64, K, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == -1
        assert lib.srgpt_lm_head_argmax_packed_bf16(P, C.byref(d), 65, K, None, 0.0, None, P, None, None, P, P, P, None) == -1
        assert lib.srgpt_unpack12_bf16(C.byref(d), 64, K, P, K, None) == -1
    assert lib.srgpt_gemv_packed_bf16(P, None, P, 64, 4096, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == -1
    if elem == "bf16":  # the half build refuses a well-formed descriptor before looking at the rest
        assert lib.srgpt_gemv_packed_bf16(P, C.byref(ok), P, 63, 4096, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == -1
        assert lib.srgpt_gemv_packed_bf16(P, C.byref(ok), P, 64, 4096, None, 0.0, None, 7, 0, 0, 0, None, None, None, None, None, 0, None) == -1
    assert lib.srgpt_pack12_scan_bf16(P, 1000, 4, 1000, P, P, P, None) == -1
    assert lib.srgpt_pack12_bf16(P, 4096, 4, 4096, P, None, P, P, P, None) == -1
    assert "invalid argument" in lib.srgpt_last_error().decode()
    assert lib.srgpt_llama_decode_step_packed_bf16(P, P, None, 1, P, P, P, 4096, 32, 8, 128, 14336, 1e-5, P, P, P, P, 16, P, P, None, 65, P, P,
                                                   None, P, P, None) == -1


def test_f16_build_refuses_the_packing():
    import ctypes as C

    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem="f16")
    d = _desc()
    assert lib.srgpt_gemv_packed_bf16(P, C.byref(d), P, 64, 4096, None, 0.0, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) == -3
    assert lib.srgpt_pack12_scan_bf16(P, 4096, 4, 4096, P, P, P, None) == -3
    assert "bfloat16" in lib.srgpt_last_error().decode()


def test_packed12_gemv_kernels_are_in_the_library_without_spills():
    from spatialrgpt_b200 import _lib
    _lib.load()
    r = subprocess.run(["cuobjdump", "-sass", _lib.lib_path()], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    funcs = re.split(r"\n\s*Function : ", r.stdout)
    packed = [f for f in funcs if re.match(r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-3]ENS0_8Packed12EEE", f)]
    assert len(packed) == 4, "one packed GEMV per mode (plain, SwiGLU, QKV + RoPE, lm_head)"
    for f in packed:
        assert "PRMT" in f and "LDG.E.NA.128" in f
        assert "STL" not in f and "LDL" not in f, "the packed GEMV must keep everything in registers"
