"""The NF4 GEMM and the multi-token NF4 GEMV checked without a GPU: a numpy replay of the GEMM producer's addressing over the decode GEMV's
planes (tests/nf4_ref.py), the C-ABI's argument checks and exports in both builds, the new kernels' resources in SASS, and the loader's
argument validation."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from tests import nf4_ref as R
from tests.test_packed_ring_cpu import cuda_tool

BM = BN = 128
BK = 64


def _replay_b_stage(plane, scale, n0, kb, N, elem):
    """The 128B-swizzled B stage gemm_nf4_kernel's producer writes for n-tile n0, k-block kb: thread pt fills 16-byte slot j = pt % 8 of
    tile rows pt / 8 + 16 i at byte r * 128 + ((j ^ (r & 7)) << 4), from the word at lane_offset(8 kb + j) of row n0 + r and the scale
    kb of that row; rows at or beyond N hold code 7 with scale 0.  Returns the stage as fp32 [128 rows, 64 weights] in smem order."""
    K = plane.shape[1] * 2
    stage = np.zeros(BN * 128 // 2, dtype=np.float32)  # 64 two-byte elements per 128-byte row
    for pt in range(128):
        j, r0 = pt & 7, pt >> 3
        for i in range(8):
            r = r0 + 16 * i
            row = n0 + r
            if row < N:
                off = R.lane_offset(8 * kb + j)
                word = int.from_bytes(plane[row, off:off + 4].tobytes(), "little")
                s = scale[row, kb]
            else:
                word, s = 0x77777777, np.float32(0)
            vals = R.round_to_elem((R.NF4_CODE[[(word >> (4 * t)) & 15 for t in range(8)]] * s).astype(np.float32), elem)
            byte = r * 128 + ((j ^ (r0 & 7)) << 4)
            assert (r & 7) == (r0 & 7)
            stage[byte // 2: byte // 2 + 8] = vals
    return stage


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_producer_addressing_rebuilds_the_natural_order_tile(elem):
    rng = np.random.default_rng(1)
    N, K = 200, 2048  # a partial second n-tile
    w = (rng.standard_normal((N, K)) * 0.02).astype(np.float32)
    w[3, :64] = 0
    q, s, deq = R.quantize_all(w, elem)
    plane = R.lane_order(q)
    for n0 in (0, 128):
        for kb in (0, 1, 5, 15, 16, 31):
            stage = _replay_b_stage(plane, s, n0, kb, N, elem)
            for r in range(BN):
                for c in range(8):  # the swizzle: chunk c of row r at 16-byte slot c ^ (r & 7)
                    got = stage[(r * 128 + ((c ^ (r & 7)) << 4)) // 2:][:8]
                    want = deq[n0 + r, kb * BK + 8 * c: kb * BK + 8 * c + 8] if n0 + r < N else np.zeros(8, np.float32)
                    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (n0, kb, r, c)


@pytest.fixture(scope="module", params=["bf16", "f16"])
def lib(request):
    from spatialrgpt_b200 import _lib
    return _lib.load(elem=request.param)


def test_nf4_gemm_rejects_bad_arguments_without_a_gpu(lib):
    from spatialrgpt_b200 import _lib
    fake = 1 << 20  # aligned, never dereferenced: the checks run before any CUDA call
    d = _lib.Nf4(q=fake, scale=fake)

    def gemm(desc, K=4096, epi=0, A=fake, M=32, N=256):
        return lib.srgpt_gemm_nf4_bf16(A, K, None if desc is None else C.byref(desc), fake + (1 << 24), N, M, N, K, None, 0, epi, None)
    assert gemm(None) == -1
    assert gemm(_lib.Nf4(q=None, scale=fake)) == -1
    assert gemm(_lib.Nf4(q=fake, scale=None)) == -1
    assert gemm(d, K=640) == -1 and b"BATCH" in lib.srgpt_last_error()
    assert gemm(_lib.Nf4(q=fake + 4, scale=fake)) == -1  # a misaligned q
    assert gemm(d, epi=1) == -1  # SRGPT_EPI_BIAS: not one of the three
    assert gemm(d, epi=6) == -1
    assert gemm(d, A=None) == -1


def test_multi_token_nf4_gemv_rejects_bad_arguments_without_a_gpu(lib):
    from spatialrgpt_b200 import _lib
    fake = 1 << 20
    d = _lib.Nf4(q=fake, scale=fake)

    def multi(desc, T=2, K=1024):
        return lib.srgpt_gemv_multi_nf4_bf16(fake, K, None if desc is None else C.byref(desc), fake + (1 << 24), 64, T, 64, K, None, 0.0, None, 0,
                                             0, 0, 0, None, None, None, None, None, 0, None)
    assert multi(None) == -1
    assert multi(_lib.Nf4(q=None, scale=fake)) == -1
    assert multi(_lib.Nf4(q=fake + 4, scale=fake)) == -1
    assert multi(d, K=640) == -1
    assert multi(d, T=0) == -1 and multi(d, T=9) == -1
    assert lib.srgpt_llama_prefill_layers_nf4_bf16(*([None] * 2), None, 1, *([None] * 4), 16, 64, 1, 1, 64, 64, 1e-5, *([None] * 4), 16, 1,
                                                   None, 16, 0, None) == -1
    assert lib.srgpt_llama_verify_step_nf4_bf16(*([None] * 3), 1, *([None] * 3), 2, 64, 1, 1, 64, 64, 1e-5, *([None] * 5), 16, *([None] * 3), 8,
                                                *([None] * 6), 2, *([None] * 2), 8, *([None] * 3)) == -1


NEW_SYMBOLS = ["srgpt_gemm_nf4_bf16", "srgpt_gemv_multi_nf4_bf16", "srgpt_llama_prefill_layers_nf4_bf16", "srgpt_llama_prefill_chunk_layers_nf4_bf16",
               "srgpt_llama_verify_step_nf4_bf16"]


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_builds_export_the_new_entries(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.lib_path(elem)], capture_output=True, text=True, check=True).stdout
    for s in NEW_SYMBOLS:
        assert re.search(rf"\sT\s+{s}$", out, flags=re.M), s


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_new_kernels_fit_their_launch_bounds_without_local_memory(elem):
    """gemm_nf4_kernel: 384 threads, 1 CTA per SM (at most 168 registers); nf4_gemv_multi_kernel: 256 threads, 2 CTAs (128)."""
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    r = subprocess.run([cuda_tool("cuobjdump"), "--dump-resource-usage", _lib.lib_path(elem)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", r.stdout))
    gemm = {k: v for k, v in usage.items() if "gemm_nf4_kernel" in k}
    multi = {k: v for k, v in usage.items() if re.match(r"_ZN5srgpt4gemv21nf4_gemv_multi_kernelILi[0-2]ENS0_3Nf4EEEvNS0_7MParamsE", k)}
    assert len(gemm) == 6 and len(multi) == 3
    for group, cap in ((gemm, 168), (multi, 128)):
        for name, u in group.items():
            reg, stack, local = (int(re.search(f"{k}:(\\d+)", u).group(1)) for k in ("REG", "STACK", "LOCAL"))
            assert reg <= cap and stack == 0 and local == 0, (name, u)


def test_loader_validates_the_option_before_any_device_work():
    from spatialrgpt_b200 import builder
    from spatialrgpt_b200.weights import from_state_dicts
    for q in (None, "fp8"):
        with pytest.raises(ValueError, match="nf4_dequantized_copy"):
            from_state_dicts(None, {}, "cpu", quantization=q, nf4_dequantized_copy=False)
    with pytest.raises(ValueError, match="quantization"):
        from_state_dicts(None, {}, "cpu", quantization="int4")


@pytest.mark.parametrize("script", ["eval_spatial", "eval_region_cls"])
def test_eval_flag_needs_nf4(script, tmp_path):
    import importlib
    mod = importlib.import_module(f"spatialrgpt_b200.{script}")
    p = mod.build_arg_parser()
    args = p.parse_args(["--model-path", str(tmp_path), "--nf4-planes-only"])
    assert args.nf4_planes_only and args.quantization is None
    with pytest.raises(ValueError, match="--nf4-planes-only"):
        mod.eval_model(args, loader=lambda *a, **k: pytest.fail("the loader must not run"))
    seen = {}

    def loader(*a, **k):
        seen.update(k)
        raise RuntimeError("stop")
    with pytest.raises(RuntimeError, match="stop"):
        mod.eval_model(p.parse_args(["--model-path", str(tmp_path), "--quantization", "nf4", "--nf4-planes-only"]), loader=loader)
    assert seen["quantization"] == "nf4" and seen["nf4_dequantized_copy"] is False


def test_load_pretrained_model_validates_the_option_first(tmp_path):
    from spatialrgpt_b200 import builder
    for kw in ({}, {"quantization": "fp8"}):
        with pytest.raises(ValueError, match="nf4_dequantized_copy"):
            builder.load_pretrained_model(str(tmp_path), "x", None, nf4_dequantized_copy=False, **kw)
