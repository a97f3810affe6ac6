"""FP8 (E4M3) W8A8 quantization without a GPU: the CPU restatement (tests/fp8_ref.py) against hand-worked E4M3 values, the C-ABI argument
checks, the exports of both builds, the new kernels' SASS, and the combinations that raise."""
import ctypes as C
import re
import subprocess

import pytest
import torch

from tests import fp8_ref as R

NEW_SYMBOLS = ("srgpt_fp8_quantize_weight_bf16", "srgpt_fp8_quantize_act_bf16", "srgpt_gemm_fp8_bf16", "srgpt_llama_prefill_layers_fp8_bf16",
               "srgpt_llama_prefill_chunk_layers_fp8_bf16", "srgpt_llama_decode_step_fp8_bf16", "srgpt_gemv_fp8_bf16")


def test_e4m3_rounding_on_hand_worked_values():
    v = torch.tensor([448.0, 464.0, 470.0, 1000.0, -1000.0, 17.0, 19.0, 1.0, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, -2.0 ** -9, 0.0])
    # 448 = 1.75 * 2^8 is the largest finite code (0x7E; 0x7F is NaN); 464 is the tie above it and 470 / 1000 lie beyond: all saturate
    # to 448.  17 and 19 are ties (step 2 in [16, 32)) and go to the even mantissa: 16 (0x58) and 20 (0x5A).  2^-9 is the smallest
    # subnormal (0x01); 2^-10 ties between 0 and it and flushes to 0; 3 * 2^-10 ties between 2^-9 and 2^-8 and goes to 2^-8 (0x02).
    expect = [0x7E, 0x7E, 0x7E, 0x7E, 0xFE, 0x58, 0x5A, 0x38, 0x01, 0x00, 0x02, 0x81, 0x00]
    assert R.e4m3(v).tolist() == expect
    assert R.decode(torch.tensor(expect, dtype=torch.uint8)).tolist() == [448, 448, 448, 448, -448, 16, 20, 1, 2.0 ** -9, 0, 2.0 ** -8, -2.0 ** -9, 0]
    # the clamp matters: a plain cast turns an out-of-range value into NaN instead of saturating
    assert torch.isnan(torch.tensor([470.0]).to(torch.float8_e4m3fn).float()).all()


def test_row_quantizer_restatement():
    x = torch.tensor([[2.0, -1.0, 0.5, 0.0], [0.0, 0.0, 0.0, 0.0], [-3.0, 1.5, 2.0 ** -20, 0.75]])
    q, s = R.quantize_rows(x)
    # row 0: a = 2, inv = 224, s = 2 / 448; the maximum maps to 448 exactly
    assert s.tolist() == [torch.tensor(2.0 / 448.0).item(), 1.0, torch.tensor(3.0 / 448.0).item()]
    assert R.decode(q[0]).tolist() == [448.0, -224.0, 112.0, 0.0]
    assert q[1].tolist() == [0, 0, 0, 0]  # all-zero row: scale 1, codes 0
    assert R.decode(q[2]).tolist()[0] == -448.0 and q[2, 2].item() == 0  # 2^-20 * 448 / 3 is below half the smallest subnormal
    # the linear reproduces the unquantized product up to the E4M3 step (3 mantissa bits)
    w = torch.randn(5, 64, generator=torch.Generator().manual_seed(0))
    xa = torch.randn(3, 64, generator=torch.Generator().manual_seed(1))
    qw, sw = R.quantize_rows(w)
    y = R.linear(xa, qw, sw)
    assert (y - xa @ w.t()).abs().max() < 0.1 * (xa @ w.t()).abs().max()


def test_host_argument_validation_needs_no_gpu():
    from spatialrgpt_b200 import _lib
    lib = _lib.load()
    assert lib.srgpt_gemm_fp8_bf16(None, 16, None, None, 16, None, None, 16, 1, 1, 16, None, 0, 0, None) == -1
    assert "invalid argument" in _lib.last_error()
    # K must be a multiple of 16, strides 16-byte aligned, and only the three decoder epilogues exist
    p = 1 << 12
    assert lib.srgpt_gemm_fp8_bf16(p, 24, p, p, 24, p, p, 16, 1, 16, 24, None, 0, 0, None) == -1
    assert lib.srgpt_gemm_fp8_bf16(p, 32, p, p, 32, p, p, 16, 1, 16, 32, None, 0, 1, None) == -1  # EPI_BIAS
    assert lib.srgpt_fp8_quantize_act_bf16(p, 24, 1, 24, p, 32, p, None) == -1
    assert lib.srgpt_fp8_quantize_weight_bf16(p, 32, 1, 32, p, p, None, None) == -1  # n_bad is required
    assert lib.srgpt_llama_decode_step_fp8_bf16(None, None, 1, None, None, None, 16, 1, 1, 16, 16, 1e-5, *([None] * 4), 16, None, None, None, 16,
                                                *([None] * 6)) == -1
    # the FP8 GEMV: K a multiple of 16, an even N, 16-byte aligned codes
    from spatialrgpt_b200 import ops
    d = _lib.Fp8(p, p)
    assert lib.srgpt_gemv_fp8_bf16(p, C.byref(d), p + 4096, 8, 24, None, 0.0, None, 0, 0, 0, 0, *([None] * 5), 0, None) == -1
    assert lib.srgpt_gemv_fp8_bf16(p, C.byref(d), p + 4096, 7, 32, None, 0.0, None, 0, 0, 0, 0, *([None] * 5), 0, None) == -1
    assert lib.srgpt_gemv_fp8_bf16(p, C.byref(_lib.Fp8(p + 4, p)), p + 4096, 8, 32, None, 0.0, None, 0, 0, 0, 0, *([None] * 5), 0, None) == -1
    assert ops.GEMV_PLAIN == 0


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_builds_export_the_fp8_entry_points(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.lib_path(elem)], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\sT\s+(srgpt_[a-z0-9_]+)", out))
    assert set(NEW_SYMBOLS) <= exported and set(NEW_SYMBOLS) <= set(_lib.SIGNATURES)


def _functions(text):
    """cuobjdump output -> {mangled name: body text}."""
    parts = re.split(r"\n\s*Function : (\S+)\n", text)
    return {parts[i]: parts[i + 1] for i in range(1, len(parts) - 1, 2)}


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_fp8_kernels_use_e4m3_tensor_cores_and_no_local_memory(elem):
    from spatialrgpt_b200 import _lib
    _lib.load(elem=elem)
    path = _lib.lib_path(elem)
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True)
    res = subprocess.run(["cuobjdump", "-res-usage", path], capture_output=True, text=True)
    if sass.returncode != 0 or res.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    fns = _functions(sass.stdout)
    gemm = {n: b for n, b in fns.items() if "gemm_fp8_kernel" in n}
    # the three decoder epilogues (EPI_NONE, EPI_BIAS_RESIDUAL, EPI_SWIGLU), each whole-tile and stream-K
    assert sorted(re.search(r"ILi(\d)ELb(\d)", n).groups() for n in gemm) == [(e, s) for e in "045" for s in "01"]
    for body in gemm.values():
        assert "QGMMA.64x128x32.F32.E4M3.E4M3" in body and "UTMALDG" in body
    # the FP8 decode GEMV: its own kernel (not a decode_gemv_kernel format), one instantiation per mode, the staged x quantized in place
    # (cvt.rn.satfinite.e4m3x2.f32) and the weight codes turned into element-type chunks by cvt.e4m3x2 -> f16x2, 2 CTAs of 256 threads per SM
    gemv = {n: b for n, b in fns.items() if "fp8_gemv_kernel" in n}
    assert len(gemv) == 3 and not any("decode_gemv" in n for n in gemv)
    for body in gemv.values():
        assert "F2FP.F16.E4M3.UNPACK_B" in body and "F2FP.SATFINITE.E4M3.F32" in body and "HMMA" not in body
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", res.stdout))
    new = [n for n in usage if "gemm_fp8_kernel" in n or "fp820quantize_rows_kernel" in n or "fp8_gemv_kernel" in n]
    assert len(new) == 10
    for n in new:
        assert "LOCAL:0 " in usage[n] and "STACK:0 " in usage[n], (n, usage[n])
        if "fp8_gemv_kernel" in n:  # __launch_bounds__(256, 2): 2 CTAs per SM need <= 128 registers
            assert int(re.search(r"REG:(\d+)", usage[n]).group(1)) <= 128, usage[n]


def test_unsupported_combinations_raise():
    from spatialrgpt_b200 import ops
    from spatialrgpt_b200.config import LlamaDims
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    from spatialrgpt_b200.weights import LlamaW, from_state_dicts
    with pytest.raises(NotImplementedError, match="model.layers.0.mlp.down_proj.weight has 520"):
        ops.fp8_quantize_weight(torch.zeros(8, 520, dtype=torch.bfloat16), name="model.layers.0.mlp.down_proj.weight")
    with pytest.raises(ValueError, match="'fp8'"):
        from_state_dicts(None, {}, "cpu", quantization="int8")
    w = LlamaW(embed=torch.zeros(4, 4), norm=torch.zeros(4), lm_head=torch.zeros(4, 4), quantization="fp8")
    with pytest.raises(NotImplementedError, match="fp8"):
        TPLlamaDecoder(LlamaDims(), w, 0, 2)
