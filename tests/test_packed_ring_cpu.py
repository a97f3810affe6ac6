"""The one-token decode GEMV (csrc/gemv.cu, DESIGN.md §4-5), checked without a GPU: every weight format keeps everything in
registers within the 3-CTAs-per-SM budget, the packed kernels contain the ring's waits, no kernel carries the rejected L2 bulk
prefetch, and the bf16 decode GEMV is pinned instruction for instruction."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "gemv_bf16_sass.json")
PACKED = r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-3]ENS0_8Packed12EEE"
BF16 = r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-3]ENS0_4Bf16EEE"
ONE_TOKEN = r"_ZN5srgpt4gemv18decode_gemv_kernelI"


def cuda_tool(name):
    path = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    if not os.path.exists(path):
        pytest.skip(f"{name} unavailable")
    return path


def sass_functions(path):
    """{mangled name: SASS text of the function} from `cuobjdump -sass`."""
    r = subprocess.run([cuda_tool("cuobjdump"), "-sass", path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    out = {}
    for f in re.split(r"\n\s*Function : ", r.stdout)[1:]:
        name, body = f.split("\n", 1)
        out[name.strip()] = body.split("\n\t\t..........")[0]
    return out


@pytest.fixture(scope="module")
def lib_path():
    from spatialrgpt_b200 import _lib
    _lib.load()
    return _lib.lib_path()


def one_token_kernels_fit_three_ctas_per_sm(path, n_packed):
    """4 bf16, n_packed packed and 3 NF4 instantiations of decode_gemv_kernel, each within 80 registers and without local memory."""
    r = subprocess.run([cuda_tool("cuobjdump"), "--dump-resource-usage", path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", r.stdout))
    kernels = {k: v for k, v in usage.items() if re.match(ONE_TOKEN, k)}
    assert len([k for k in kernels if re.match(PACKED, k)]) == n_packed, "one packed GEMV per mode (plain, SwiGLU, QKV + RoPE, lm_head)"
    assert len([k for k in kernels if re.match(BF16, k)]) == 4
    assert len(kernels) == 7 + n_packed, sorted(kernels)
    for name, u in kernels.items():
        reg, stack, local = (int(re.search(f"{k}:(\\d+)", u).group(1)) for k in ("REG", "STACK", "LOCAL"))
        # 80 registers x 256 threads x 3 CTAs fit the 64 K register file; 88 would leave 2 CTAs per SM
        assert reg <= 80 and stack == 0 and local == 0, (name, u)


def test_one_token_gemv_kernels_fit_three_ctas_per_sm_without_local_memory(lib_path):
    one_token_kernels_fit_three_ctas_per_sm(lib_path, 4)


def test_fp16_build_gemv_kernels_fit_three_ctas_per_sm_without_local_memory():
    """The fp16 build has the bf16 and NF4 kernels (computing in fp16), not the packed ones."""
    from spatialrgpt_b200 import _lib
    _lib.load(elem="f16")
    one_token_kernels_fit_three_ctas_per_sm(_lib.lib_path("f16"), 0)


def test_packed12_gemv_kernels_wait_on_the_ring(lib_path):
    funcs = sass_functions(lib_path)
    packed = [f for n, f in funcs.items() if re.match(PACKED, n)]
    assert len(packed) == 4
    for f in packed:
        assert "LDGSTS" in f and "STL" not in f and "LDL" not in f
        # cp.async.wait_group n for n = 0, 1: one per possible number of batches still in flight behind the one being read
        assert all(f"DEPBAR.LE SB0, 0x{n}" in f for n in range(2))


def test_no_decode_gemv_carries_an_l2_bulk_prefetch(lib_path):
    funcs = sass_functions(lib_path)
    gemvs = {n: f for n, f in funcs.items() if "decode_gemv" in n}
    assert len(gemvs) == 19  # 11 one-token kernels and 8 verify-pass kernels
    assert not [n for n, f in gemvs.items() if "UBLKPF" in f]


def test_bf16_format_gemv_sass_matches_the_golden_file(lib_path):
    """Every bf16 instantiation of decode_gemv_kernel is byte-identical to the SASS recorded in the golden file: a change to
    another weight format or to the host side must leave the bf16 kernels alone.  The golden file holds the sha256 of each
    function's text in `cuobjdump -sass` of libsrgpt_b200.so, split as sass_functions() does, built by _build.py with the nvcc
    release named there (another release schedules differently)."""
    golden = json.load(open(GOLDEN))
    v = subprocess.run([cuda_tool("nvcc"), "--version"], capture_output=True, text=True)
    if v.returncode != 0 or golden["nvcc"] not in v.stdout:
        pytest.skip(f"the golden SASS was produced by nvcc {golden['nvcc']}")
    funcs = sass_functions(lib_path)
    got = {n: hashlib.sha256(f.encode()).hexdigest() for n, f in funcs.items() if re.match(BF16, n)}
    assert sorted(got) == sorted(golden["sass_sha256"])
    for n, h in golden["sass_sha256"].items():
        assert got[n] == h, f"{n}: SASS differs from the recorded bf16 kernel"
