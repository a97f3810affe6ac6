"""The packed decode GEMV's shared-memory ring (csrc/gemv.cu, DESIGN.md §5), checked without a GPU: the packed kernels keep
everything in registers within the 3-CTAs-per-SM budget and contain the ring's waits, and the bf16 decode GEMV is unchanged
instruction for instruction."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "gemv_bf16_sass.json")
PACKED = r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-3]ELi1ELb1EEE"
BF16 = r"_ZN5srgpt4gemv18decode_gemv_kernelILi[0-3]ELi[124]ELb0EEE"


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


def test_packed_gemv_kernels_fit_three_ctas_per_sm_without_local_memory(lib_path):
    r = subprocess.run([cuda_tool("cuobjdump"), "--dump-resource-usage", lib_path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", r.stdout))
    packed = {k: v for k, v in usage.items() if re.match(PACKED, k)}
    assert len(packed) == 4, "one packed GEMV per mode (plain, SwiGLU, QKV + RoPE, lm_head)"
    for name, u in packed.items():
        reg, stack, local = (int(re.search(f"{k}:(\\d+)", u).group(1)) for k in ("REG", "STACK", "LOCAL"))
        # 80 registers x 256 threads x 3 CTAs fit the 64 K register file; 88 would leave 2 CTAs per SM
        assert reg <= 80 and stack == 0 and local == 0, (name, u)


def test_packed_gemv_kernels_wait_on_the_ring(lib_path):
    funcs = sass_functions(lib_path)
    packed = [f for n, f in funcs.items() if re.match(PACKED, n)]
    assert len(packed) == 4
    for f in packed:
        assert "LDGSTS" in f and "STL" not in f and "LDL" not in f
        # cp.async.wait_group n for n = 0..3: one per possible number of batches still in flight behind the one being read
        assert all(f"DEPBAR.LE SB0, 0x{n}" in f for n in range(4))


def test_bf16_decode_gemv_sass_is_unchanged(lib_path):
    """The ring changes the packed kernels only: every bf16 instantiation of decode_gemv_kernel is byte-identical to the SASS
    recorded in the golden file (built by the nvcc release named there; another release schedules differently)."""
    golden = json.load(open(GOLDEN))
    v = subprocess.run([cuda_tool("nvcc"), "--version"], capture_output=True, text=True)
    if v.returncode != 0 or golden["nvcc"] not in v.stdout:
        pytest.skip(f"the golden SASS was produced by nvcc {golden['nvcc']}")
    funcs = sass_functions(lib_path)
    got = {n: hashlib.sha256(f.encode()).hexdigest() for n, f in funcs.items() if re.match(BF16, n)}
    assert sorted(got) == sorted(golden["sass_sha256"])
    for n, h in golden["sass_sha256"].items():
        assert got[n] == h, f"{n}: SASS differs from the recorded bf16 kernel"
