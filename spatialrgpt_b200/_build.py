"""In-tree build of the sm_90a C-ABI library (libsrgpt_b200.so) with nvcc.

Used by ``__graft_entry__.build()`` and, lazily, by ``_lib.load()`` when the shared object is
missing or older than its sources.  nvcc cross-compiles without a GPU."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
INCLUDE = os.path.join(ROOT, "include")
BUILD_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(PKG_DIR, "libsrgpt_b200.so")
# the same sources compiled with IEEE half as the 16-bit element type (csrc/common.cuh): the reference loader's default dtype
# (llava/model/builder.py:62)
LIB_PATH_F16 = os.path.join(PKG_DIR, "libsrgpt_b200_f16.so")
VARIANTS = {"bf16": (LIB_PATH, []), "f16": (LIB_PATH_F16, ["-DSRGPT_ELEM_F16"])}

SOURCES = ["capi.cu", "gemm_wgmma.cu", "gemv.cu", "attention.cu", "attention_wgmma.cu", "attention_paged_wgmma.cu", "rowops.cu", "region.cu", "sampling.cu", "tp_comm.cu", "preprocess.cu", "layers.cu", "pack12.cu", "logits_process.cu", "nf4.cu", "fp8.cu", "beam.cu",
           "logprob.cu", "guidance.cu", "contrastive.cu", "attention_probs.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; cannot build libsrgpt_b200.so")
    return cand


def _deps():
    files = [os.path.join(CSRC, s) for s in SOURCES]
    files += [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "tma.cuh"), os.path.join(CSRC, "pack12.cuh"), os.path.join(CSRC, "nf4.cuh"), os.path.join(CSRC, "gemv_multi_kernel.inc"), os.path.join(CSRC, "fp8.cuh"),
              os.path.join(INCLUDE, "srgpt_b200.h")]
    return files


def is_stale() -> bool:
    for path, _ in VARIANTS.values():
        if not os.path.exists(path):
            return True
        t = os.path.getmtime(path)
        if any(os.path.getmtime(f) > t for f in _deps() if os.path.exists(f)):
            return True
    return False


def build(force: bool = False, verbose: bool = True) -> str:
    """Builds under an inter-process file lock: N eval workers started at once (scripts/srgpt_bench.sh) must not compile into
    the same object directory / link the same .so concurrently; the losers of the race find a fresh library and return."""
    if not force and not is_stale():
        return LIB_PATH
    import fcntl

    os.makedirs(BUILD_DIR, exist_ok=True)
    with open(os.path.join(BUILD_DIR, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():  # another process built it while we waited
                return LIB_PATH
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose: bool) -> str:
    nvcc = _nvcc()

    def compile_one(job):
        variant, src = job
        obj = os.path.join(BUILD_DIR, f"{variant}_" + src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, *VARIANTS[variant][1], "-I", INCLUDE, "-I", CSRC, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src} ({variant}):\n{r.stdout}\n{r.stderr}")
        return obj

    jobs = [(v, s) for v in VARIANTS for s in SOURCES]
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(compile_one, jobs))
    for vi, (variant, (path, _)) in enumerate(VARIANTS.items()):
        tmp = f"{path}.{os.getpid()}.tmp"
        cmd = [nvcc, "-shared", "--cudart", "shared", "-o", tmp, *objs[vi * len(SOURCES):(vi + 1) * len(SOURCES)],
               "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed ({variant}):\n{r.stdout}\n{r.stderr}")
        os.replace(tmp, path)
        if verbose:
            print(f"[srgpt_b200] built {path}", file=sys.stderr)
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
