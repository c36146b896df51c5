"""In-tree build of libeffort_b200.so (nvcc, sm_90a only: H100).  The .so is a build product and is git-ignored."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libeffort_b200.so")
SOURCES = ["effort_capi.cu", "safetensors_io.cpp"]
HEADERS = ["common.cuh", "cutoff.cuh", "bucket_mul.cuh", "bucket_mul_v2.cuh", "bucket_mul_v3.cuh", "bucket_mul_v4.cuh",
           "convert.cuh", "q4.cuh", "decode.cuh", "comm.cuh", "sample.cuh", "score.cuh", "prefill.cuh", "batch.cuh"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the effort_b200 CUDA extension cannot be built")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.join(HERE, "..", "include", "effort_b200.h")]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    extra = os.environ.get("EFFORT_NVCC_EXTRA", "").split()   # extra nvcc flags for A/B builds (tools/ab_op.py + EFFORT_LIB)
    cmd = [_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    host_cc = "/usr/bin/g++"
    if os.path.exists(host_cc):
        cmd += ["-ccbin", host_cc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
