"""Static check of the compiled prefill kernels (no GPU needed: cuobjdump reads the in-tree .so): no spills to local
memory, and the multi-token GEMV runs on the CUDA cores (no tensor-core instruction), like the decode's GEMV."""
import os
import re
import shutil
import subprocess

import pytest

from effort_b200 import build as B

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
KERNELS = ["prefill_cutoff_kernel", "prefill_mul_kernel", "prefill_reduce_kernel", "prefill_embed_kernel",
           "prefill_rmsnorm_kernel", "chunk_attention_kernel", "prefill_head_kernel", "prefill_advance_kernel"]


def _run(args):
    return subprocess.run([CUOBJDUMP] + args + [B.LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def usage():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    B.build()
    recs = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", _run(["--dump-resource-usage"]))
    return {name: (int(reg), int(stack), int(local)) for name, reg, stack, _, local in recs}


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_spills(usage, kernel):
    hit = [n for n in usage if re.search(rf"\d{kernel}E", n)]
    assert len(hit) == 1, hit
    reg, stack, local = usage[hit[0]]
    assert local == 0, (kernel, usage[hit[0]])
    sass = _run(["-sass", "-fun", hit[0]])
    if kernel == "chunk_attention_kernel":
        # the only stack is sinf/cosf's slow-path argument reduction, as in the decode's attention_kernel
        dec = [v for n, v in usage.items() if re.search(r"\dattention_kernelE", n)]
        assert len(dec) == 1 and stack <= dec[0][1], (stack, dec)
    else:
        assert stack == 0 and "STL" not in sass and "LDL" not in sass, (kernel, usage[hit[0]])


def test_multi_gemv_uses_no_tensor_cores(usage):
    name = [n for n in usage if re.search(r"\dprefill_mul_kernelE", n)][0]
    sass = _run(["-sass", "-fun", name])
    assert "FFMA" in sass
    assert not re.search(r"\b(HMMA|IMMA|HGMMA|IGMMA|QGMMA|WGMMA|DMMA)\b", sass)
