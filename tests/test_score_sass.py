"""Static check of the compiled scorer (no GPU needed: cuobjdump reads the in-tree .so): score_kernel runs 1024 threads
in one CTA, so it must fit 64 registers without spilling to local memory."""
import os
import re
import shutil
import subprocess

import pytest

from effort_b200 import build as B

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def _run(args):
    return subprocess.run([CUOBJDUMP] + args + [B.LIB], capture_output=True, text=True, check=True).stdout


def test_score_kernel_does_not_spill():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    B.build()
    recs = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)",
                      _run(["--dump-resource-usage"]))
    hit = [r for r in recs if "score_kernel" in r[0]]
    assert len(hit) == 1, hit
    name, reg, stack, _, local = hit[0]
    assert int(stack) == 0 and int(local) == 0 and int(reg) <= 64, (name, reg, stack, local)
    sass = _run(["-sass", "-fun", name])
    assert "STL" not in sass and "LDL" not in sass
