"""CPU checks of the batch decode (DESIGN.md section 4.9): the batch attention kernel keeps to attention_kernel's resources
(no local memory, no more stack than its sinf/cosf slow path), and every batch entry point refuses a NULL handle with
EFFORT_EINVAL without touching a device."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from effort_b200 import _lib
from effort_b200 import build as B

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
EINVAL = -1


@pytest.fixture(scope="module")
def usage():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    B.build()
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", B.LIB], capture_output=True, text=True, check=True).stdout
    recs = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", out)
    return {name: (int(reg), int(stack), int(local)) for name, reg, stack, _, local in recs}


def test_batch_attention_resources(usage):
    hit = [v for n, v in usage.items() if re.search(r"\dbatch_attention_kernelE", n)]
    dec = [v for n, v in usage.items() if re.search(r"\dattention_kernelE", n)]
    assert len(hit) == 1 and len(dec) == 1, (hit, dec)
    assert hit[0][2] == 0, hit
    assert hit[0][1] <= dec[0][1], (hit, dec)


def test_null_handles_are_refused():
    L = _lib.load()
    h = C.c_void_p()
    n = C.c_size_t(7)
    assert L.effort_batch_create(None, 4, C.byref(h)) == EINVAL and not h.value
    assert L.effort_batch_destroy(None) == EINVAL
    assert L.effort_batch_reset(None, -1, None) == EINVAL
    assert L.effort_batch_fork(None, -1, None) == EINVAL
    assert L.effort_batch_step(None, None, 0.25, None) == EINVAL
    assert L.effort_batch_set_sampler(None, 0, None) == EINVAL
    assert L.effort_batch_set_scoring(None, 1) == EINVAL
    assert L.effort_batch_set_score_targets(None, 0, None, 0, None) == EINVAL
    assert L.effort_batch_logits(None) is None
    assert L.effort_batch_next_tokens(None) is None
    assert L.effort_batch_scores(None) is None
    assert L.effort_batch_buffer(None, 0, 0, 0, C.byref(n)) is None and n.value == 0
