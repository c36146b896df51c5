"""Static checks on the compiled sm_90a code of the hot kernels (no GPU needed: cuobjdump reads the in-tree .so).
They pin the properties DESIGN.md section 4 claims: no local-memory spills, the packed bf16 counting of the cutoff,
non-allocating streaming loads, no tensor-core instructions on this HBM-bound path."""
import re
import shutil
import subprocess

import pytest

from effort_b200 import build as B

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def _run(args):
    return subprocess.run([CUOBJDUMP] + args + [B.LIB], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def lib():
    import os
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    B.build()
    return B.LIB


def test_hot_kernels_do_not_spill(lib):
    usage = _run(["--dump-resource-usage"])
    recs = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    assert recs, "no resource usage parsed"
    hot = [r for r in recs if "bucket_mul_fused_kernel" in r[0] or "integrate_kernel" in r[0]]
    assert len(hot) >= 6           # FP16 / Q4 x plain / norm (+ ring variants) + integrate
    for name, reg, stack, _, local in hot:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        if "bucket_mul_fused_kernel" in name:
            assert int(reg) <= 128, (name, reg)   # 512 threads per CTA must fit the register file


def test_fused_kernel_instruction_selection(lib):
    names = [l.split()[-1].rstrip(":") for l in _run(["--dump-resource-usage"]).splitlines() if l.strip().startswith("Function")]
    main = [n for n in names if "bucket_mul_fused_kernelILi16ELi4ELi8ELi16ELb0ELi0E" in n]
    assert len(main) == 1, names
    sass = _run(["-sass", "-fun", main[0]])
    assert "HSET2.BF16_V2" in sass and "HADD2.BF16_V2" in sass      # cutoff: two products per compare / add
    assert len(re.findall(r"LDG\.E\.NA\.64\.CONSTANT", sass)) >= 16  # streaming: 8-byte no-allocate loads, 2 x U
    assert "BAR.SYNC.DEFER_BLOCKING 0x1, 0x80" in sass              # the four-warp named barrier of the cutoff
    assert not re.search(r"\b(HMMA|IMMA|UTCHMMA|UTCQMMA|QGMMA|HGMMA)\b", sass)   # no tensor cores on this path
    assert "STL" not in sass and "LDL" not in sass


def _fn(lib, pattern):
    names = [l.split()[-1].rstrip(":") for l in _run(["--dump-resource-usage"]).splitlines() if l.strip().startswith("Function")]
    hit = [n for n in names if pattern in n]
    assert len(hit) == 1, (pattern, hit)
    return hit[0]


def test_pairs_kernel_cp_async_variant(lib):
    """bucket_mul_v4_kernel<select, cp.async> ("pairs-ldgsts", stage 3): weights reach shared memory through LDGSTS
    (16-byte cp.async), completion through ARRIVES.LDGSTSBAR on an mbarrier, the consumer warps wait with
    SYNCS.PHASECHK, results leave as 16-byte vector reductions; no spills, no tensor-core instructions."""
    usage = _run(["--dump-resource-usage"])
    recs = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", usage)
    v4 = [r for r in recs if "bucket_mul_v4_kernel" in r[0]]
    assert len(v4) == 4            # select / bisect x cp.async / bulk
    for name, reg, stack, _, local in v4:
        assert int(stack) == 0 and int(local) == 0 and int(reg) <= 128, (name, reg, stack, local)
    sass = _run(["-sass", "-fun", _fn(lib, "bucket_mul_v4_kernelILi0ELb0")])
    assert "LDGSTS.E.BYPASS.128" in sass and "ARRIVES.LDGSTSBAR" in sass
    assert "SYNCS.PHASECHK.TRANS64.TRYWAIT" in sass and "SYNCS.ARRIVE.TRANS64" in sass
    assert "REDG.E.ADD.F32x4" in sass
    assert "HSET2.BF16_V2" in sass and "HADD2.BF16_V2" in sass      # the exact select counts two products per op
    assert not re.search(r"\b(HMMA|IMMA|UTCHMMA|UTCQMMA|QGMMA|HGMMA)\b", sass)
    assert "STL" not in sass and "LDL" not in sass


def test_default_kernel_streams_with_bulk_async_copies(lib):
    """bucket_mul_v4_kernel<select, bulk> -- the default path: one UBLKCP (cp.async.bulk) per unit, completion through the
    mbarrier's transaction count, 16-byte vector reductions into `out`, packed bf16 counting in the exact select"""
    sass = _run(["-sass", "-fun", _fn(lib, "bucket_mul_v4_kernelILi0ELb1")])
    assert "UBLKCP.S.G" in sass and "LDGSTS" not in sass
    assert "SYNCS.ARRIVE.TRANS64" in sass and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in sass
    assert "REDG.E.ADD.F32x4" in sass
    assert "HSET2.BF16_V2" in sass and "HADD2.BF16_V2" in sass
    assert not re.search(r"\b(HMMA|IMMA|UTCHMMA|UTCQMMA|QGMMA|HGMMA)\b", sass)
    assert "STL" not in sass and "LDL" not in sass
