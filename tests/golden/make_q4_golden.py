"""Generates tests/golden/q4_golden_*.npz by running the REFERENCE's own Q4 converter
(q4_draft.py:70-322 of kolinko/effort, function convert) on small seeded matrices.

Needs a checkout of the reference; the tests read only the stored fixtures:
    python tests/golden/make_q4_golden.py <path to the reference's q4_draft.py>
q4_draft.convert reads a module-global `v` (q4_draft.py:209) that the reference never defines at
module level, so it is injected before the call.  Nothing is copied from the reference: the
fixtures hold only its INPUTS and OUTPUTS.
"""
import contextlib
import importlib.util
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
def load_ref(path):
    spec = importlib.util.spec_from_file_location("q4_draft_ref", path)
    mod = importlib.util.module_from_spec(spec)
    with contextlib.redirect_stdout(io.StringIO()):
        spec.loader.exec_module(mod)
    return mod


def main():
    ref = load_ref(sys.argv[1])
    for name, inn, out, seed in [("a", 64, 64, 11), ("b", 96, 128, 12), ("c", 32, 256, 13)]:
        rng = np.random.default_rng(seed)
        core2 = (rng.standard_normal((inn, out)) * 0.02).astype(np.float16)  # W^T [in, out]
        v = rng.standard_normal(inn).astype(np.float32)
        v[rng.integers(0, inn, size=max(1, inn // 50))] *= 10.0
        ref.v = v
        with contextlib.redirect_stdout(io.StringIO()):
            t = ref.convert(core2)
        np.savez_compressed(
            os.path.join(HERE, f"q4_golden_{name}.npz"),
            core2=core2.view(np.uint16), v=v,
            probes=np.asarray(t["probes"]).astype(np.float16).view(np.uint16),
            bucket_stats=np.asarray(t["bucket.stats"], dtype=np.float32),
            buckets=np.ascontiguousarray(t["buckets"]).view(np.uint16),
            outliers=np.asarray(t["outliers"], dtype=np.float32),
        )
        print(name, {k: (np.asarray(x).shape, np.asarray(x).dtype) for k, x in t.items()})


if __name__ == "__main__":
    sys.exit(main())
