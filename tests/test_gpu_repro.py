"""Run-to-run reproducibility of the default operator: the same inputs give the same bits.

The pairs kernel (bucket_mul_v4) fixes which rows each warp pair accumulates and in which order, and the row splits of a
column slice meet in a fixed order, so no result may depend on timing.  Both staging variants are checked: 4 (bulk
copies, the default) and 3 (16-byte cp.async)."""
import numpy as np
import pytest

from tests.test_gpu_parity import SHAPES
from tests.util import make_v, make_w

pytestmark = pytest.mark.gpu

_weights = {}


def _ew(in_dim, out_dim):
    import torch
    from effort_b200 import ops
    key = (in_dim, out_dim)
    if key not in _weights:
        g = ops.bucketize(torch.from_numpy(make_w(out_dim, in_dim, seed=1234)).cuda())
        _weights[key] = ops.ExpertWeights(g["buckets"], g["bucket.stats"], g["probes"], inDim=in_dim, outDim=out_dim)
    return _weights[key]


@pytest.mark.parametrize("stage", [4, 3])
@pytest.mark.parametrize("in_dim,out_dim", SHAPES)
def test_operator_same_bits_twice(in_dim, out_dim, stage):
    import torch
    from effort_b200 import ops
    ew = _ew(in_dim, out_dim)
    v = torch.from_numpy(make_v(in_dim, seed=9)).cuda()
    ctx = ops.default_context()
    try:
        ctx.setCutoffMode("select")
        ctx.setOption("stage", stage)
        for effort in (1.0, 0.25, 0.1):
            outs = []
            for _ in range(2):
                out = torch.full((out_dim,), 7.0, dtype=torch.float32, device="cuda")
                ops.bucketMul(v, ew, None, out, effort)
                torch.cuda.synchronize()
                outs.append(out.cpu().numpy())
            assert np.isfinite(outs[0]).all()
            assert outs[0].tobytes() == outs[1].tobytes(), (effort, int((outs[0] != outs[1]).sum()))
        assert ctx.errorFlag() == 0
    finally:
        ctx.setOption("stage", 4)


def test_decode_same_logits_twice():
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=2048, max_seq=64)
    m = DecodeModel.random_init(cfg, seed=7)
    runs = []
    for _ in range(2):
        m.reset()
        logits = []
        for t in (1, 17, 400, 999, 5, 1234):
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=0.25)
            torch.cuda.synchronize()
            logits.append(m.logits().cpu().numpy().copy())
        runs.append(logits)
    for k, (a, b) in enumerate(zip(*runs)):
        assert a.tobytes() == b.tobytes(), (k, float(np.abs(a - b).max()))
    assert ops.default_context().errorFlag() == 0
