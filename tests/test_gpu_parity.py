"""GPU parity tests (run on an H100): every call goes through the C-ABI (effort_b200.ops -> ctypes ->
libeffort_b200.so) and is checked against the CPU oracle on the same seeded inputs.

Bars (SURVEY.md section 8c):
  convert     byte-exact                                  (deterministic)
  cutoff      hooks + "bisect" mode: bit-exact fp32 and the same loop count as the literal findCutoff32 bisection;
              "select" mode (the default of the fused operator): bit-exact vs oracle_select_cutoff, the exact order
              statistic the bisection approximates, and a probe count within the bisection's own +-2 slack
  selection   identical row set / identical dispatch list (ascending order here); the fused operator's selected-row
              count equals the oracle's in the same cutoff mode
  output      fp32 sum up to reordering: rel. L2 error <= 2e-6 vs the oracle's float64 sum of the same rows
              (the reference itself is order-nondeterministic, docs/gpu.html:196-198; the round-2 kernel adds its
              CTA sums into `out` with reductions, so its order is not fixed either), and cos-sim vs dense fp16 at
              the levels the reference claims.
Every operator test runs in both cutoff modes (fixture `mode`).
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests.util import make_v, make_w, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 2e-6


@pytest.fixture(scope="module")
def T():
    import torch
    return torch


@pytest.fixture(scope="module")
def ops():
    from effort_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _default_modes(ops):
    """default state of every test: the operator and the oracle both in the build's default cutoff mode"""
    ops.default_context().setCutoffMode("select")
    with O.cutoff_mode("select"):
        yield
    ops.default_context().setCutoffMode("select")
    assert ops.default_context().errorFlag() == 0


@pytest.fixture(params=["select", "bisect"])
def mode(request, ops):
    ops.default_context().setCutoffMode(request.param)
    with O.cutoff_mode(request.param):
        yield request.param


_conv_cache = {}


def conv(out_dim, in_dim, seed=1234):
    key = (out_dim, in_dim, seed)
    if key not in _conv_cache:
        w = make_w(out_dim, in_dim, seed)
        _conv_cache[key] = (w, O.bucketize(w))
    return _conv_cache[key]


def dev(T, a):
    return T.from_numpy(np.ascontiguousarray(a)).cuda()


def make_weights(T, ops, r, in_dim, out_dim, **kw):
    return ops.ExpertWeights(dev(T, r["buckets"]), dev(T, r["bucket.stats"]), dev(T, r["probes"]), inDim=in_dim,
                             outDim=out_dim, **kw)


# ---------------------------------------------------------------------------------------------------------
# convert
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dim,in_dim", [(4096, 4096), (1024, 4096), (11008, 4096), (4096, 14336)])
def test_bucketize_byte_exact(T, ops, out_dim, in_dim):
    w, r = conv(out_dim, in_dim)
    g = ops.bucketize(dev(T, w))
    T.cuda.synchronize()
    for k in ("buckets", "bucket.stats", "probes"):
        got = g[k].cpu().numpy().view(np.uint16)
        want = np.ascontiguousarray(r[k]).view(np.uint16)
        assert got.shape == want.shape, k
        assert np.array_equal(got, want), f"{k}: {np.count_nonzero(got != want)} words differ"


def test_bucketize_ties_and_zeros_byte_exact(T, ops):
    """ties in |w| (rule: lower output index first), +-0, denormals, a row of all-equal magnitudes"""
    rng = np.random.default_rng(9)
    w = make_w(4096, 4096, seed=77)
    w[:, 0] = np.float16(0.25) * np.where(rng.random(4096) < 0.5, 1, -1)
    w[:, 1] = 0
    w[::2, 1] = -0.0
    w[:, 2] = np.float16(6e-8)
    w[:64, 3] = w[64:128, 3]
    r = O.bucketize(w)
    g = ops.bucketize(dev(T, w))
    for k in ("buckets", "bucket.stats", "probes"):
        assert np.array_equal(g[k].cpu().numpy().view(np.uint16), np.ascontiguousarray(r[k]).view(np.uint16)), k


def test_bucketize_preconditions_return_errors(T, ops):
    from effort_b200 import EffortError
    with pytest.raises(EffortError):
        ops.bucketize(dev(T, make_w(4096, 2048)))
    with pytest.raises(EffortError):
        ops.bucketize(T.zeros((4096, 4096), dtype=T.float32, device="cuda"))


# ---------------------------------------------------------------------------------------------------------
# cutoff / dispatch hooks
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("effort", [1.0, 0.9, 0.75, 0.5, 0.3, 0.25, 0.1, 0.02, 0.0])
@pytest.mark.parametrize("seed", [42, 7])
def test_cutoff_bit_exact(T, ops, effort, seed):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = make_v(4096, seed)
    c, loops = ops.findCutoff(dev(T, v), ew, effort=effort)
    c_ref, loops_ref = O.find_cutoff(v, r["probes"], effort, return_loops=True)
    assert np.float32(c).view(np.uint32) == np.float32(c_ref).view(np.uint32), (c, c_ref)
    assert loops == loops_ref


def test_cutoff_edge_inputs(T, ops):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    cases = {
        "zeros": np.zeros(4096, np.float32),
        "ones": np.ones(4096, np.float32),
        "huge": make_v(4096, 3) * 1e4,          # every product >= 1000 -> the 999 -> 1000 sentinel path
        "tiny": make_v(4096, 4) * 1e-6,
        "one_hot": np.eye(1, 4096, 17, dtype=np.float32)[0] * 5,
    }
    for name, v in cases.items():
        for effort in (1.0, 0.25):
            c, loops = ops.findCutoff(dev(T, v), ew, effort=effort)
            c_ref, loops_ref = O.find_cutoff(v, r["probes"], effort, return_loops=True)
            assert np.float32(c).view(np.uint32) == np.float32(c_ref).view(np.uint32), (name, effort, c, c_ref)
            assert loops == loops_ref, (name, effort)


@pytest.mark.parametrize("effort", [1.0, 0.5, 0.25, 0.05])
def test_dispatch_list_identical(T, ops, effort):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = make_v(4096)
    ops.calcDispatch(dev(T, v), ew, effort=effort)
    d = ops.readDispatch(ew)
    c_ref = O.find_cutoff(v, r["probes"], effort)
    want = O.prepare_dispatch(v, r["bucket.stats"], c_ref, 4096, 256, 65536)
    n = want.shape[0]
    assert d["n_selected"] == n
    assert d["padded_size"] == (1 + n // 2048) * 2048            # roundUp, bucketMul.metal:22-31
    assert np.array_equal(d["dispatch"][:n].view(np.uint32), want.view(np.uint32))
    assert not d["dispatch"][n:].any()                            # zeroRange32 padding {0,0}


@pytest.mark.parametrize("effort", [1.0, 0.25])
def test_mul_hook_matches_oracle(T, ops, effort):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = make_v(4096)
    out = T.full((4096,), 7.0, dtype=T.float32, device="cuda")    # FP16 path overwrites (bucketMul.metal:133)
    ops.calcDispatch(dev(T, v), ew, effort=effort)
    ops.mul(ew, out)
    with O.cutoff_mode("bisect"):   # the hooks always run the reference's bisection
        res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 4096, 4096, effort)
    assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL


@pytest.mark.parametrize("effort", [1.0, 0.9, 0.75, 0.5, 0.3, 0.25, 0.1, 0.02, 0.0])
@pytest.mark.parametrize("seed", [42, 7])
def test_select_cutoff_exact_order_statistic(T, ops, effort, seed):
    """the fused operator's default cutoff: bit-equal to the oracle's (k+1)-th largest probe product; the number of
    products above it is within the slack the reference's own exit rule accepts (|count - k| < 3, bucketMul.metal:236)
    of the count the bisection ends with"""
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = make_v(4096, seed)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    ops.bucketMul(dev(T, v), ew, None, out, effort)
    c = ops.lastCutoff()
    c_ref = O.select_cutoff(v, r["probes"], effort)
    assert np.float32(c).view(np.uint32) == np.float32(c_ref).view(np.uint32), (c, c_ref)
    pv = O.probe_vals(v, r["probes"])
    k = 4096 - O.effort_to_q(effort)
    n_sel, n_bis = int((pv > c).sum()), int((pv > O.find_cutoff(v, r["probes"], effort)).sum())
    assert n_sel <= k
    assert abs(n_sel - n_bis) <= 3 or n_sel == k, (n_sel, n_bis, k)


def test_select_cutoff_edge_inputs(T, ops):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    cases = {
        "zeros": np.zeros(4096, np.float32),
        "ones": np.ones(4096, np.float32),
        "huge": make_v(4096, 3) * 1e4,
        "tiny": make_v(4096, 4) * 1e-6,
        "one_hot": np.eye(1, 4096, 17, dtype=np.float32)[0] * 5,
        "ties": np.sign(make_v(4096, 5)).astype(np.float32),
    }
    for name, v in cases.items():
        for effort in (1.0, 0.5, 0.25, 0.0):
            ops.bucketMul(dev(T, v), ew, None, out, effort)
            c, c_ref = ops.lastCutoff(), O.select_cutoff(v, r["probes"], effort)
            assert np.float32(c).view(np.uint32) == np.float32(c_ref).view(np.uint32), (name, effort, c, c_ref)
            res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 4096, 4096, effort)
            assert ops.lastSelected() == res["n_selected"], (name, effort)


# ---------------------------------------------------------------------------------------------------------
# the operator
# ---------------------------------------------------------------------------------------------------------
SHAPES = [(4096, 4096), (4096, 1024), (4096, 11008), (4096, 14336), (14336, 4096)]


@pytest.mark.parametrize("in_dim,out_dim", SHAPES)
@pytest.mark.parametrize("effort", [1.0, 0.5, 0.25, 0.1])
def test_bucket_mul_matches_oracle(T, ops, mode, in_dim, out_dim, effort):
    w, r = conv(out_dim, in_dim)
    ew = make_weights(T, ops, r, in_dim, out_dim)
    v = make_v(in_dim)
    out = T.full((out_dim,), -3.0, dtype=T.float32, device="cuda")
    ops.bucketMul(dev(T, v), ew, None, out, effort)
    n_sel = ops.lastSelected()
    res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], in_dim, out_dim, effort)
    assert n_sel == res["n_selected"]
    assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL
    # expertMul routes FP16 weights to bucketMul (expertMul.swift:32-33)
    out2 = T.zeros_like(out)
    ops.expertMul(dev(T, v), ew, None, out2, effort)
    assert rel_err(out2.cpu().numpy(), out.cpu().numpy()) <= 1e-6  # same rows; the CTA sums meet in `out` in any order


def test_no_repack_layout_same_selection_and_sum(T, ops):
    w, r = conv(4096, 4096)
    v = make_v(4096, 5)
    a = make_weights(T, ops, r, 4096, 4096)
    b = make_weights(T, ops, r, 4096, 4096, flags=ops.NO_REPACK)
    assert a.owned_bytes > 33_000_000 and b.owned_bytes < 1_000_000
    oa = T.empty(4096, dtype=T.float32, device="cuda")
    ob = T.empty_like(oa)
    ops.bucketMul(dev(T, v), a, None, oa, 0.3)
    na = ops.lastSelected()
    ops.bucketMul(dev(T, v), b, None, ob, 0.3)
    assert na == ops.lastSelected()
    assert rel_err(oa.cpu().numpy(), ob.cpu().numpy()) <= OUT_TOL


@pytest.mark.parametrize("in_dim,out_dim", [(4096, 4096), (4096, 1024), (4096, 11008), (14336, 4096)])
@pytest.mark.parametrize("stage,flags", [(0, 2), (2, 2), (3, 2), (4, 2), (0, 4), (3, 4)])
def test_layouts_and_bulk_stage(T, ops, mode, in_dim, out_dim, stage, flags):
    """device layouts (2 = slice-major: contiguous row sets per column slice, the default; 4 = input-major) x staging
    (3 = consumer/producer warp pairs, the default; 2 = one TMA producer warp + byte ring; 0 = self-serving warps with
    private cp.async rings): every combination computes the same operator (input-major weights always take stage 0)"""
    w, r = conv(out_dim, in_dim)
    v = make_v(in_dim, 5)
    ctx = ops.default_context()
    ew = make_weights(T, ops, r, in_dim, out_dim, flags=flags)
    out = T.full((out_dim,), 9.0, dtype=T.float32, device="cuda")
    try:
        ctx.setOption("stage", stage)
        for effort in (1.0, 0.25):
            ops.bucketMul(dev(T, v), ew, None, out, effort)
            res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], in_dim, out_dim, effort)
            assert ops.lastSelected() == res["n_selected"]
            assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL
    finally:
        ctx.setOption("stage", 3)


@pytest.mark.parametrize("opt,val", [("dynamic", 1), ("engine", 1)])
def test_engine_options_same_result(T, ops, opt, val):
    """static unit deal / the round-1 engine (fused kernel + integrate) against the oracle"""
    w, r = conv(4096, 14336)
    ew = make_weights(T, ops, r, 14336, 4096, flags=ops.INPUT_MAJOR)
    v = make_v(14336)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    ctx = ops.default_context()
    try:
        ctx.setOption(opt, val)
        ctx.setOption("stage", 0)
        if opt == "engine":   # the round-1 engine only knows the bisection
            ctx.setCutoffMode("bisect")
            O.set_cutoff_mode("bisect")
        ops.bucketMul(dev(T, v), ew, None, out, 0.25)
        res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 14336, 4096, 0.25)
        assert ops.lastSelected() == res["n_selected"]
        assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL
    finally:
        ctx.setOption(opt, 0 if opt == "dynamic" else 2)
        ctx.setOption("stage", 3)


def test_expert_number_selects_expert(T, ops, mode):
    """expNo is a DEVICE scalar read by the kernels (bucketMul.metal:49,143; runNetwork.swift:186-191)."""
    w0, r0 = conv(4096, 4096, seed=1234)
    w1, r1 = conv(4096, 4096, seed=99)
    cat = {k: np.concatenate([np.ascontiguousarray(r0[k]), np.ascontiguousarray(r1[k])]) for k in r0}
    ew = make_weights(T, ops, cat, 4096, 4096, numExperts=2)
    v = make_v(4096)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    for e, r in ((0, r0), (1, r1)):
        exp_no = T.tensor([e], dtype=T.int32, device="cuda")
        ops.bucketMul(dev(T, v), ew, exp_no, out, 0.25)
        res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 4096, 4096, 0.25)
        assert ops.lastSelected() == res["n_selected"]
        assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL


def test_percent_load_truncation(T, ops, mode):
    """loader.swift:113-166: only the first percentLoad ranks are loaded; expertSize = percentLoad*inSize."""
    w, r = conv(4096, 4096)
    P = 10
    rows = P * 4096
    cut = {"buckets": r["buckets"][:rows], "bucket.stats": r["bucket.stats"][:rows], "probes": r["probes"]}
    ew = make_weights(T, ops, cut, 4096, 4096, percentLoad=P)
    v = make_v(4096)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    ops.bucketMul(dev(T, v), ew, None, out, 0.9)
    res = O.bucket_mul(v, cut["buckets"], cut["bucket.stats"], cut["probes"], 4096, 4096, 0.9, expert_size=rows)
    assert ops.lastSelected() == res["n_selected"] <= rows
    assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL


def test_edge_vectors(T, ops, mode):
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    out = T.full((4096,), 1.0, dtype=T.float32, device="cuda")
    ops.bucketMul(T.zeros(4096, dtype=T.float32, device="cuda"), ew, None, out, 0.25)
    assert not out.any()                                           # nothing selected, out overwritten with 0
    v = np.zeros(4096, np.float32)
    v[123] = 2.5                                                   # a single active input dim
    ops.bucketMul(dev(T, v), ew, None, out, 1.0)
    res = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 4096, 4096, 1.0)
    assert ops.lastSelected() == res["n_selected"]
    assert rel_err(out.cpu().numpy(), res["out64"]) <= OUT_TOL


def test_batch_equals_sequential(T, ops):
    """q/k/v share v (runNetwork.swift:132-134); one launch group must equal three expertMul calls."""
    v = dev(T, make_v(4096))
    ws = [make_weights(T, ops, conv(o, 4096, seed=s)[1], 4096, o) for o, s in ((4096, 1), (1024, 2), (1024, 3))]
    outs_a = [T.empty(w.outSize, dtype=T.float32, device="cuda") for w in ws]
    outs_b = [T.empty_like(o) for o in outs_a]
    ops.expertMulBatch([(v, w, None, o, 0.25) for w, o in zip(ws, outs_a)])
    for w, o in zip(ws, outs_b):
        ops.expertMul(v, w, None, o, 0.25)
    for a, b in zip(outs_a, outs_b):   # same selection; the CTA split (hence the fp32 order) differs
        assert rel_err(a.cpu().numpy(), b.cpu().numpy()) <= OUT_TOL


def test_error_behaviour(T, ops):
    from effort_b200 import EffortError
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = dev(T, make_v(4096))
    out = T.empty(4096, dtype=T.float32, device="cuda")
    with pytest.raises(EffortError):
        ops.bucketMul(v, ew, None, out, 1.5)
    with pytest.raises(EffortError):
        ops.bucketMul(v.half(), ew, None, out, 0.25)
    with pytest.raises(EffortError):
        ops.bucketMul(v.cpu(), ew, None, out, 0.25)               # no CPU path
    with pytest.raises(EffortError):
        ops.bucketMul(v[:100], ew, None, out, 0.25)
    with pytest.raises(EffortError):
        ops.bucketMulQ4(v, ew, None, out, 0.25)                   # FP16 weights through the Q4 entry point
    with pytest.raises(EffortError):
        ops.mul(ew, out, ctx=ops.Context())                        # mul without calcDispatch


# ---------------------------------------------------------------------------------------------------------
# dense comparator + full-size properties
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dim,in_dim", [(4096, 4096), (32000, 4096), (4096, 14336)])
def test_basic_mul_matches_oracle(T, ops, out_dim, in_dim):
    w = make_w(out_dim, in_dim, seed=21)
    v = make_v(in_dim, seed=22)
    out = T.empty(out_dim, dtype=T.float32, device="cuda")
    ops.basicMul(dev(T, v), dev(T, w), out)
    _, want = O.basic_mul(v, w, cast_v=True)
    assert rel_err(out.cpu().numpy(), want) <= OUT_TOL


def test_config0_full_effort_vs_dense(T, ops):
    """BASELINE.json configs[0] on the GPU: 4096x4096 FP16 bucketMul at effort 1.0 vs dense GEMV."""
    w, r = conv(4096, 4096)
    ew = make_weights(T, ops, r, 4096, 4096)
    v = make_v(4096)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    ops.bucketMul(dev(T, v), ew, None, out, 1.0)
    dense = T.empty_like(out)
    ops.basicMul(dev(T, v), dev(T, w), dense)
    assert O.cossim(out.cpu().numpy(), dense.cpu().numpy()) >= 0.999


@pytest.mark.parametrize("in_dim,out_dim", [(4096, 14336), (14336, 4096)])
def test_full_size_cossim_and_monotone(T, ops, in_dim, out_dim):
    """size-independent properties at BASELINE's largest matrices: cos-sim vs dense rises with effort;
    selected rows rise with effort; halving v halves the output exactly-ish (linearity in v up to the 1e-5
    absolute give-up threshold of the bisection)."""
    w, r = conv(out_dim, in_dim)
    ew = make_weights(T, ops, r, in_dim, out_dim)
    v = make_v(in_dim)
    dense = T.empty(out_dim, dtype=T.float32, device="cuda")
    ops.basicMul(dev(T, v), dev(T, w), dense)
    d = dense.cpu().numpy()
    out = T.empty(out_dim, dtype=T.float32, device="cuda")
    prev_c, prev_n = -1.0, -1
    for effort in (0.1, 0.25, 0.5, 1.0):
        ops.bucketMul(dev(T, v), ew, None, out, effort)
        n = ops.lastSelected()
        c = O.cossim(out.cpu().numpy(), d)
        assert c >= prev_c - 1e-4 and n >= prev_n
        prev_c, prev_n = c, n
    assert prev_c >= 0.999
    ops.bucketMul(dev(T, v), ew, None, out, 0.25)
    a = out.cpu().numpy().copy()
    ops.bucketMul(dev(T, v * 0.5), ew, None, out, 0.25)
    assert rel_err(out.cpu().numpy() * 2.0, a) < 2e-2


# ---------------------------------------------------------------------------------------------------------
# Q4 (bucketMulQ4.swift / bucketMulQ4.metal; format of q4_draft.py pinned by tests/golden)
# ---------------------------------------------------------------------------------------------------------
_q4_cache = {}


def conv_q4(in_dim, out_dim, seed=31):
    key = (in_dim, out_dim, seed)
    if key not in _q4_cache:
        w = make_w(out_dim, in_dim, seed)                     # HF [out, in]
        t = O.q4_convert(np.ascontiguousarray(w.T))           # q4_convert.py:53 passes W^T
        _q4_cache[key] = (w, t)
    return _q4_cache[key]


def make_q4_weights(T, ops, w, t, in_dim, out_dim, with_buckets=True, with_core=True):
    if with_buckets:
        return ops.ExpertWeights(dev(T, t["buckets"]), dev(T, t["bucket.stats"]), dev(T, t["probes"]),
                                 dev(T, t["outliers"]), dev(T, w) if with_core else None, inDim=in_dim,
                                 outDim=out_dim, kind=ops.KIND_Q4)
    return ops.ExpertWeights(core=dev(T, w), inDim=in_dim, outDim=out_dim, kind=ops.KIND_Q4)


@pytest.mark.parametrize("in_dim,out_dim", [(4096, 4096), (4096, 14336)])
@pytest.mark.parametrize("effort", [1.0, 0.5, 0.25])
def test_q4_expert_mul_matches_oracle(T, ops, mode, in_dim, out_dim, effort):
    w, t = conv_q4(in_dim, out_dim)
    ew = make_q4_weights(T, ops, w, t, in_dim, out_dim)
    v = make_v(in_dim)
    out = T.full((out_dim,), 5.0, dtype=T.float32, device="cuda")   # expertMul zeroes it (expertMul.swift:27)
    ops.expertMul(dev(T, v), ew, None, out, effort)
    res = O.bucket_mul_q4(v, t["buckets"], t["bucket.stats"], t["probes"], t["outliers"], in_dim, out_dim, effort)
    assert ops.lastSelected() == res["n_selected"]
    assert rel_err(out.cpu().numpy(), res["out64"]) <= 5e-6
    # bucketMulQ4 itself accumulates into out (bucketMulQ4.metal:89)
    base = T.full((out_dim,), 1.0, dtype=T.float32, device="cuda")
    ops.bucketMulQ4(dev(T, v), ew, None, base, effort)
    assert rel_err(base.cpu().numpy() - 1.0, res["out64"]) <= 1e-4


def test_q4_dispatch_hook_and_payload(T, ops):
    w, t = conv_q4(4096, 4096)
    ew = make_q4_weights(T, ops, w, t, 4096, 4096)
    v = make_v(4096)
    ops.calcDispatch(dev(T, v), ew, effort=0.5)
    d = ops.readDispatch(ew)
    c_ref = O.find_cutoff(v, t["probes"], 0.5)   # hooks: the reference's bisection
    want = O.prepare_dispatch_q4(v, t["bucket.stats"], c_ref, 4096 // 32, 8 * 4096)
    assert d["n_selected"] == want.shape[0]
    assert np.array_equal(d["dispatch"][: want.shape[0]].view(np.uint32), want.view(np.uint32))
    out = T.zeros(4096, dtype=T.float32, device="cuda")
    ops.mul(ew, out)
    o32 = np.zeros(4096, np.float32)
    o64 = np.zeros(4096, np.float64)
    import ctypes as C
    O.lib().oracle_bucket_mul_q4_dispatch(np.ascontiguousarray(t["buckets"]).view(np.uint16).ctypes.data_as(C.POINTER(C.c_uint16)),
                                          want.ctypes.data_as(C.POINTER(C.c_float)), want.shape[0], 128,
                                          o32.ctypes.data_as(C.POINTER(C.c_float)), o64.ctypes.data_as(C.POINTER(C.c_double)))
    assert rel_err(out.cpu().numpy(), o64) <= 5e-6


def test_q4_routing_dense_fallback(T, ops):
    """expertMul.swift:26-31: Q4 weights whose buckets are not loaded (wk/wo/wv, q4_convert.py:53) use basicMul(core)."""
    w, t = conv_q4(4096, 4096)
    ew = make_q4_weights(T, ops, w, t, 4096, 4096, with_buckets=False)
    assert not ew.bucketsLoaded
    v = make_v(4096)
    out = T.empty(4096, dtype=T.float32, device="cuda")
    ops.expertMul(dev(T, v), ew, None, out, 0.25)
    _, want = O.basic_mul(v, w, cast_v=True)
    assert rel_err(out.cpu().numpy(), want) <= OUT_TOL
    q4 = make_q4_weights(T, ops, w, t, 4096, 4096)
    o2 = T.empty_like(out)
    ops.expertMul(dev(T, v), q4, None, o2, 1.0)
    assert O.cossim(o2.cpu().numpy(), want) > 0.9              # sign * row-average quantisation, 2 % outliers exact


# ---------------------------------------------------------------------------------------------------------
# tensor-parallel shards on the real kernels (ranks simulated one after the other on one GPU)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 8])
def test_tp_shards_reproduce_unsharded(T, ops, mode, world):
    from effort_b200 import sharding
    w, r = conv(4096, 4096)
    v = make_v(4096)
    full = O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], 4096, 4096, 0.25)
    vd = dev(T, v)
    col = np.zeros(4096, np.float32)
    row = np.zeros(4096, np.float64)
    n_row = 0
    for g in range(world):
        sc = sharding.shard_columns(r, 4096, 4096, g, world)
        ew = ops.ExpertWeights(dev(T, sc["buckets"]), dev(T, sc["bucket.stats"]), dev(T, sc["probes"]), inDim=4096,
                               outDim=sc["out"])
        out = T.empty(sc["out"], dtype=T.float32, device="cuda")
        ops.expertMul(vd, ew, None, out, 0.25)
        assert ops.lastSelected() == full["n_selected"]              # identical selection on every rank
        col[sc["out_offset"]: sc["out_offset"] + sc["out"]] = out.cpu().numpy()
        sr = sharding.shard_rows(r, 4096, 4096, g, world)
        ewr = ops.ExpertWeights(dev(T, sr["buckets"]), dev(T, sr["bucket.stats"]), dev(T, sr["probes"]),
                                inDim=sr["in"], outDim=4096)
        outr = T.empty(4096, dtype=T.float32, device="cuda")
        v_loc = dev(T, v[sr["in_offset"]: sr["in_offset"] + sr["in"]])
        ops.expertMulBatch([(v_loc, ewr, None, outr, 0.25, vd)])     # cutoff from the full vector's first 4096 dims
        n_row += ops.lastSelected()
        row += outr.cpu().numpy().astype(np.float64)                 # the all-reduce
    assert rel_err(col, full["out64"]) <= OUT_TOL
    assert n_row == full["n_selected"]
    assert rel_err(row, full["out64"]) <= OUT_TOL


def test_q4_convert_gpu_byte_exact(T):
    """effort_q4_bucketize vs the numpy restatement that is itself pinned to the reference's q4_draft.convert.
    The outlier choice at |w| ties on the 2 % boundary is unpinned (numpy's unstable argsort), so the kernel is
    checked on the oracle's outlier-zeroed matrix and the host-side outlier pick by its defining property."""
    from effort_b200 import convert
    for (inn, out, seed) in [(4096, 4096, 31), (64, 128, 11), (96, 4096 + 32, 12)]:
        w = make_w(out, inn, seed)
        core2 = np.ascontiguousarray(w.T)
        want = O.q4_convert(core2)
        zeroed = core2.copy()
        zeroed[want["outliers"][:, 1].astype(int), want["outliers"][:, 2].astype(int)] = 0
        got = convert.q4_bucketize(dev(T, zeroed))
        assert np.array_equal(got["buckets"].cpu().numpy().view(np.uint16), np.ascontiguousarray(want["buckets"]).view(np.uint16))
        assert np.array_equal(got["bucket.stats"].cpu().numpy(), want["bucket.stats"])
        assert np.array_equal(got["probes"].cpu().numpy().view(np.uint16), np.ascontiguousarray(want["probes"]).view(np.uint16))
        full = convert.q4_convert(dev(T, core2))
        go = full["outliers"].cpu().numpy()
        assert go.shape == want["outliers"].shape
        picked = np.zeros(core2.shape, bool)
        picked[go[:, 1].astype(int), go[:, 2].astype(int)] = True
        a = np.abs(core2.astype(np.float32))
        assert a[picked].min() >= a[~picked].max()                     # the top-2 % by |w|
