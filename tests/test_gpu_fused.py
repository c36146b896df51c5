"""GPU: the fused decode chain's launch groups (effort_fused_mul_batch) against the oracle, one group at a time, with the
glue each group applies on load: rmsNorm(h) * w ([q,k,v], [w1,w3]), silu(x1) * x3 (w2), accumulation into a residual
stream that already holds a value (wo, w2, [q,k,v] and the dense [w1,w3]), and the routed experts (device expNo, and the
gate value as a device out_scale on w2).  Every group runs at the chain's shapes, in both cutoff modes, on every
staging variant (stage 4 = warp pairs fed by bulk copies, the default; 3 = the pairs with cp.async; 2 = one TMA
producer warp; 0 = per-warp cp.async rings), at efforts 1.0, 0.5, 0.25 and 0.1.

Bars (measured maxima over the file in brackets as error / bar, on an H100 80GB HBM3 at 700 W):
  grid inputs (tests/fused_ref.py: the glue is bit-exact in any summation order) and edge inputs:
      cutoff fp32-bit-equal to the oracle's on the restated input, selected rows equal, and
      |out - (prior + s * out64)| <= 2e-6 * |s * out64| + 2^-24 * |prior + s * out64|  (L2 norms: the operator bar plus
      one fp32 rounding of the final add; overwrite calls have no prior and start from NaN)     [grid 0.28, edge 0.275]
  realistic inputs:
      norm groups: the kernel's fp32 sum of squares may give a denominator a few ulps off the float64 one, so the oracle
      runs on d0 + {0, +-1, +-2} ulps; cutoff and count must equal one candidate's and the output meet the bar against it
      [0.111; the matching candidate was up to 2 ulps off d0]
      silu groups, plain wo: the grid bars unchanged (expf may differ from numpy's exp in the last ulp; no wider bar was
      needed)                                                                                    [silu 0.284, wo 0.129]
  edges: h = 0 (out exactly the prior, or exactly 0), one-hot h, the wo input and x3 x1e4 (the bisection's 999 -> 1000
      sentinel), x1 <= -90 everywhere (nothing selected)
  hint / prefetch: byte-identical outputs; with the hint a repeated norm call selects in <= 3 rounds, 8 from scratch
  chain: replaying a 1-layer dense and a 1-layer MoE model's step through the hook, from the model's own buffers, gives
      q/k/v, the post-wo h (MoE) and the final h byte for byte on the bit-reproducible stages 4 and 3; on stages 2 and 0
      (atomic CTA sums) q/k/v and the post-wo h within the operator bar"""
import numpy as np
import pytest

from oracle import oracle as O
from tests import fused_ref as F
from tests.util import make_v

pytestmark = pytest.mark.gpu

OUT_TOL = 2e-6
EPS = 1e-5
STAGES = (4, 3, 2, 0)
EFFORTS = (1.0, 0.5, 0.25, 0.1)
SCALE = float(np.float32(0.37))
HID = 14336
N_EXP = 4
CASES = ["qkv", "w13", "wo", "w2", "moe_w13-1", "moe_w13-3", "moe_w2-1", "moe_w2-3"]
REPORT = {}   # worst error / bar ratio per tier, printed by the last test


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def T():
    import torch
    return torch


@pytest.fixture(scope="module")
def ops():
    from effort_b200 import ops as _ops
    return _ops


def _defaults(ctx):
    ctx.setCutoffMode("select")
    ctx.setOption("stage", 4)
    ctx.setOption("hint", 1)
    ctx.setOption("prefetch", 0)


@pytest.fixture(autouse=True)
def _default_modes(ops):
    _defaults(ops.default_context())
    with O.cutoff_mode("select"):
        yield
    _defaults(ops.default_context())
    assert ops.default_context().errorFlag() == 0


@pytest.fixture(params=["select", "bisect"])
def mode(request, ops):
    ops.default_context().setCutoffMode(request.param)
    with O.cutoff_mode(request.param):
        yield request.param


class Mat:
    """one weight handle (n_experts experts) and the host copy of its reference-layout tensors for the oracle"""

    def __init__(self, ops, t, in_dim, out_dim, n_exp=1):
        self.ew = ops.ExpertWeights(t["buckets"], t["bucket.stats"], t["probes"], inDim=in_dim, outDim=out_dim,
                                    numExperts=n_exp)
        self.host = {k: t[k].cpu().numpy() for k in t}
        self.inn, self.out = in_dim, out_dim

    def oracle(self, x, effort, exp_no=0):
        h = self.host
        return O.bucket_mul(x, h["buckets"], h["bucket.stats"], h["probes"], self.inn, self.out, effort, exp_no=exp_no)


@pytest.fixture(scope="module")
def W(T, ops):
    """the chain's matrices, converted with ops.bucketize: q/k/v/o, and w1/w2/w3 with 4 experts whose expert 0 also
    serves as the dense layer's matrix"""
    gen = T.Generator(device="cuda").manual_seed(2026)

    def conv(out_dim, in_dim, n_exp=1):
        ts = [ops.bucketize((T.randn((out_dim, in_dim), generator=gen, device="cuda") * 0.02).half()) for _ in range(n_exp)]
        return {k: T.cat([x[k] for x in ts]) for k in ts[0]}

    def first(t, in_dim):
        return {"buckets": t["buckets"][: 16 * in_dim], "bucket.stats": t["bucket.stats"][: 16 * in_dim],
                "probes": t["probes"][:4096]}

    m = {"wq": Mat(ops, conv(4096, 4096), 4096, 4096), "wk": Mat(ops, conv(1024, 4096), 4096, 1024),
         "wv": Mat(ops, conv(1024, 4096), 4096, 1024), "wo": Mat(ops, conv(4096, 4096), 4096, 4096)}
    for name, (o, i) in (("w1", (HID, 4096)), ("w3", (HID, 4096)), ("w2", (4096, HID))):
        t = conv(o, i, N_EXP)
        m[name + "e"] = Mat(ops, t, i, o, N_EXP)
        m[name] = Mat(ops, first(t, i), i, o)
    gen2 = np.random.default_rng(7)
    m["attn_norm"] = (1.0 + 0.1 * gen2.standard_normal(4096)).astype(np.float16)
    m["ffn_norm"] = (1.0 + 0.1 * gen2.standard_normal(4096)).astype(np.float16)
    T.cuda.synchronize()
    return m


def _case(name):
    """(matrix names, glue, expert or None, out_scale or None, accumulate)"""
    base, _, e = name.partition("-")
    return {"qkv": (["wq", "wk", "wv"], "norm", None, None, True),
            "w13": (["w1", "w3"], "norm", None, None, True),
            "wo": (["wo"], "plain", None, None, True),
            "w2": (["w2"], "silu", None, None, True),
            "moe_w13": (["w1e", "w3e"], "norm", int(e or 0), None, False),
            "moe_w2": (["w2e"], "silu", int(e or 0), SCALE, True)}[base]


def _inputs(name, variant, seed=11):
    """host inputs of one case: dict(v[, x3][, norm]) by variant"""
    names, glue, *_ = _case(name)
    rng = np.random.default_rng(seed)
    if glue == "norm":
        h = {"grid": lambda: F.grid_h(seed), "real": lambda: make_v(4096, seed), "zero": lambda: np.zeros(4096, np.float32),
             "onehot": lambda: np.eye(1, 4096, 17, dtype=np.float32)[0] * 5}[variant]()
        return {"v": h, "norm": "attn_norm" if names[0] == "wq" else "ffn_norm"}
    if glue == "plain":
        v = {"grid": lambda: make_v(4096, seed), "real": lambda: make_v(4096, seed + 1), "zero": lambda: np.zeros(4096, np.float32),
             "onehot": lambda: np.eye(1, 4096, 17, dtype=np.float32)[0] * 5, "huge": lambda: make_v(4096, seed) * 1e4}[variant]()
        return {"v": v.astype(np.float32)}
    x3 = rng.standard_normal(HID).astype(np.float32)
    if variant == "real":
        return {"v": (rng.standard_normal(HID) * 2).astype(np.float32), "x3": x3}
    x1 = F.grid_x1(seed, HID)
    if variant == "neg":
        x1 = -np.abs(x1) - np.float32(90)
    if variant == "huge":
        x3 = (x3 * 1e4).astype(np.float32)
    return {"v": x1, "x3": x3}


def _restated(inp, W, denom=None):
    if "norm" in inp:
        return F.norm_input(inp["v"], W[inp["norm"]], EPS, denom)
    if "x3" in inp:
        return F.silu_input(inp["v"], inp["x3"])
    return inp["v"]


_memo = {}


def _ref(W, name, slot, x_key, x, mode, effort):
    """oracle result of one slot on the restated input x (memoised per case, slot, input, mode and effort)"""
    key = (name, slot, x_key, mode, effort)
    if key not in _memo:
        names, _, exp, _, _ = _case(name)
        _memo[key] = W[names[slot]].oracle(x, effort, exp or 0)
    return _memo[key]


def _prior(name, slot, n, scale_like):
    rng = np.random.default_rng(1000 + 10 * CASES.index(name) + slot)
    return (rng.standard_normal(n) * max(scale_like, 1e-3)).astype(np.float32)


def _launch(T, ops, W, name, inp, effort, priors):
    """one launch group through the hook; returns [(out, cutoff, n_selected)] per slot"""
    names, glue, exp, scale, acc = _case(name)
    dev = {k: T.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in inp.items() if k != "norm"}
    nw = T.from_numpy(W[inp["norm"]]).cuda() if "norm" in inp else None
    e = T.tensor([exp], dtype=T.int32, device="cuda") if exp is not None else None
    s = T.tensor([scale], dtype=T.float32, device="cuda") if scale is not None else None
    outs, calls = [], []
    for k, n in enumerate(names):
        m = W[n]
        out = T.from_numpy(priors[k].copy()).cuda() if acc else T.full((m.out,), float("nan"), dtype=T.float32, device="cuda")
        outs.append(out)
        calls.append(dict(v=dev["v"], by=m.ew, out=out, effort=effort, x3=dev.get("x3"), norm=nw, eps=EPS, expNo=e,
                          scale=s, accumulate=acc))
    ops.fusedMulBatch(calls)
    probs = [ops.lastProblem(k) for k in range(len(names))]
    return [(o.cpu().numpy(), c, n) for o, (c, n) in zip(outs, probs)]


def _out_err(got, ref, prior, scale):
    """error / bar of one slot's output (<= 1 passes)"""
    s = 1.0 if scale is None else scale
    want = s * ref["out64"] + (0.0 if prior is None else prior.astype(np.float64))
    if not np.isfinite(got).all():
        return np.inf
    bar = OUT_TOL * np.linalg.norm(s * ref["out64"]) + 2.0 ** -24 * np.linalg.norm(want)
    err = np.linalg.norm(got.astype(np.float64) - want)
    return 0.0 if err == 0 else err / max(bar, 1e-30)


def _note(tier, ratio):
    REPORT[tier] = max(REPORT.get(tier, 0.0), ratio)


def _run_exact(T, ops, W, name, variant, mode, effort, tier):
    """one launch on an input whose glue is exact: every slot bit-exact cutoff, equal count, output within the bar"""
    names, glue, exp, scale, acc = _case(name)
    inp = _inputs(name, variant)
    x = _restated(inp, W)
    refs = [_ref(W, name, k, variant, x, mode, effort) for k in range(len(names))]
    priors = [_prior(name, k, W[n].out, float(np.std(r["out64"]))) if acc else None for k, (n, r) in enumerate(zip(names, refs))]
    got = _launch(T, ops, W, name, inp, effort, priors)
    for k, ((out, c, n), r) in enumerate(zip(got, refs)):
        what = (name, variant, mode, effort, names[k])
        assert _bits(c) == _bits(r["cutoff"]), (what, c, r["cutoff"])
        assert n == r["n_selected"], (what, n, r["n_selected"])
        ratio = _out_err(out, r, priors[k], scale)
        _note(tier, ratio)
        assert ratio <= 1.0, (what, ratio)
        if r["n_selected"] == 0:   # nothing selected: out is exactly the prior, or exactly zero
            assert np.array_equal(_bits(out), _bits(priors[k])) if acc else not out.any(), what
    return got


@pytest.mark.parametrize("stage", STAGES)
@pytest.mark.parametrize("name", CASES)
def test_grid_inputs_match_oracle(T, ops, W, mode, name, stage):
    ops.default_context().setOption("stage", stage)
    for effort in EFFORTS:
        _run_exact(T, ops, W, name, "grid", mode, effort, "grid")


@pytest.mark.parametrize("name", CASES)
def test_edge_inputs_match_oracle(T, ops, W, mode, name):
    glue = _case(name)[1]
    variants = {"norm": ["zero", "onehot"], "plain": ["zero", "onehot", "huge"], "silu": ["huge", "neg"]}[glue]
    for stage in STAGES:
        ops.default_context().setOption("stage", stage)
        for variant in variants:
            for effort in (1.0, 0.25):
                got = _run_exact(T, ops, W, name, variant, mode, effort, "edge")
                if variant in ("zero", "neg"):
                    assert all(n == 0 for _, _, n in got), (name, variant)


@pytest.mark.parametrize("stage", STAGES)
@pytest.mark.parametrize("name", CASES)
def test_realistic_inputs_match_oracle(T, ops, W, mode, name, stage):
    names, glue, exp, scale, acc = _case(name)
    ops.default_context().setOption("stage", stage)
    if glue != "norm":
        for effort in EFFORTS:
            _run_exact(T, ops, W, name, "real", mode, effort, "real " + glue)
        return
    inp = _inputs(name, "real")
    d0 = F.norm_denom(inp["v"], EPS)
    cands = [F.ulp_step(d0, u) for u in (0, -1, 1, -2, 2)]
    for effort in EFFORTS:
        base = [_ref(W, name, k, ("real", 0), _restated(inp, W, cands[0]), mode, effort) for k in range(len(names))]
        priors = [_prior(name, k, W[n].out, float(np.std(r["out64"]))) if acc else None for k, (n, r) in enumerate(zip(names, base))]
        got = _launch(T, ops, W, name, inp, effort, priors)
        for k, (out, c, n) in enumerate(got):
            best = np.inf
            for u, d in zip((0, -1, 1, -2, 2), cands):
                r = _ref(W, name, k, ("real", u), _restated(inp, W, d), mode, effort)
                if _bits(c) == _bits(r["cutoff"]) and n == r["n_selected"]:
                    best = min(best, _out_err(out, r, priors[k], scale))
                    if u:
                        _note("real norm: denominator off d0", abs(u))
            _note("real norm", best)
            assert best <= 1.0, (name, mode, effort, names[k], c, n, best)


def _group_outputs(T, ops, W, name, variant="real", effort=0.25):
    names, _, _, _, acc = _case(name)
    priors = [np.zeros(W[n].out, np.float32) for n in names] if acc else None
    return [_bits(o).copy() for o, _, _ in _launch(T, ops, W, name, _inputs(name, variant), effort, priors)]


@pytest.mark.parametrize("name", ["qkv", "w13", "w2", "moe_w13-3", "moe_w2-1"])
def test_hint_and_prefetch_do_not_change_the_result(T, ops, W, mode, name):
    """bucket_mul_v4's select starts from the matrix's last cutoff (kVNorm: stored times that call's denominator) and may
    prefetch the rows that cutoff selects; neither may change a bit of the result"""
    ctx = ops.default_context()
    for stage in (4, 3):
        ctx.setOption("stage", stage)
        outs = {}
        for hint in (0, 1):
            for pf in (0, 1):
                ctx.setOption("hint", hint)
                ctx.setOption("prefetch", pf)
                for effort in (0.5, 0.25):
                    outs[(hint, pf, effort)] = _group_outputs(T, ops, W, name, effort=effort)
        for (hint, pf, effort), o in outs.items():
            for a, b in zip(o, outs[(0, 0, effort)]):
                assert np.array_equal(a, b), (name, stage, hint, pf, effort)


def _loops(ops):
    import ctypes as C
    ctx = ops.default_context()
    loops = C.c_int(0)
    from effort_b200._lib import check
    check(ctx._L.effort_read_dispatch(ctx._h, None, 0, None, None, None, C.byref(loops), ops._stream_ptr()), "read")
    return int(loops.value)


def test_hint_round_trip_saves_select_rounds(T, ops, W):
    """select mode, norm group: the hint stored as cutoff x denominator and read back / denominator must land on the same
    key, so a repeated identical call brackets the cutoff in its first round"""
    ctx = ops.default_context()
    for name in ("qkv", "w13"):
        for effort in (0.5, 0.25, 0.1):
            ctx.setOption("hint", 0)
            a = _group_outputs(T, ops, W, name, effort=effort)
            scratch = _loops(ops)
            ctx.setOption("hint", 1)
            _group_outputs(T, ops, W, name, effort=effort)
            b = _group_outputs(T, ops, W, name, effort=effort)
            hinted = _loops(ops)
            assert scratch == 8 and hinted <= 3, (name, effort, scratch, hinted)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
            _note("select rounds with the hint", hinted)


def test_hook_validation(T, ops, W):
    from effort_b200 import EffortError
    ctx = ops.default_context()
    h = T.zeros(4096, dtype=T.float32, device="cuda")
    x = T.zeros(HID, dtype=T.float32, device="cuda")
    nw = T.from_numpy(W["attn_norm"]).cuda()
    out = T.zeros(4096, dtype=T.float32, device="cuda")
    ok = dict(v=h, by=W["wq"].ew, out=out, effort=0.25, norm=nw)
    ops.fusedMulBatch([ok])
    with pytest.raises(EffortError):
        ops.fusedMulBatch([dict(ok, x3=h)])                                     # norm and silu together
    with pytest.raises(EffortError):
        ops.fusedMulBatch([dict(v=x, by=W["w2"].ew, out=out, effort=0.25, norm=nw)])   # norm needs in == 4096
    with pytest.raises(EffortError):
        ops.fusedMulBatch([dict(ok, effort=1.5)])
    with pytest.raises(EffortError):
        ops.fusedMulBatch([ok] * 5)                                             # more than one launch group holds
    core = (T.randn((4096, 4096), device="cuda") * 0.02).half()
    q4 = ops.ExpertWeights(core=core, inDim=4096, outDim=4096, kind=ops.KIND_Q4)
    with pytest.raises(EffortError):
        ops.fusedMulBatch([dict(v=h, by=q4, out=out, effort=0.25)])             # not FP16 buckets
    ops.fusedMulBatch([ok, ok])
    assert ops.lastProblem(1)[1] == 0
    with pytest.raises(EffortError):
        ops.lastProblem(2)                                                      # no such slot in the last group
    try:
        ctx.setOption("engine", 1)
        with pytest.raises(EffortError):
            ops.fusedMulBatch([ok])
    finally:
        ctx.setOption("engine", 2)


def _replay(T, ops, m, token, effort, moe, exact):
    """the step's layer 0 through the hook from the model's own buffers; returns the buffers the replay missed.  exact:
    byte equality.  Otherwise (stages 2 and 0 add their CTA sums with atomics, in an order that changes from run to run)
    q/k/v and the post-wo h within the operator bar; each of these GEMVs gets the same input as in the step, so the same
    rows, but the later ones would not, so the final h is left to the bit-reproducible stages."""
    L = m.layers[0]
    wq, wk, wv, wo, w1, w2, w3, attn_norm, ffn_norm = L[:9]
    eps = m.cfg.norm_eps
    bad = []

    def same(name, mine):
        want = m.buffer(name)
        ok = T.equal(mine.view(T.int32), want.view(T.int32)) if exact else \
            float((mine.double() - want.double()).norm()) <= OUT_TOL * float(want.double().norm())
        if not ok:
            bad.append(name)

    h = m.head[2][token].float()
    q, k, v = (T.zeros(w.outSize, dtype=T.float32, device="cuda") for w in (wq, wk, wv))
    ops.fusedMulBatch([dict(v=h, by=w, out=o, effort=effort, norm=attn_norm, eps=eps, accumulate=True)
                       for w, o in ((wq, q), (wk, k), (wv, v))])
    for name, mine in (("Q", q), ("K", k), ("V", v)):
        same(name, mine)
    h = h.clone()
    ops.fusedMulBatch([dict(v=m.buffer("ATTN"), by=wo, out=h, effort=effort, accumulate=True)])
    if moe:
        same("GATE_IN", h)
        if not exact:
            return bad
        idx, val = m.buffer("GATE_IDX"), m.buffer("GATE_VAL")
        hk = h.clone()
        for r in range(2):
            x1, x3 = (T.full((w1.outSize,), float("nan"), device="cuda") for _ in range(2))
            ops.fusedMulBatch([dict(v=hk, by=w, out=o, effort=effort, norm=ffn_norm, eps=eps, expNo=idx[r:r + 1])
                               for w, o in ((w1, x1), (w3, x3))])
            ops.fusedMulBatch([dict(v=x1, x3=x3, by=w2, out=h, effort=effort, expNo=idx[r:r + 1], scale=val[r:r + 1],
                                    accumulate=True)])
    else:
        if not exact:
            return bad
        x1, x3 = (T.zeros(w1.outSize, dtype=T.float32, device="cuda") for _ in range(2))
        ops.fusedMulBatch([dict(v=h, by=w, out=o, effort=effort, norm=ffn_norm, eps=eps, accumulate=True)
                           for w, o in ((w1, x1), (w3, x3))])
        ops.fusedMulBatch([dict(v=x1, x3=x3, by=w2, out=h, effort=effort, accumulate=True)])
    same("HIDDEN", h)
    return bad


@pytest.mark.parametrize("moe", [False, True], ids=["dense", "moe"])
def test_hook_is_the_chain(T, ops, mode, moe):
    """the hook runs what model_enqueue_token_v2 runs: eager steps (a captured graph keeps the stage and mode it was
    captured with) of a 1-layer model in every cutoff mode x stage, replayed through the hook"""
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=1, vocab=1024, max_seq=32)
    m = DecodeModel.random_init_moe(cfg, n_experts=N_EXP, seed=91) if moe else DecodeModel.random_init(cfg, seed=90)
    m.set_graphs(False)
    ctx = ops.default_context()
    for stage in STAGES:
        ctx.setOption("stage", stage)
        for effort in (1.0, 0.25):
            m.reset()
            for t in (3, 77, 500):
                m.step(T.tensor([t], dtype=T.int32, device="cuda"), effort=effort)
                T.cuda.synchronize()
                bad = _replay(T, ops, m, t, effort, moe, exact=stage in (4, 3))
                assert not bad, (mode, stage, effort, t, bad)
                assert m.buffer("NORMED") is None   # the fused chain ran
    assert ctx.errorFlag() == 0


def test_zz_report():
    """the measured maxima of the bars above (error / bar, 1 = at the bar)"""
    print("fused GEMV tiers, worst error / bar:", {k: float(f"{v:.3g}") for k, v in sorted(REPORT.items())})
