"""GPU: prefill (effort_model_prefill, DESIGN.md section 4.8) -- the multi-token GEMV against the oracle token by token,
the chunk attention and cache append on the inputs it consumed, whole prompts against the CPU restatement stepping the
same tokens, scoring and sampling, the limits and the configurations that fall back to stepping, and reproducibility.

Bars: the operator's (cutoff bit-exact, count equal, output rel. L2 <= 2e-6 against the oracle's float64 sum of the same
rows), the glue kernels' of test_gpu_glue.py (V rows byte-exact, K rows a rotation, attention rel. L2 <= 1e-5 per head),
and the decode's (last logits cos-sim > 0.9995 against the restatement)."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import glue_ref as G
from tests.util import make_v, make_w, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 2e-6
ATTN_BAR = 1e-5
ROPE_NORM_BAR = 8 * 2.0 ** -24
EFFORTS = [1.0, 0.5, 0.25, 0.1]
SHAPES = [(4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096)]


@pytest.fixture(autouse=True)
def _select_mode():
    with O.cutoff_mode("select"):
        yield


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


_conv = {}


def _weights(in_dim, out_dim, shuffle_stats=False, **kw):
    from effort_b200 import ops
    key = (in_dim, out_dim, shuffle_stats)
    if key not in _conv:
        r = dict(O.bucketize(make_w(out_dim, in_dim, 1234)))
        if shuffle_stats:  # arbitrary statistics: the selected ranks of an input are no longer a prefix
            st = r["bucket.stats"].reshape(16, in_dim, 4).copy()
            rng = np.random.default_rng(5)
            for i in range(in_dim):
                st[:, i] = st[rng.permutation(16), i]
            r["bucket.stats"] = st.reshape(r["bucket.stats"].shape)
        _conv[key] = r
    r = _conv[key]
    return r, ops.ExpertWeights(_dev(r["buckets"]), _dev(r["bucket.stats"]), _dev(r["probes"]), inDim=in_dim, outDim=out_dim, **kw)


def _tokens(in_dim):
    """16 input vectors: seeded ones, a repeat, zero, a dominant entry, and test_gpu_parity's edge inputs (one-hot, ones,
    huge, tiny, ties)"""
    vs = [make_v(in_dim, s) for s in range(8)]
    vs.append(np.eye(1, in_dim, 17, dtype=np.float32)[0] * 5)
    vs.append(vs[0].copy())
    vs.append(np.zeros(in_dim, np.float32))
    dom = make_v(in_dim, 20) * 1e-4
    dom[17] = 50.0
    vs.append(dom)
    vs.append(np.ones(in_dim, np.float32))
    vs.append(make_v(in_dim, 3) * 1e4)
    vs.append(make_v(in_dim, 4) * 1e-6)
    vs.append(np.sign(make_v(in_dim, 5)).astype(np.float32))
    return np.stack(vs)


CHUNKS = [list(range(16)), list(range(8, 16)), [10, 0, 11], [12, 3], [5]]  # T = 16, 8, 3, 2, 1


def _check_operator(in_dim, out_dim, efforts, shuffle_stats=False):
    from effort_b200 import ops
    r, ew = _weights(in_dim, out_dim, shuffle_stats)
    V = _tokens(in_dim)
    for effort in efforts:
        ref = [O.bucket_mul(v, r["buckets"], r["bucket.stats"], r["probes"], in_dim, out_dim, effort) for v in V]
        first = {}
        for chunk in CHUNKS:
            Vd = _dev(V[chunk])
            out, cut, cnt = ops.bucket_mul_multi(Vd, ew, effort)
            out2, _, _ = ops.bucket_mul_multi(Vd, ew, effort)
            out, cut, cnt, out2 = out.cpu().numpy(), cut.cpu().numpy(), cnt.cpu().numpy(), out2.cpu().numpy()
            assert np.array_equal(_u32(out), _u32(out2)), (effort, chunk)   # run to run
            for j, t in enumerate(chunk):
                c_ref = np.float32(O.select_cutoff(V[t], r["probes"], effort))
                assert _u32(cut[j]) == _u32(c_ref), (effort, t, cut[j], c_ref)
                assert cnt[j] == ref[t]["n_selected"], (effort, t, cnt[j], ref[t]["n_selected"])
                assert rel_err(out[j], ref[t]["out64"]) <= OUT_TOL, (effort, t, rel_err(out[j], ref[t]["out64"]))
                # a token's bits depend on its own input only, not on the chunk it shares
                if t in first:
                    assert np.array_equal(_u32(out[j]), _u32(first[t])), (effort, t, chunk)
                first.setdefault(t, out[j].copy())
        # equal inputs give equal outputs (tokens 0 and 9 are the same vector)
        assert np.array_equal(_u32(first[0]), _u32(first[9]))


@pytest.mark.parametrize("in_dim,out_dim", SHAPES)
def test_multi_gemv_matches_oracle(in_dim, out_dim):
    # effort 0.0 (select rank k = 1) on the square shape only: the oracle's float64 sums dominate the run time
    _check_operator(in_dim, out_dim, EFFORTS + ([0.0] if (in_dim, out_dim) == (4096, 4096) else []))


def test_multi_gemv_arbitrary_statistics():
    _check_operator(4096, 4096, [0.5, 0.25], shuffle_stats=True)


def test_multi_gemv_refuses_other_weights():
    import torch
    from effort_b200 import EffortError, ops
    r, ew = _weights(4096, 4096)
    V = torch.zeros(2, 4096, dtype=torch.float32, device="cuda")
    inp = ops.ExpertWeights(_dev(r["buckets"]), _dev(r["bucket.stats"]), _dev(r["probes"]), inDim=4096, outDim=4096,
                            flags=ops.INPUT_MAJOR)
    with pytest.raises(EffortError, match="shape"):
        ops.bucket_mul_multi(V, inp, 0.25)
    two = ops.ExpertWeights(_dev(np.concatenate([r["buckets"]] * 2)), _dev(np.concatenate([r["bucket.stats"]] * 2)),
                            _dev(np.concatenate([r["probes"]] * 2)), inDim=4096, outDim=4096, numExperts=2)
    with pytest.raises(EffortError, match="shape"):
        ops.bucket_mul_multi(V, two, 0.25)
    from effort_b200.model import DecodeModel, MistralConfig
    q4 = DecodeModel.random_init_q4(MistralConfig(n_layers=1, vocab=256, max_seq=8), seed=3)
    with pytest.raises(EffortError, match="shape"):
        ops.bucket_mul_multi(V, q4.layers[0][0], 0.25)
    with pytest.raises(EffortError, match="invalid"):
        ops.bucket_mul_multi(torch.zeros(17, 4096, dtype=torch.float32, device="cuda"), ew, 0.25)


# ---------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------
def _cpu(t):
    return t.cpu().numpy()


def _model(n_layers=2, vocab=32000, max_seq=64, seed=7, spec=True, n_kv_heads=8):
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=n_layers, vocab=vocab, max_seq=max_seq, n_kv_heads=n_kv_heads)
    m = DecodeModel.random_init(cfg, seed=seed, keep_reference_layout=spec)
    if not spec:
        return m, None
    names = ["wq", "wk", "wv", "wo", "w1", "w2", "w3"]
    layers = []
    for L in m.layers:
        d = {n: {"buckets": _cpu(ew.buckets), "stats": _cpu(ew.stats), "probes": _cpu(ew.probes), "in": ew.inSize,
                 "out": ew.outSize} for n, ew in zip(names, L[:7])}
        d["attn_norm"], d["ffn_norm"] = _cpu(L[7]), _cpu(L[8])
        layers.append(d)
    return m, (layers, [_cpu(t) for t in m.head[:3]])


@pytest.fixture(scope="module")
def small():
    return _model()


@pytest.fixture(scope="module")
def one_kv():
    """GQA ratio 32: a chunk has 32 * T (head, token) pairs per KV head, more than one attention CTA takes"""
    return _model(n_layers=1, vocab=4096, seed=13, spec=False, n_kv_heads=1)


def _side_stream():
    """A non-default stream: the model captures and replays CUDA graphs only there (the legacy stream cannot capture)."""
    import torch
    return torch.cuda.stream(torch.cuda.Stream())


def _seq(n, vocab, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, vocab, n)]


def _ref(spec, fast=True):
    from tests.ref_decode import RefModel
    layers, head = spec
    return RefModel(layers, *head, fast=fast)


def _cache(m, name, li):
    c = m.cfg
    return m.buffer_view(name, li).cpu().numpy().reshape(c.max_seq, c.n_kv_heads, 128)


@pytest.mark.parametrize("which", ["gqa4", "gqa32"])
def test_chunk_glue(small, one_kv, which):
    """the last chunk's last layer: V rows byte-exact, K rows a rotation, each query's attention against float64"""
    with _side_stream():
        _chunk_glue(small if which == "gqa4" else one_kv)


def _chunk_glue(model):
    import torch
    m, _ = model
    c = m.cfg
    m.set_graphs(True)
    for start, n in ((0, 16), (5, 11), (c.max_seq - 16, 16)):
        m.reset()
        toks = _seq(start + n, c.vocab, start)
        if start:
            m.prefill(toks[:start], 0.25)
        m.prefill(toks[start:], 0.25)
        torch.cuda.synchronize()
        T = int(m.buffer_view("CHUNK_LEN").cpu()[0])
        p0 = start + n - T
        xq = m.buffer("CHUNK_Q").cpu().numpy().reshape(T, -1)
        xk = m.buffer("CHUNK_K").cpu().numpy().reshape(T, -1)
        xv = m.buffer("CHUNK_V").cpu().numpy().reshape(T, -1)
        attn = m.buffer("CHUNK_ATTN").cpu().numpy().reshape(T, c.n_heads, 128)
        K, V = _cache(m, "KCACHE", -1), _cache(m, "VCACHE", -1)
        assert int(m.buffer_view("POS").cpu()[0]) == start + n
        worst = 0.0
        for t in range(T):
            p = p0 + t
            assert np.array_equal(_u32(V[p].reshape(-1)), _u32(xv[t])), (start, t)
            norm_err, angle = G.rope_check(xk[t], K[p].reshape(-1), p, c.rope_theta)
            assert norm_err <= ROPE_NORM_BAR and angle <= 1.0, (start, t, norm_err, angle)
            want = G.attention_step(xq[t], xk[t], K, V, p)
            worst = max(worst, max(float(np.linalg.norm(attn[t, h] - want[h]) / np.linalg.norm(want[h]))
                                   for h in range(c.n_heads)))
        assert worst <= ATTN_BAR, (start, worst)


@pytest.mark.parametrize("effort", [1.0, 0.5])
def test_prefill_matches_stepping_restatement(small, effort):
    with _side_stream():
        _matches_restatement(small, effort)


def _matches_restatement(small, effort):
    import torch
    m, spec = small
    c = m.cfg
    m.set_graphs(True)
    for n in (1, 15, 16, 17, 40):
        for pre in (0, 3):
            toks = _seq(pre + n, c.vocab, 100 + n + pre)
            ref = _ref(spec)
            m.reset()
            for t in toks[:pre]:
                m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort)
            m.prefill(toks[pre:], effort)
            torch.cuda.synchronize()
            for t in toks:
                want = ref.step(t, effort)
            got = m.logits().cpu().numpy()
            assert O.cossim(got, want) > 0.9995, (n, pre, O.cossim(got, want))
            assert int(m.buffer_view("POS").cpu()[0]) == pre + n
            assert m.next_token() == G.greedy(got)
            for li in range(c.n_layers):
                K, V = _cache(m, "KCACHE", li), _cache(m, "VCACHE", li)
                for p in range(pre + n):
                    assert O.cossim(V[p].reshape(-1), ref.vc[li][p].reshape(-1)) > 0.9995, (n, pre, li, p)
                    assert O.cossim(K[p].reshape(-1), ref.kc[li][p].reshape(-1)) > 0.9995, (n, pre, li, p)


def test_32_layers_full_effort():
    import torch
    m, _ = _model(n_layers=32, vocab=4096, max_seq=80, seed=11, spec=False)
    toks = _seq(64, 4096, 9)
    m.reset()
    m.prefill(toks, 1.0)
    torch.cuda.synchronize()
    got = m.logits().cpu().numpy()
    m.reset()
    for t in toks:
        m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), 1.0)
    torch.cuda.synchronize()
    assert O.cossim(got, m.logits().cpu().numpy()) > 0.9995


def test_scoring_and_sampling(small):
    with _side_stream():
        _scoring_and_sampling(small)


def _scoring_and_sampling(small):
    import torch
    from effort_b200 import ops
    m, _ = small
    c = m.cfg
    toks = _seq(37, c.vocab, 3)
    for graphs in (False, True):
        m.set_graphs(graphs)
        m.set_scoring(True)
        try:
            m.set_score_targets(torch.tensor(toks[1:] + [5], dtype=torch.int32, device="cuda"))
            m.reset()
            m.prefill(toks[:4], 0.25)
            m.prefill(toks[4:], 0.25)
            torch.cuda.synchronize()
            T = int(m.buffer_view("CHUNK_LEN").cpu()[0])
            rows = m.buffer("CHUNK_LOGITS").view(T, c.vocab)
            assert torch.equal(rows[-1], m.logits())
            p0 = len(toks) - T
            got = m.scores()
            for j in range(T):
                w = ops.score(rows[j], torch.tensor([(toks[1:] + [5])[p0 + j]], dtype=torch.int32, device="cuda"))
                for a, b in zip(w, got):
                    assert torch.equal(a[0].cpu(), b[p0 + j].cpu()), (graphs, j)
            assert m.next_token() == G.greedy(m.logits().cpu().numpy())
        finally:
            m.set_scoring(False)
        m.set_sampler(0.8, 50, 0.9, seed=1234)
        try:
            m.reset()
            m.prefill(toks, 0.25)
            torch.cuda.synchronize()
            want = ops.sample(m.logits(), 0.8, 50, 0.9, seed=1234, position=len(toks))
            assert m.next_token() == int(want.cpu()[0])
        finally:
            m.set_sampler(None)


def test_limits(small):
    import torch
    from effort_b200 import EffortError
    m, _ = small
    c = m.cfg
    m.reset()
    m.prefill(_seq(c.max_seq - 3, c.vocab, 1), 0.25)
    torch.cuda.synchronize()
    with pytest.raises(EffortError, match="call sequence"):
        m.prefill(_seq(4, c.vocab, 2), 0.25)
    torch.cuda.synchronize()
    assert int(m.buffer_view("POS").cpu()[0]) == c.max_seq - 3
    with pytest.raises(EffortError, match="invalid"):
        m.prefill([], 0.25)
    m.prefill(_seq(3, c.vocab, 2), 0.25)   # exactly to max_seq
    torch.cuda.synchronize()
    assert int(m.buffer_view("POS").cpu()[0]) == c.max_seq


def _state(m, scored=False):
    import torch
    torch.cuda.synchronize()
    caches = [m.buffer(n, li).cpu().numpy() for li in range(m.cfg.n_layers) for n in ("KCACHE", "VCACHE")]
    records = [col.cpu().numpy() for col in m.scores()] if scored else []
    return m.logits().cpu().numpy(), m.next_token(), caches + records


def _same(a, b):
    assert np.array_equal(_u32(a[0]), _u32(b[0]))
    assert a[1] == b[1]
    assert len(a[2]) == len(b[2])
    for x, y in zip(a[2], b[2]):
        assert np.array_equal(_u32(x), _u32(y))


def _runtime_calls(fn):
    """CUDA runtime calls `fn` makes, by name (torch.profiler with CUDA activities)"""
    import torch
    from collections import Counter
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(e.name.split("_v")[0] for e in prof.events() if e.name.startswith("cuda"))


@pytest.mark.parametrize("mode", ["greedy", "scoring", "sampling"])
def test_graphs_on_and_off_identical(small, mode):
    """45 tokens = chunks of 16, 16 and 13: eager (graphs off) against captured and replayed graphs, byte for byte in the
    logits, next token, every KV cache row and, with scoring, every record; the replayed prefill launches no kernel
    itself (three cudaGraphLaunch calls) and counts the same launches as the eager one"""
    import torch
    from effort_b200 import ops
    m, _ = small
    toks = _seq(45, m.cfg.vocab, 8)
    scored = mode == "scoring"
    with _side_stream():
        m.set_scoring(scored)
        if scored:
            m.set_score_targets(torch.tensor(toks[1:], dtype=torch.int32, device="cuda"))
        if mode == "sampling":
            m.set_sampler(0.8, 50, 0.9, seed=99)
        try:
            def run():
                m.reset()
                m.prefill(toks, 0.25)

            m.set_graphs(False)
            run()
            eager = _state(m, scored)
            torch.cuda.synchronize()
            l0 = ops.launchCount()
            run()
            torch.cuda.synchronize()
            eager_launches = ops.launchCount() - l0
            _same(eager, _state(m, scored))
            m.set_graphs(True)
            for _ in range(2):   # the first chunk of a model runs eagerly; every (effort, length) is captured once
                run()
                _same(eager, _state(m, scored))
            l0 = ops.launchCount()
            calls = _runtime_calls(run)
            assert ops.launchCount() - l0 == eager_launches
            _same(eager, _state(m, scored))
            assert calls["cudaGraphLaunch"] == 3, calls
            assert not any("LaunchKernel" in k for k in calls), calls
        finally:
            m.set_scoring(False)
            m.set_sampler(None)
            m.set_graphs(True)


def test_fallbacks_are_stepping():
    """chain 1, Q4 and MoE models step: prefill enqueues exactly the launches of one step per token and ends in the
    stepping's state.  Where two steppings of the same tokens repeat bit for bit, prefill must give the same bits
    (logits, next token, every KV cache row); where they do not (chain 1's generic GEMVs add their CTA sums with
    atomics), it must agree with stepping to the decode bar in the logits and every cache row, and pick greedy's token."""
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=2048, max_seq=32)
    toks = _seq(20, 2048, 4)
    dense = DecodeModel.random_init(cfg, seed=7)
    dense.set_chain(1)
    models = {"chain1": dense, "q4": DecodeModel.random_init_q4(cfg, seed=7),
              "moe": DecodeModel.random_init_moe(cfg, n_experts=4, seed=7)}
    with _side_stream():
        for name, m in models.items():
            for graphs in (False, True):
                m.set_graphs(graphs)

                def steps():
                    m.reset()
                    for t in toks:
                        m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), 0.5)
                    return _state(m)

                first = steps()          # includes the first (eager) step and the capture
                l0 = ops.launchCount()
                second = steps()
                l1 = ops.launchCount()
                m.reset()
                m.prefill(toks, 0.5)
                got = _state(m)
                assert ops.launchCount() - l1 == l1 - l0, name
                assert int(m.buffer_view("POS").cpu()[0]) == len(toks)
                assert m.buffer_view("CHUNK_LEN") is None
                try:
                    _same(first, second)
                    repeats = True
                except AssertionError:
                    repeats = False
                if repeats:
                    _same(got, second)
                    continue
                assert O.cossim(got[0], second[0]) > 0.9995, name
                assert got[1] == G.greedy(got[0]), name
                for x, y in zip(got[2], second[2]):
                    rows_x, rows_y = x.reshape(cfg.max_seq, -1), y.reshape(cfg.max_seq, -1)
                    for p in range(len(toks)):
                        assert O.cossim(rows_x[p], rows_y[p]) > 0.9995, (name, p)


@pytest.mark.parametrize("scoring", [False, True])
def test_long_prefill_repeats(scoring):
    with _side_stream():   # 128 chunks replayed from the captured graph
        _long_repeats(scoring)


def _long_repeats(scoring):
    import torch
    m, _ = _model(max_seq=2048, seed=9, spec=False)
    toks = _seq(2048, m.cfg.vocab, 77)
    m.set_scoring(scoring)
    if scoring:
        m.set_score_targets(torch.tensor(toks[1:], dtype=torch.int32, device="cuda"))
    runs = []
    for _ in range(2):
        m.reset()
        m.prefill(toks, 0.25)
        runs.append(_state(m, scoring))   # with scoring: all three record columns of positions 0..2047
    _same(runs[0], runs[1])
