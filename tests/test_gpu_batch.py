"""GPU: batch decode (effort_batch_*, DESIGN.md section 4.9) -- batch invariance byte for byte, slots against the CPU
restatement stepping the same tokens, the batch attention on the inputs it consumed, fork, the per-slot tails, graphs,
the model left untouched, the limits, and repeatability with the Python entry points.

Bars: the decode's (cos-sim > 0.9995 against the restatement) and the glue kernels' of test_gpu_glue.py (V rows
byte-exact, K rows a rotation, attention rel. L2 <= 1e-5 per head); everything else is byte-exact."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import glue_ref as G

pytestmark = pytest.mark.gpu

ATTN_BAR = 1e-5
ROPE_NORM_BAR = 8 * 2.0 ** -24


@pytest.fixture(autouse=True)
def _select_mode():
    with O.cutoff_mode("select"):
        yield


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """the modules after this one start with the device memory they would have had without it"""
    yield
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


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
    """GQA ratio 32"""
    return _model(n_layers=1, vocab=4096, seed=13, spec=False, n_kv_heads=1)


def _side_stream():
    """A non-default stream: graphs are captured and replayed only there (the legacy stream cannot capture)."""
    import torch
    return torch.cuda.stream(torch.cuda.Stream())


def _seq(n, vocab, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(0, vocab, n)]


def _i32(x):
    import torch
    return torch.tensor(x, dtype=torch.int32, device="cuda")


def _batch(m, n):
    from effort_b200.model import DecodeBatch
    return DecodeBatch(m, n)


def _cache(obj, name, li, seq=None):
    c = obj.cfg
    v = obj.buffer_view(name, li) if seq is None else obj.buffer_view(name, li, seq)
    return v.cpu().numpy().reshape(c.max_seq, c.n_kv_heads, 128)


def _slot_state(bt, b):
    """slot b's logits row, next token, position, and its cache rows and records below its position"""
    import torch
    torch.cuda.synchronize()
    c = bt.cfg
    pos = int(bt.buffer_view("POS").cpu()[b])
    caches = [_cache(bt, n, li, b)[:pos].copy() for li in range(c.n_layers) for n in ("KCACHE", "VCACHE")]
    return {"logits": _cpu(bt.logits()[b]), "next": bt.next_tokens()[b], "pos": pos, "caches": caches,
            "records": [_cpu(col)[:pos] for col in bt.scores(b)]}


def _same_state(a, b, what=""):
    assert a["pos"] == b["pos"], what
    assert a["next"] == b["next"], what
    assert np.array_equal(_u32(a["logits"]), _u32(b["logits"])), what
    for x, y in zip(a["caches"] + a["records"], b["caches"] + b["records"]):
        assert np.array_equal(_u32(x), _u32(y)), what


# ---------------------------------------------------------------------------------------------------------------
# 1. invariance
# ---------------------------------------------------------------------------------------------------------------
N_EXPLICIT, N_GREEDY = 4, 3


def _plan(c):
    """16 slots: slot i starts from prompt i % 3 (lengths 5, 12, 1), except slots 5 and 11 which start from a reset;
    every slot has its own explicit tokens and targets, and slots 1, 5, 9, 13 sample with their own seed"""
    prompts = [_seq(5, c.vocab, 1), _seq(12, c.vocab, 2), _seq(1, c.vocab, 3)]
    slots = []
    for i in range(16):
        slots.append({"prompt": None if i in (5, 11) else i % 3, "tokens": _seq(N_EXPLICIT, c.vocab, 50 + i),
                      "targets": _seq(c.max_seq, c.vocab, 80 + i), "sampler": dict(temperature=0.9, top_k=40, top_p=0.95,
                                                                                  seed=1000 + i) if i % 4 == 1 else None})
    return prompts, slots


def _run_slots(m, prompts, plan, effort):
    """a batch whose slot k follows plan[k]; returns it after N_EXPLICIT explicit and N_GREEDY greedy steps"""
    import torch
    bt = _batch(m, len(plan))
    bt.set_scoring(True)
    for k, p in enumerate(plan):
        if p["sampler"]:
            bt.set_sampler(k, **p["sampler"])
        bt.set_score_targets(k, _i32(p["targets"]))
    for pi, pr in enumerate(prompts):
        ks = [k for k, p in enumerate(plan) if p["prompt"] == pi]
        if ks:
            m.reset()
            m.prefill(pr, effort)
            for k in ks:
                bt.fork(k)
    for k, p in enumerate(plan):
        if p["prompt"] is None:
            bt.reset(k)
    feed = torch.tensor([[p["tokens"][j] for p in plan] for j in range(N_EXPLICIT)], dtype=torch.int32, device="cuda")
    for j in range(N_EXPLICIT):
        bt.step(feed[j], effort)
    for _ in range(N_GREEDY):
        bt.step(None, effort)
    return bt


@pytest.mark.parametrize("effort", [1.0, 0.25])
def test_batch_invariance(small, effort):
    m, _ = small
    prompts, slots = _plan(m.cfg)
    filler = [{"prompt": 1, "tokens": _seq(N_EXPLICIT, m.cfg.vocab, 900 + j), "targets": _seq(m.cfg.max_seq, m.cfg.vocab, 950 + j),
               "sampler": None} for j in range(4)]
    with _side_stream():
        big = _run_slots(m, prompts, slots, effort)
        full = [_slot_state(big, i) for i in range(16)]
        del big
        for i in range(16):
            alone = _run_slots(m, prompts, [slots[i]], effort)
            _same_state(full[i], _slot_state(alone, 0), ("alone", effort, i))
            five = _run_slots(m, prompts, filler[:3] + [slots[i]] + filler[3:], effort)
            _same_state(full[i], _slot_state(five, 3), ("five", effort, i))


# ---------------------------------------------------------------------------------------------------------------
# 2. restatement
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("effort", [1.0, 0.5])
def test_batch_matches_stepping_restatement(small, effort):
    import torch
    from tests.ref_decode import RefModel
    m, spec = small
    c = m.cfg
    prompts = [_seq(n, c.vocab, 200 + n) for n in (1, 15, 17)]
    extra = [_seq(3, c.vocab, 300 + b) for b in range(3)]
    with _side_stream():
        bt = _batch(m, 3)
        for b, p in enumerate(prompts):
            m.reset()
            m.prefill(p, effort)
            bt.fork(b)
        for j in range(3):
            bt.step(_i32([extra[b][j] for b in range(3)]), effort)
        torch.cuda.synchronize()
    logits = _cpu(bt.logits())
    nxt = bt.next_tokens()
    for b in range(3):
        ref = RefModel(spec[0], *spec[1], fast=True)
        for t in prompts[b] + extra[b]:
            want = ref.step(t, effort)
        assert O.cossim(logits[b], want) > 0.9995, (b, O.cossim(logits[b], want))
        assert nxt[b] == G.greedy(logits[b])
        n = len(prompts[b]) + 3
        assert int(bt.buffer_view("POS").cpu()[b]) == n
        for li in range(c.n_layers):
            K, V = _cache(bt, "KCACHE", li, b), _cache(bt, "VCACHE", li, b)
            for p in range(n):
                assert O.cossim(K[p].reshape(-1), ref.kc[li][p].reshape(-1)) > 0.9995, (b, li, p)
                assert O.cossim(V[p].reshape(-1), ref.vc[li][p].reshape(-1)) > 0.9995, (b, li, p)


def test_32_layers_full_effort():
    import torch
    m, _ = _model(n_layers=32, vocab=4096, max_seq=48, seed=11, spec=False)
    toks = _seq(24, 4096, 9)
    m.reset()
    m.prefill(toks[:20], 1.0)
    bt = _batch(m, 2)
    bt.fork()
    for t in toks[20:]:
        bt.step(_i32([t, t]), 1.0)
    torch.cuda.synchronize()
    got = _cpu(bt.logits())
    m.reset()
    for t in toks:
        m.step(_i32([t]), 1.0)
    torch.cuda.synchronize()
    want = _cpu(m.logits())
    assert np.array_equal(_u32(got[0]), _u32(got[1]))
    assert O.cossim(got[0], want) > 0.9995, O.cossim(got[0], want)


# ---------------------------------------------------------------------------------------------------------------
# 3. attention glue
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["gqa4", "gqa32"])
def test_batch_attention_glue(small, one_kv, which):
    """slots at positions 0, mid-range and max_seq - 1 in one step"""
    import torch
    m, _ = small if which == "gqa4" else one_kv
    c = m.cfg
    starts = [0, c.max_seq // 2, c.max_seq - 1]
    with _side_stream():
        bt = _batch(m, 3)
        for b, p0 in enumerate(starts):
            if p0 == 0:
                bt.reset(b)
                continue
            m.reset()
            m.prefill(_seq(p0, c.vocab, p0), 0.25)
            bt.fork(b)
        bt.step(_i32(_seq(3, c.vocab, 5)), 0.25)
        torch.cuda.synchronize()
    kvd = c.n_kv_heads * 128
    xq = _cpu(bt.buffer("Q")).reshape(3, -1)
    xk = _cpu(bt.buffer("K")).reshape(3, kvd)
    xv = _cpu(bt.buffer("V")).reshape(3, kvd)
    attn = _cpu(bt.buffer("ATTN")).reshape(3, c.n_heads, 128)
    assert _cpu(bt.buffer("POS")).tolist() == [p + 1 for p in starts]
    for b, p in enumerate(starts):
        K, V = _cache(bt, "KCACHE", -1, b), _cache(bt, "VCACHE", -1, b)
        assert np.array_equal(_u32(V[p].reshape(-1)), _u32(xv[b])), b
        norm_err, angle = G.rope_check(xk[b], K[p].reshape(-1), p, c.rope_theta)
        assert norm_err <= ROPE_NORM_BAR and angle <= 1.0, (b, norm_err, angle)
        want = G.attention_step(xq[b], xk[b], K, V, p)
        worst = max(float(np.linalg.norm(attn[b, h] - want[h]) / np.linalg.norm(want[h])) for h in range(c.n_heads))
        assert worst <= ATTN_BAR, (b, worst)


# ---------------------------------------------------------------------------------------------------------------
# 4. fork, 5. tails
# ---------------------------------------------------------------------------------------------------------------
SAMPLER = dict(temperature=0.8, top_k=50, top_p=0.9, seed=4321)


def test_fork(small):
    import torch
    from effort_b200 import ops
    m, _ = small
    c = m.cfg
    toks = _seq(20, c.vocab, 11)
    targets = _seq(c.max_seq, c.vocab, 12)
    with _side_stream():
        m.reset()
        m.prefill(toks, 0.25)
        bt = _batch(m, 2)
        bt.set_sampler(1, **SAMPLER)
        bt.set_scoring(True)
        bt.set_score_targets(None, _i32(targets))
        bt.fork()
        torch.cuda.synchronize()
    logits = m.logits()
    assert _cpu(bt.buffer("POS")).tolist() == [20, 20]
    want_rec = [_cpu(x[0]) for x in ops.score(logits, _i32([targets[19]]))]
    for b in range(2):
        assert np.array_equal(_u32(_cpu(bt.logits()[b])), _u32(_cpu(logits)))
        for li in range(c.n_layers):
            for name in ("KCACHE", "VCACHE"):
                assert np.array_equal(_u32(_cache(bt, name, li, b)[:20]), _u32(_cache(m, name, li)[:20])), (b, li, name)
        rec = [_cpu(col[19]) for col in bt.scores(b)]
        for x, y in zip(rec, want_rec):
            assert np.array_equal(_u32(x), _u32(y)), b
    nxt = bt.next_tokens()
    assert nxt[0] == m.next_token()
    assert nxt[1] == int(ops.sample(logits, position=20, **SAMPLER).cpu()[0])


def _runtime_calls(fn):
    """CUDA runtime calls `fn` makes, by name (torch.profiler with CUDA activities)"""
    import torch
    from collections import Counter
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return Counter(e.name.split("_v")[0] for e in prof.events() if e.name.startswith("cuda"))


def _check_tails(bt, samplers, targets):
    import torch
    from effort_b200 import ops
    torch.cuda.synchronize()
    rows = bt.logits()
    pos = _cpu(bt.buffer("POS")).tolist()
    nxt = bt.next_tokens()
    for b, s in enumerate(samplers):
        want = G.greedy(_cpu(rows[b])) if s is None else int(ops.sample(rows[b], position=pos[b], **s).cpu()[0])
        assert nxt[b] == want, (b, s)
        p = pos[b] - 1
        rec = [_cpu(col[p]) for col in bt.scores(b)]
        for x, y in zip(rec, [_cpu(w[0]) for w in ops.score(rows[b], _i32([targets[b][p]]))]):
            assert np.array_equal(_u32(x), _u32(y)), b


def test_tails(small):
    m, _ = small
    c = m.cfg
    samplers = [None, SAMPLER, dict(temperature=1.3, top_k=0, top_p=1.0, seed=7), None]
    targets = [_seq(c.max_seq, c.vocab, 60 + b) for b in range(4)]
    with _side_stream():
        m.reset()
        m.prefill(_seq(9, c.vocab, 13), 0.25)
        bt = _batch(m, 4)
        bt.set_scoring(True)
        for b in range(4):
            bt.set_score_targets(b, _i32(targets[b]))
            if samplers[b]:
                bt.set_sampler(b, **samplers[b])
        bt.fork()
        _check_tails(bt, samplers, targets)
        for _ in range(3):   # eager, capture, replay
            bt.step(None, 0.25)
            _check_tails(bt, samplers, targets)
        samplers[1] = dict(temperature=0.5, top_k=5, top_p=0.8, seed=99)   # a new parameter set: no recapture
        bt.set_sampler(1, **samplers[1])
        calls = _runtime_calls(lambda: bt.step(None, 0.25))
        assert calls["cudaStreamBeginCapture"] == 0 and calls["cudaGraphLaunch"] == 1, calls
        _check_tails(bt, samplers, targets)


# ---------------------------------------------------------------------------------------------------------------
# 6. graphs
# ---------------------------------------------------------------------------------------------------------------
def test_graphs_identical_to_eager(small):
    import torch
    from effort_b200 import ops
    m, _ = small
    c = m.cfg
    toks = [_seq(4, c.vocab, 70 + j) for j in range(5)]
    with _side_stream():
        m.reset()
        m.prefill(_seq(10, c.vocab, 14), 0.5)
        bt = _batch(m, 4)
        bt.set_scoring(True)
        bt.set_score_targets(None, _i32(_seq(c.max_seq, c.vocab, 15)))
        bt.set_sampler(2, **SAMPLER)

        def run():
            bt.fork()
            for j in range(5):
                bt.step(_i32(toks[j]), 0.5)

        def state():
            return [_slot_state(bt, b) for b in range(4)]

        m.set_graphs(False)
        try:
            run()
            eager = state()
            l0 = ops.launchCount()
            bt.step(None, 0.5)
            torch.cuda.synchronize()
            eager_launches = ops.launchCount() - l0
            eager_next = state()
            m.set_graphs(True)
            for _ in range(2):   # the first graphed step runs eagerly, the second captures
                run()
                for a, b in zip(eager, state()):
                    _same_state(a, b, "graphs")
            l0 = ops.launchCount()
            calls = _runtime_calls(lambda: bt.step(None, 0.5))
            assert ops.launchCount() - l0 == eager_launches
            assert calls["cudaGraphLaunch"] == 1, calls
            assert not any("LaunchKernel" in k for k in calls), calls
            for a, b in zip(eager_next, state()):
                _same_state(a, b, "replay")
        finally:
            m.set_graphs(True)


# ---------------------------------------------------------------------------------------------------------------
# 7. the model is untouched
# ---------------------------------------------------------------------------------------------------------------
def test_model_untouched(small):
    import torch
    m, _ = small
    c = m.cfg
    toks = _seq(14, c.vocab, 16)
    m.set_scoring(True)
    m.set_score_targets(_i32(toks[1:] + [3]))

    def model_state():
        torch.cuda.synchronize()
        caches = [_cpu(m.buffer(n, li)) for li in range(c.n_layers) for n in ("KCACHE", "VCACHE")]
        return [_cpu(m.logits()), np.array([m.next_token()]), _cpu(m.buffer("POS"))] + caches + [_cpu(x) for x in m.scores()]

    try:
        with _side_stream():
            runs = []
            for use_batch in (False, True):
                m.reset()
                m.prefill(toks[:10], 0.25)
                if use_batch:
                    bt = _batch(m, 3)
                    bt.set_scoring(True)
                    bt.fork()
                    for _ in range(3):
                        bt.step(None, 0.25)
                    torch.cuda.synchronize()
                for t in toks[10:]:
                    m.step(_i32([t]), 0.25)
                runs.append(model_state())
        for x, y in zip(*runs):
            assert np.array_equal(_u32(x), _u32(y))
    finally:
        m.set_scoring(False)


# ---------------------------------------------------------------------------------------------------------------
# 8. limits
# ---------------------------------------------------------------------------------------------------------------
def test_limits(small):
    import ctypes as C
    import torch
    from effort_b200 import EffortError
    from effort_b200.model import DecodeModel, MistralConfig
    m, _ = small
    c = m.cfg
    L = m._L
    h = C.c_void_p()
    for n in (0, 17):
        assert L.effort_batch_create(m._h, n, C.byref(h)) == -1 and not h.value
    assert L.effort_batch_create(m._h, 2, None) == -1
    bt = _batch(m, 2)
    for seq in (-2, 2):
        assert L.effort_batch_reset(bt._h, seq, None) == -1
        assert L.effort_batch_fork(bt._h, seq, None) == -1
        assert L.effort_batch_set_sampler(bt._h, seq, None) == -1
        assert L.effort_batch_set_score_targets(bt._h, seq, None, 0, None) == -1
    assert L.effort_batch_set_score_targets(bt._h, 0, None, 3, None) == -1
    assert L.effort_batch_set_score_targets(bt._h, 0, None, -1, None) == -1
    assert L.effort_batch_buffer(bt._h, 4, 0, 2, None) is None
    assert L.effort_batch_buffer(bt._h, 6, 0, 0, None) is None
    assert L.effort_batch_buffer(bt._h, 0, 0, 0, None) is None   # no step yet
    for e in (-0.1, 1.5, float("nan")):
        with pytest.raises(EffortError, match="invalid"):
            bt.step(None, e)
    bad = MistralConfig(n_layers=1, vocab=2048, max_seq=16)
    with pytest.raises(EffortError, match="shape"):
        _batch(DecodeModel.random_init_q4(bad, seed=3), 2)
    with _side_stream():
        m.reset()
        torch.cuda.synchronize()
        with pytest.raises(EffortError, match="call sequence"):   # fork from position 0
            bt.fork()
        m.prefill(_seq(c.max_seq - 2, c.vocab, 17), 0.25)
        bt.fork(0)
        bt.reset(1)
        bt.step(None, 0.25)
        bt.step(None, 0.25)
        torch.cuda.synchronize()
        assert _cpu(bt.buffer("POS")).tolist() == [c.max_seq, 2]
        with pytest.raises(EffortError, match="call sequence"):   # slot 0 sits at max_seq
            bt.step(None, 0.25)
        torch.cuda.synchronize()
        assert _cpu(bt.buffer("POS")).tolist() == [c.max_seq, 2]
        m.set_chain(1)
        try:
            with pytest.raises(EffortError, match="shape"):
                bt.reset(0)
                bt.step(None, 0.25)
            with pytest.raises(EffortError, match="shape"):
                bt.fork(1)
            with pytest.raises(EffortError, match="shape"):
                _batch(m, 1)
        finally:
            m.set_chain(2)
        torch.cuda.synchronize()
        assert _cpu(bt.buffer("POS")).tolist() == [0, 2]


# ---------------------------------------------------------------------------------------------------------------
# 9. repeatability and the Python entry points
# ---------------------------------------------------------------------------------------------------------------
def test_long_batch_repeats():
    """16 slots from one 16-token prompt, every slot its own explicit tokens up to max_seq 2048, twice"""
    import torch
    m, _ = _model(max_seq=2048, seed=9, spec=False)
    c = m.cfg
    feed = torch.randint(0, c.vocab, (c.max_seq - 16, 16), generator=torch.Generator().manual_seed(3),
                         dtype=torch.int32).cuda()
    runs = []
    with _side_stream():
        m.reset()
        m.prefill(_seq(16, c.vocab, 18), 0.25)
        bt = _batch(m, 16)
        for _ in range(2):
            bt.fork()
            for j in range(feed.shape[0]):
                bt.step(feed[j], 0.25)
            torch.cuda.synchronize()
            runs.append([bt.logits(), _cpu(bt.buffer("POS"))] +
                        [bt.buffer(n, li, b) for b in range(16) for li in range(c.n_layers) for n in ("KCACHE", "VCACHE")])
    assert runs[0][1].tolist() == [c.max_seq] * 16
    for x, y in zip(*runs):
        if isinstance(x, np.ndarray):
            assert np.array_equal(x, y)
        else:
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_generate_batch_and_score_continuations(small):
    import torch
    m, _ = small
    c = m.cfg
    prompts = [_seq(6, c.vocab, 20), _seq(3, c.vocab, 21), _seq(6, c.vocab, 20)]
    samplers = [None, None, SAMPLER]
    with _side_stream():
        got = m.generate_batch(prompts, 5, 0.25, samplers)
        bt = _batch(m, 3)
        bt.set_sampler(2, **SAMPLER)
        for b in (0, 1, 2):
            m.reset()
            m.prefill(prompts[b], 0.25)
            bt.fork(b)
        want = [bt.next_tokens()]
        for _ in range(4):
            bt.step(None, 0.25)
            want.append(bt.next_tokens())
    assert got == [list(x) for x in zip(*want)]

    context = _seq(11, c.vocab, 22)
    conts = [_seq(4, c.vocab, 23), _seq(1, c.vocab, 24), _seq(7, c.vocab, 25)]
    with _side_stream():
        res = m.score_continuations(context, conts, 0.5)
        # step-level: one slot per continuation, teacher-forced, records read per position
        for k, t in enumerate(conts):
            bt = _batch(m, 1)
            bt.set_scoring(True)
            bt.set_score_targets(0, _i32([-1] * (len(context) - 1) + t))
            m.reset()
            m.prefill(context, 0.5)
            bt.fork(0)
            for j in range(len(t) - 1):
                bt.step(_i32([t[j]]), 0.5)
            _, rank, lp = bt.scores(0)
            sl = slice(len(context) - 1, len(context) - 1 + len(t))
            assert res[k][0] == float(lp[sl].cpu().double().sum()), k
            assert res[k][1] == bool((rank[sl] == 0).all()), k
        # a continuation's score does not depend on its companions
        alone = [m.score_continuations(context, [t], 0.5)[0] for t in conts]
        mixed = m.score_continuations(context, [conts[2], conts[0]], 0.5)
    assert alone == res
    assert mixed == [res[2], res[0]]
