"""GPU: the decode-loop mirror (effort_model_*, runNetwork.swift:113-209) against the CPU restatement built on
the oracle's bucketMul, on a 2-layer model of the Mistral-7B layer shape."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.ref_decode import RefModel

pytestmark = pytest.mark.gpu


def _cpu(t):
    return t.cpu().numpy()


def _restatements(layers, head):
    """The CPU restatement in both of its summation forms: the sequential oracle (float64 sums) and its OpenMP port
    (float32 sums, as on the device).  They alone can differ by more than the decode bars below: in bisect mode a
    last-bit change of one layer's output moves the next layer's bisection cutoff, and the two forms drift to cos-sim
    0.998 on the 2-layer model after one token.  A decoded token must match one of them within the bar.

    Measured on an H100 (first token, the 2-layer model of `_small`): bisect mode (engines 1 and 2), GPU vs float64
    oracle 0.998189, GPU vs float32 port 1.000000, oracle vs port 0.998189; select mode 1.000000 for all three.  The MoE
    model against the float64 oracle alone: 0.99928 on its first token."""
    return RefModel(layers, *head), RefModel(layers, *head, fast=True)


def _reset(refs):
    for r in refs:
        r.pos, r.kc, r.vc = 0, [[] for _ in r.layers], [[] for _ in r.layers]


def _cossim_best(got, refs, token, effort):
    return max(O.cossim(got, r.step(token, effort)) for r in refs)


def _small(flags):
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=2048, max_seq=64)
    m = DecodeModel.random_init(cfg, seed=7, keep_reference_layout=True, weight_flags=flags)
    names = ["wq", "wk", "wv", "wo", "w1", "w2", "w3"]
    layers = []
    for L in m.layers:
        d = {}
        for n, ew in zip(names, L[:7]):
            d[n] = {"buckets": _cpu(ew.buckets), "stats": _cpu(ew.stats), "probes": _cpu(ew.probes), "in": ew.inSize,
                    "out": ew.outSize}
        d["attn_norm"], d["ffn_norm"] = _cpu(L[7]), _cpu(L[8])
        layers.append(d)
    return m, _restatements(layers, [_cpu(t) for t in m.head[:3]])


@pytest.fixture(scope="module")
def small_model():
    return _small(0)


@pytest.fixture(scope="module")
def small_model_input_major():
    """device copy input-major: what the round-1 engine (and the per-warp cp.async rings of round 2) read"""
    from effort_b200 import ops
    return _small(ops.INPUT_MAJOR)


@pytest.fixture(autouse=True)
def _select_mode():
    """the decode loop runs the operator in its default cutoff mode"""
    with O.cutoff_mode("select"):
        yield


# chain 2 = the fused round-2 chain (default), chain 1 = one kernel per reference op; engine 1 = round-1 kernels
@pytest.mark.parametrize("use_graph,chain,engine,fused_glue", [(False, 2, 2, False), (True, 2, 2, False), (True, 1, 2, False),
                                                               (False, 1, 1, False), (True, 1, 1, True)])
def test_decode_matches_cpu_restatement(small_model, small_model_input_major, use_graph, chain, engine, fused_glue):
    import torch
    from effort_b200 import ops
    m, refs = small_model_input_major if engine == 1 else small_model
    ctx = ops.default_context()
    try:
        ctx.setOption("engine", engine)
        if engine == 1:
            ctx.setCutoffMode("bisect")
            O.set_cutoff_mode("bisect")
        m.set_graphs(use_graph)
        m.set_chain(chain)
        m.set_fused_glue(fused_glue)
        m.reset()
        _reset(refs)
        toks = [1, 17, 400, 999, 5]
        for t in toks:
            tok = torch.tensor([t], dtype=torch.int32, device="cuda")
            m.step(tok, effort=0.5)
            torch.cuda.synchronize()
            got = m.logits().cpu().numpy()
            cs = _cossim_best(got, refs, t, 0.5)
            assert cs > 0.9995, cs     # tiny selection flips (fp32 reorder of v near the cutoff) allowed
            assert m.next_token() == int(np.argmax(got))
        assert ctx.errorFlag() == 0
    finally:
        ctx.setOption("engine", 2)
        ctx.setCutoffMode("select")
        m.set_chain(2)
        m.set_fused_glue(False)


def test_step_past_max_seq_is_refused(small_model):
    """the KV cache holds max_seq positions: the next step is an error, not an out-of-bounds write (ADVICE r1)"""
    import torch
    from effort_b200 import EffortError
    m, _ = small_model
    m.set_graphs(True)
    m.reset()
    tok = torch.tensor([1], dtype=torch.int32, device="cuda")
    m.step(tok, effort=0.25)
    for _ in range(m.cfg.max_seq - 1):
        m.step(None, effort=0.25)
    torch.cuda.synchronize()
    with pytest.raises(EffortError):
        m.step(None, effort=0.25)
    m.reset()
    m.step(tok, effort=0.25)      # usable again after a reset
    torch.cuda.synchronize()


def test_32_layers_and_long_context():
    """BASELINE configs[1] shape: all 32 layers against the CPU restatement (OpenMP port of the oracle), a few tokens.
    Effort 1.0 is a smooth function of the weights, so 32 layers must agree tightly.  At effort 0.25 the selection is a
    hard threshold: an fp32-rounding difference that moves one row across the cutoff changes a layer's output by
    ~1e-3, and on iid-Gaussian random weights such flips compound from layer to layer (two CPU runs of the SAME
    restatement that differ only in their fp32 summation order drift to cos-sim 0.996 after 32 layers, measured with
    3 vs 8 OpenMP threads), so the deep low-effort comparison is reported and bounded loosely; the tight low-effort
    bars are the per-operator tests and the 2-layer decode test.  Then positions >= 1024 (attention over a long KV
    cache) stay finite and self-consistent."""
    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=32, vocab=4096, max_seq=1100)
    m = DecodeModel.random_init(cfg, seed=21, keep_reference_layout=True)
    names = ["wq", "wk", "wv", "wo", "w1", "w2", "w3"]
    layers = []
    for L in m.layers:
        d = {n: {"buckets": _cpu(ew.buckets), "stats": _cpu(ew.stats), "probes": _cpu(ew.probes), "in": ew.inSize, "out": ew.outSize}
             for n, ew in zip(names, L[:7])}
        d["attn_norm"], d["ffn_norm"] = _cpu(L[7]), _cpu(L[8])
        layers.append(d)
    ref = RefModel(layers, _cpu(m.head[0]), _cpu(m.head[1]), _cpu(m.head[2]), fast=True)
    worst = {}
    for effort in (1.0, 0.25):
        m.reset()
        ref.pos, ref.kc, ref.vc = 0, [[] for _ in ref.layers], [[] for _ in ref.layers]
        w = 1.0
        for t in (1, 77, 2049):
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=effort)
            torch.cuda.synchronize()
            got = m.logits().cpu().numpy()
            want = ref.step(t, effort)
            assert np.isfinite(got).all()
            w = min(w, O.cossim(got, want))
        worst[effort] = w
    print("32-layer decode, worst logit cos-sim vs the CPU restatement:", worst)
    assert worst[1.0] > 0.9995, worst
    assert worst[0.25] > 0.5, worst          # see the docstring: chaotic regime on iid-Gaussian weights
    del ref, layers
    m.reset()
    m.step(torch.tensor([1], dtype=torch.int32, device="cuda"), effort=0.25)
    for _ in range(1050):
        m.step(None, effort=0.25)
    torch.cuda.synchronize()
    lg = m.logits().cpu().numpy()
    assert np.isfinite(lg).all()
    assert m.next_token() == int(np.argmax(lg))


def test_step_host_and_self_feeding(small_model):
    import torch
    m, _ = small_model
    m.set_graphs(True)
    m.reset()
    logits = np.zeros(m.cfg.vocab, np.float32)
    t = m.step_host(3, effort=0.25, logits=logits)
    assert t == int(np.argmax(logits))
    seq_a = [t]
    for _ in range(5):
        t = m.step_host(None, effort=0.25)
        seq_a.append(t)
    m.reset()
    t = m.step_host(3, effort=0.25)
    seq_b = [t]
    for _ in range(5):
        t = m.step_host(None, effort=0.25)
        seq_b.append(t)
    assert seq_a == seq_b                                  # same greedy continuation (argmax gaps >> fp32 reorder noise)


def test_model_directory_roundtrip(tmp_path):
    """convert -> bucketed-safetensors directory -> load (C-ABI loader and Python reader) -> decode: the loaded models
    reproduce the in-memory model of the same seed (same weights); a percentLoad-truncated load
    (loader.swift:113-166) runs and correlates."""
    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=1, vocab=1024, max_seq=32)
    index = DecodeModel.convert_random_to_directory(str(tmp_path), cfg, seed=11)
    assert index.endswith("buckets-FP16.safetensors.index.json")
    mem = DecodeModel.random_init(cfg, seed=11)
    models = {"native": DecodeModel.from_directory(str(tmp_path), cfg, native=True),
              "python": DecodeModel.from_directory(str(tmp_path), cfg, native=False),
              "load8": DecodeModel.from_directory(str(tmp_path), cfg, percent_load=8)}
    outs = {}
    for name, m in [("mem", mem)] + list(models.items()):
        m.set_graphs(False)
        m.reset()
        seq = []
        for t in (3, 500, 77):
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=0.25)
            torch.cuda.synchronize()
            seq.append(m.logits().cpu().numpy())
        outs[name] = seq
    for name in ("native", "python"):   # same weights in separately converted copies
        for a, b in zip(outs["mem"], outs[name]):
            assert O.cossim(a, b) > 0.999999, name
    # percentLoad 8 drops ranks 8..15.  On iid-Gaussian weights those ranks ARE selected at effort 0.25 (the row means
    # fall slowly with rank), so the truncated model only correlates with the full one (measured 0.86 on the first
    # token); real Mistral weights are what the reference's percentLoad knob is for (loader.swift:113-166).
    assert all(np.isfinite(x).all() for x in outs["load8"])
    assert O.cossim(outs["mem"][0], outs["load8"][0]) > 0.7


def test_q4_decode_matches_cpu_restatement():
    """BASELINE configs[2]: a Q4 model (bucketMulQ4 for wq/w1/w2/w3, dense core fallback for wk/wv/wo,
    q4_convert.py:53) through the C++ token loop against the CPU restatement on the oracle's Q4 operators, effort 0.5."""
    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=1, vocab=1024, max_seq=32)
    m = DecodeModel.random_init_q4(cfg, seed=5, keep_tensors=True)
    d = {}
    for n, ew in zip(["wq", "wk", "wv", "wo", "w1", "w2", "w3"], m.layers[0][:7]):
        if hasattr(ew, "q4_tensors"):
            t = ew.q4_tensors
            d[n] = {"kind": "q4", "buckets": _cpu(t["buckets"]), "stats": _cpu(t["bucket.stats"]), "probes": _cpu(t["probes"]),
                    "outliers": _cpu(t["outliers"]), "in": ew.inSize, "out": ew.outSize}
        else:
            d[n] = {"kind": "core", "core": _cpu(ew.dense), "in": ew.inSize, "out": ew.outSize}
    d["attn_norm"], d["ffn_norm"] = _cpu(m.layers[0][7]), _cpu(m.layers[0][8])
    ref = RefModel([d], _cpu(m.head[0]), _cpu(m.head[1]), _cpu(m.head[2]))
    for use_graph in (False, True):
        m.set_graphs(use_graph)
        m.reset()
        ref.pos, ref.kc, ref.vc = 0, [[]], [[]]
        for t in (1, 17, 400):
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=0.5)
            torch.cuda.synchronize()
            got = m.logits().cpu().numpy()
            want = ref.step(t, 0.5)
            assert O.cossim(got, want) > 0.9995
            assert m.next_token() == int(np.argmax(got))


def test_moe_decode_matches_cpu_restatement():
    """Mixtral-style routing (runNetwork.swift:185-200): dense gate, top-2 on the device, the expert index reaches the
    GEMVs as a device scalar (expNo), outputs weighted by the softmaxed gate values -- against the CPU restatement."""
    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=1024, max_seq=32)
    m = DecodeModel.random_init_moe(cfg, n_experts=4, seed=9)
    layers = []
    for L in m.layers:
        d = {}
        for n, ew in zip(["wq", "wk", "wv", "wo", "w1", "w2", "w3"], L[:7]):
            d[n] = {"buckets": _cpu(ew.buckets), "stats": _cpu(ew.stats), "probes": _cpu(ew.probes), "in": ew.inSize,
                    "out": ew.outSize, "n_experts": ew.numExperts}
        d["attn_norm"], d["ffn_norm"], d["gate"] = _cpu(L[7]), _cpu(L[8]), _cpu(L[9])
        layers.append(d)
    refs = _restatements(layers, [_cpu(t) for t in m.head[:3]])
    for use_graph in (False, True):
        m.set_graphs(use_graph)
        m.reset()
        _reset(refs)
        for t in (1, 17, 400):
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=0.5)
            torch.cuda.synchronize()
            got = m.logits().cpu().numpy()
            assert _cossim_best(got, refs, t, 0.5) > 0.9995
            assert m.next_token() == int(np.argmax(got))
