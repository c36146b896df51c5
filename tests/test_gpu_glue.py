"""GPU: the decode loop's glue kernels (effort_b200/csrc/decode.cuh) -- rope + KV cache append + attention, the fused head
(final norm, lm_head, cross-CTA argmax), the generic path's add_rmsnorm / basic_mul / argmax, the MoE gate, and the
embedding's token clamp -- each checked after a real decode step on the inputs it consumed (DecodeModel.buffer)
against the float64 restatements of tests/glue_ref.py.  No upstream GEMV noise enters these comparisons, so the bars
hold at any effort, depth and position, up to max_seq and at the bench shape.

Bars (measured maxima over all tests in brackets, on H100 80GB HBM3 cards at 400 W and 700 W power limits):
  rope:    a rotated key pair keeps its norm within 8 fp32 ulps, 4.8e-7 [1.39e-7]; its angle matches pos*theta^(-j/64)
           within 2^-20*pos*freq_j + 1e-6 [0.113 of that bound]
  cache:   the V row equals the v GEMV output byte for byte; whole caches equal a host mirror of the rows each step wrote
  attn:    per head rel. L2 <= 1e-5 against float64 on the cached K/V [1.1e-6]
  head:    fused head logits rel. L2 <= 1e-4 against float64 W @ fp16(rmsNorm(h) * w) [3.05e-5, see HEAD_BAR];
           generic paths: rmsNorm(h) * w per element <= 1e-6 relative to fp32 [3.0e-7], logits <= 2e-6 against float64
           W @ fp16(normed) [2.1e-7]
  greedy:  the next token is the lowest index among the maximal non-NaN logits, at every step [bench run: 670 exact
           ties, 1378 unique maxima]
  gate:    expert indices exact (planted ties: the lower expert first; unplanted logits within 5e-4 of each other may
           swap [none did]), gate values <= 1e-4 absolute [3.4e-5, see GATE_VAL_BAR]
  state:   after a reset, stale cache rows change no logit bit; tokens outside [0, vocab) decode as token 0"""
from collections import defaultdict

import numpy as np
import pytest

from tests import glue_ref as G
from tests.ref_decode import rmsnorm_mul

pytestmark = pytest.mark.gpu

EFFORT = 0.25
ROPE_NORM_BAR = 8 * 2.0 ** -24
ATTN_BAR = 1e-5
# The fused head casts rmsNorm(h) * w to fp16 with a denominator from its own fp32 sum order (see the gate bars below):
# a few casts round the other way than the restatement's.  Measured: 7.6e-6 over the bench run, 3.05e-5 on the 2-layer
# vocab-4096 model run eagerly; without such flips the logits agree to ~2e-7 (the generic paths' basic_mul below).
HEAD_BAR = 1e-4
NORMED_BAR = 1e-6
BASIC_BAR = 2e-6
# The gate's input is fp16(rmsNorm(h) * w).  The kernel's fp32 sum of squares runs in another order than the
# restatement's, so the denominators can differ by a few ulps, and then a few of the 4096 fp16 casts round the other
# way; each such flip moves a gate logit by up to ~4e-5.  Measured: gate values 3.4e-5 off with 8 experts (one step of
# 64), 4.5e-7 and 2.5e-7 with 16 and 64.
GATE_VAL_BAR = 1e-4
GATE_TOL = 5e-4     # unplanted gate logits closer than this may come in either order


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


class Decode:
    """Steps a model from a reset through given tokens and checks, at every step, the kernels that only depend on the
    step's own inputs: the position, the K/V cache rows (V byte for byte, K by the rope check), the attention output and
    the greedy token.  Keeps a host mirror of every cache row the steps wrote and the maxima of the measured errors."""

    def __init__(self, m, fresh):
        import torch
        self.torch = torch
        self.m, c = m, m.cfg
        self.L, self.n_kv, self.S = c.n_layers, c.n_kv_heads, c.max_seq
        self.K = np.zeros((self.L, self.S, self.n_kv, 128), np.float32)
        self.V = np.zeros_like(self.K)
        self.fresh = fresh          # a model that never stepped: rows past the position must still be zero
        self.worst = defaultdict(float)
        self.pos = 0
        m.reset()

    def step(self, token, effort=EFFORT):
        torch, m, c, pos = self.torch, self.m, self.m.cfg, self.pos
        m.step(torch.tensor([token], dtype=torch.int32, device="cuda"), effort=effort)
        torch.cuda.synchronize()
        names = ("Q", "K", "V", "ATTN", "HIDDEN")
        parts = [m.buffer_view(n) for n in names]
        rows = [m.buffer_view(n, li).view(self.S, -1)[pos] for li in range(self.L) for n in ("KCACHE", "VCACHE")]
        flat = torch.cat(parts + rows).cpu().numpy()
        sizes = [p.numel() for p in parts] + [r.numel() for r in rows]
        xq, xk, xv, attn, hidden, *cache_rows = np.split(flat, np.cumsum(sizes)[:-1])
        pos_dev = int(m.buffer_view("POS").cpu()[0])
        logits = m.logits().cpu().numpy()
        nxt = m.next_token()
        assert pos_dev == pos + 1, (pos, pos_dev)
        for li in range(self.L):
            self.K[li, pos] = cache_rows[2 * li].reshape(self.n_kv, 128)
            self.V[li, pos] = cache_rows[2 * li + 1].reshape(self.n_kv, 128)
        assert np.array_equal(_u32(self.V[-1, pos].reshape(-1)), _u32(xv)), pos
        norm_err, angle_ratio = G.rope_check(xk, self.K[-1, pos].reshape(-1), pos, c.rope_theta)
        self.worst["rope_norm"] = max(self.worst["rope_norm"], norm_err)
        self.worst["rope_angle"] = max(self.worst["rope_angle"], angle_ratio)
        want = G.attention_step(xq, xk, self.K[-1], self.V[-1], pos)
        got = attn.reshape(c.n_heads, 128)
        self.worst["attn"] = max(self.worst["attn"], max(_rel(got[h], want[h]) for h in range(c.n_heads)))
        assert nxt == G.greedy(logits), (pos, nxt, G.greedy(logits))
        self.pos += 1
        return logits, hidden

    def check_caches(self):
        """every layer's whole K and V cache against the mirror: the rows written so far, and zeros past them"""
        for li in range(self.L):
            for name, mirror in (("KCACHE", self.K), ("VCACHE", self.V)):
                dev = self.m.buffer_view(name, li).cpu().numpy().reshape(self.S, self.n_kv, 128)
                assert np.array_equal(_u32(dev[: self.pos]), _u32(mirror[li, : self.pos])), (name, li, self.pos)
                if self.fresh:
                    assert not dev[self.pos:].any(), (name, li, self.pos)

    def check_head(self, logits, hidden, w64):
        """logits against float64 W @ the lm_head's input.  The fused head (chain 2) normalises h on load; the generic
        paths leave rmsNorm(h) * w in NORMED, checked against its fp32 restatement first."""
        torch, m = self.torch, self.m
        norm = m.head[0].cpu().numpy()
        normed = m.buffer("NORMED")
        if normed is None:
            x, bar, key = G.final_norm_fp16(hidden, norm, m.cfg.norm_eps), HEAD_BAR, "head"
        else:
            normed = normed.cpu().numpy()
            want = rmsnorm_mul(hidden, norm, m.cfg.norm_eps)
            err = np.abs(normed.astype(np.float64) - want) / np.maximum(np.abs(want), 1e-30)
            self.worst["normed"] = max(self.worst["normed"], float(err.max()))
            x, bar, key = normed.astype(np.float16).astype(np.float64), BASIC_BAR, "basic"
        ref = (w64 @ torch.from_numpy(x).cuda()).cpu().numpy()
        nan = np.isnan(ref)
        assert np.array_equal(np.isnan(logits), nan)
        self.worst[key] = max(self.worst[key], _rel(logits[~nan], ref[~nan]))
        return bar, key

    def assert_bars(self, extra=()):
        print({k: f"{v:.3g}" for k, v in self.worst.items()})
        assert self.worst["rope_norm"] <= ROPE_NORM_BAR, self.worst
        assert self.worst["rope_angle"] <= 1.0, self.worst
        assert self.worst["attn"] <= ATTN_BAR, self.worst
        if "normed" in self.worst:
            assert self.worst["normed"] <= NORMED_BAR, self.worst
        for bar, key in set(extra):
            assert self.worst[key] <= bar, self.worst


def _tokens(n, vocab, seed):
    return np.random.default_rng(seed).integers(0, vocab, n).tolist()


def test_bench_shape_every_position():
    """The bench configuration -- fused chain with graphs, vocab 32000, max_seq 2048, effort 0.25 -- on 2 layers, fed
    seeded tokens through every position 0..2047.  The lm_head's rows [8000, 16000) copy rows [0, 8000) and one row is
    fp16 NaN: duplicated rows must give bitwise equal logits (one warp per row, fixed order), the NaN row never wins,
    and exact ties (the lower index wins) and unique maxima must both occur many times across the 1056 CTAs' grid-stride
    loops and the last CTA's reduction."""
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=32000, max_seq=2048)
    m = DecodeModel.random_init(cfg, seed=31)
    gen = torch.Generator(device="cuda").manual_seed(32)
    W = (torch.randn((cfg.vocab, cfg.dim), generator=gen, device="cuda") * 0.02).half()
    W[8000:16000] = W[:8000]
    nan_row = 20011
    W[nan_row] = float("nan")
    m.set_head(m.head[0], W, m.head[2])
    w64 = W.double()
    m.set_graphs(True)
    d = Decode(m, fresh=True)
    head_at = set(range(10)) | {31, 32, 33, 63, 64, 65, 2046, 2047} | set(range(0, 2048, 128))
    ties = unique = 0
    extra = set()
    for pos, t in enumerate(_tokens(cfg.max_seq, cfg.vocab, 33)):
        logits, hidden = d.step(t)
        assert np.array_equal(_u32(logits[:8000]), _u32(logits[8000:16000])), pos
        assert np.isnan(logits[nan_row]), pos
        g = G.greedy(logits)
        ties += g < 8000
        unique += g >= 16000
        if pos in head_at:
            extra.add(d.check_head(logits, hidden, w64))
        if pos in (63, 1023, 2047):
            d.check_caches()
    assert m.buffer("NORMED") is None          # the fused chain ran
    with pytest.raises(Exception):
        m.step(None, effort=EFFORT)            # max_seq reached
    print(f"greedy: {ties} exact ties, {unique} unique maxima")
    assert ties >= 100 and unique >= 100, (ties, unique)
    d.assert_bars(extra)
    assert ops.default_context().errorFlag() == 0


@pytest.mark.parametrize("n_kv,theta,n_layers", [(32, 1e6, 1), (1, 1e4, 3)])
def test_gqa_ratios_and_rope_theta(n_kv, theta, n_layers):
    """GQA ratio 1 (32 KV heads) and 32 (one KV head) with rope theta 1e6 and 1e4, 300 positions of the fused chain;
    with the 2-layer bench test both parities of the chain's q/k/v buffers are read."""
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=n_layers, n_kv_heads=n_kv, rope_theta=theta, vocab=4096, max_seq=300)
    m = DecodeModel.random_init(cfg, seed=40 + n_kv)
    m.set_graphs(True)
    d = Decode(m, fresh=True)
    for pos, t in enumerate(_tokens(cfg.max_seq, cfg.vocab, n_kv)):
        d.step(t)
        if pos in (7, 40, 299):
            d.check_caches()
    assert m.buffer("NORMED") is None
    d.assert_bars()
    assert ops.default_context().errorFlag() == 0


@pytest.fixture(scope="module")
def paths_model():
    from effort_b200.model import DecodeModel, MistralConfig
    return DecodeModel.random_init(MistralConfig(n_layers=2, vocab=4096, max_seq=512), seed=51)


@pytest.mark.parametrize("path", ["chain2-eager", "chain1", "fused-glue", "q4"])
def test_other_token_paths(paths_model, path):
    """100 positions of each remaining token path with the attention, cache and head checks.  The generic paths (chain
    1, fused glue, Q4) also pin add_rmsnorm (NORMED) and basic_mul; the fused chain run eagerly must give the same
    logit bytes as its CUDA graphs over the first 64 positions."""
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    m = paths_model
    if path == "q4":
        m = DecodeModel.random_init_q4(MistralConfig(n_layers=1, vocab=4096, max_seq=128), seed=52)
    if path == "fused-glue":   # its round-1 kernels read input-major rows
        m = DecodeModel.random_init(MistralConfig(n_layers=2, vocab=4096, max_seq=128), seed=54,
                                    weight_flags=ops.INPUT_MAJOR)
    toks = _tokens(100, m.cfg.vocab, 53)
    graph_logits = []
    if path == "chain2-eager":
        m.set_graphs(True)
        d = Decode(m, fresh=False)
        graph_logits = [d.step(t)[0] for t in toks[:64]]
    try:
        m.set_graphs(path != "chain2-eager")
        m.set_chain(2 if path == "chain2-eager" else 1)
        m.set_fused_glue(path == "fused-glue")
        w64 = m.head[1].double()
        d = Decode(m, fresh=path in ("q4", "fused-glue"))
        extra = set()
        for pos, t in enumerate(toks):
            logits, hidden = d.step(t)
            extra.add(d.check_head(logits, hidden, w64))
            if pos < len(graph_logits):
                assert np.array_equal(_u32(logits), _u32(graph_logits[pos])), pos
        d.check_caches()
        assert (m.buffer("NORMED") is None) == (path == "chain2-eager")
        d.assert_bars(extra)
        assert ops.default_context().errorFlag() == 0
    finally:
        m.set_graphs(True)
        m.set_chain(2)
        m.set_fused_glue(False)
        torch.cuda.synchronize()


def _gate_ok(idx, lg, twin_of):
    """the GPU's two experts against the float64 gate logits: exactly the reference's top 2, except that unplanted
    logits within fp16-cast noise (GATE_TOL) of each other may come in either order.  A planted duplicate is a
    bitwise tie: its lower expert must be chosen, and first."""
    ref, _ = G.gate_top2(lg)
    if idx == ref:
        return True
    i0, i1 = idx
    if i0 == i1:
        return False
    for k, e in enumerate(idx):
        a = twin_of.get(e)
        if a is not None and a < e and a not in idx[:k]:
            return False
    return lg[i0] >= lg[ref[0]] - GATE_TOL and lg[i1] >= lg[ref[1]] - GATE_TOL and lg[i0] >= lg[i1] - GATE_TOL


@pytest.mark.parametrize("n_experts,hidden_dim", [(8, 14336), (16, 14336), (64, 4096)])
def test_moe_gate(n_experts, hidden_dim):
    """moe_gate_kernel over 8 experts (one per warp), 16 and the C-ABI maximum 64 (warp w takes w, w+8, ...), 64
    positions.  Gate rows [E/2, E/2 + E/4) copy rows [0, E/4), so that the top 2 is an exact tie about half the time."""
    import torch
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=1, hidden_dim=hidden_dim, vocab=1024, max_seq=64)
    m = DecodeModel.random_init_moe(cfg, n_experts=n_experts, seed=60 + n_experts)
    gen = torch.Generator(device="cuda").manual_seed(61)
    gate = (torch.randn((n_experts, cfg.dim), generator=gen, device="cuda") * 0.02).half()
    twin_of = {}
    for a in range(n_experts // 4):
        gate[n_experts // 2 + a] = gate[a]
        twin_of[n_experts // 2 + a], twin_of[a] = a, n_experts // 2 + a
    m.set_moe(0, gate)
    gate_np = gate.cpu().numpy()
    ffn_norm = m.layers[0][8].cpu().numpy()
    m.set_graphs(True)
    d = Decode(m, fresh=True)
    planted = high = noisy = 0
    worst_val = 0.0
    for pos, t in enumerate(_tokens(cfg.max_seq, cfg.vocab, 62)):
        d.step(t)
        h_keep = m.buffer("GATE_IN").cpu().numpy()
        idx = tuple(int(i) for i in m.buffer("GATE_IDX").cpu())
        val = m.buffer("GATE_VAL").cpu().numpy()
        lg = G.gate_logits(h_keep, ffn_norm, gate_np, cfg.norm_eps)
        assert _gate_ok(idx, lg, twin_of), (pos, idx, G.gate_top2(lg)[0], lg[list(idx)])
        noisy += idx != G.gate_top2(lg)[0]
        planted += twin_of.get(idx[0]) == idx[1]
        high += max(idx) >= 8
        e = np.exp(lg[list(idx)])
        worst_val = max(worst_val, float(np.max(np.abs(val - e / e.sum()))))
    d.check_caches()
    print(f"gate: {planted} planted ties, {high} steps routed past expert 7, {noisy} near ties in another order, "
          f"worst gate value {worst_val:.3g}")
    assert planted >= 5, planted
    assert n_experts == 8 or high >= 5, high
    assert worst_val <= GATE_VAL_BAR, worst_val
    d.assert_bars()
    assert ops.default_context().errorFlag() == 0


def test_reset_and_token_clamp(paths_model):
    """effort_model_reset only rewinds the position: after 500 tokens of another sequence, the stale cache rows past
    the position must not change a fresh sequence's logits by a single bit.  embed_kernel maps tokens outside
    [0, vocab) to token 0."""
    import torch
    from effort_b200 import ops
    m = paths_model
    m.set_graphs(True)
    V = m.cfg.vocab

    def run(toks):
        m.reset()
        out = []
        for t in toks:
            m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort=EFFORT)
            out.append(m.logits())
        torch.cuda.synchronize()
        return [_u32(x.cpu().numpy()) for x in out]

    b = _tokens(40, V, 71)
    first = run(b)
    run(_tokens(500, V, 72))
    again = run(b)
    for pos, (x, y) in enumerate(zip(first, again)):
        assert np.array_equal(x, y), pos
    zero = run([0])[0]
    for bad in (-1, V, V + 100):
        assert np.array_equal(run([bad])[0], zero), bad
    assert ops.default_context().errorFlag() == 0
