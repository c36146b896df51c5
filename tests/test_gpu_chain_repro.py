"""GPU: long fused-chain decodes repeat bit for bit (DESIGN.md section 4.7).

The model of the original report: 2 layers, vocabulary 32000, 2048 positions, effort 0.25, the default context (select
cutoff, bulk staging, cutoff hints on, L2 prefetch off), CUDA graphs replayed on a side stream.  One teacher-forced decode with scoring off is
the reference; every other run is compared with it byte for byte, on the device, at every step: logits, greedy token,
score records, and every K/V row of both layers.

The budgets are fixed; section 4.7 gives this file's mismatch counts with the fix of that section reverted and applied.
The launch-level test pins the fix directly: every launch group of the chain, repeated with a cutoff hint far from
the launch's own cutoff (which CTA 0 then rewrites mid-launch), must give the hint-off bytes."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import oracle as O
from tools import chain_repro as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POSITIONS = (1200, 1500, 1750, 2047)
REPEATS = 4096
EINVAL = -1


_STREAM = []


@pytest.fixture(autouse=True)
def _select_mode():
    """select cutoff, on one side stream for the whole module: the model captures and replays its graphs only there"""
    if not _STREAM:
        _STREAM.append(torch.cuda.Stream())
    with O.cutoff_mode("select"), torch.cuda.stream(_STREAM[0]):
        yield


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """the modules after this one start with the device memory they would have had without it"""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def setup():
    if not _STREAM:
        _STREAM.append(torch.cuda.Stream())
    with O.cutoff_mode("select"), torch.cuda.stream(_STREAM[0]):
        m = R.make_model()
        toks = R.sequence(m)
        ref = R.Reference(m, toks)
    yield m, toks, ref
    m.set_scoring(False)
    m.set_sampler(None)


def _decode(m, ref, toks, scoring, sampler):
    """one whole teacher-forced decode; the steps whose logits (greedy token, record) differ, the K/V rows that differ"""
    m.set_scoring(scoring)
    m.set_sampler(0.8 if sampler else None, top_k=40, seed=3)
    if scoring:
        m.set_score_targets(ref.targets)
        ref.views.rec.fill_(0x5A5A5A5A)
    assert torch.cuda.current_stream().cuda_stream != 0
    S = m.cfg.max_seq
    bad = torch.zeros(S, dtype=torch.bool, device="cuda")
    m.reset()
    for p in range(S):
        m.step(toks[p:p + 1], R.EFFORT)
        bad[p] = R._step_bad(ref, ref.views, p, scoring, greedy=not sampler)
    rows = torch.zeros(S, dtype=torch.bool, device="cuda")
    for t, r in zip(ref.views.caches(m), ref.kv):
        rows |= (t != r).any(dim=1)
    torch.cuda.synchronize()
    return bad.nonzero().flatten().tolist(), rows.nonzero().flatten().tolist()


@pytest.mark.parametrize("scoring,sampler,runs", [(True, False, 4), (False, True, 2), (True, True, 2)],
                         ids=["scoring", "sampler", "both"])
def test_whole_decode_matches_reference(setup, scoring, sampler, runs):
    """whole 2048-token decodes with the scorer, the sampler or both after the head: greedy logits, the greedy token
    (scoring runs), every record against effort_score on the reference logits, and every K/V row, byte for byte"""
    from effort_b200 import ops
    m, toks, ref = setup
    try:
        for run in range(runs):
            steps, rows = _decode(m, ref, toks, scoring, sampler)
            assert not steps and not rows, f"run {run}: {len(steps)} steps differ (first {steps[:4]}), K/V rows {rows[:8]}"
        assert ops.default_context().errorFlag() == 0
    finally:
        m.set_scoring(False)
        m.set_sampler(None)


@pytest.mark.parametrize("steps", [2, 1], ids=["from-previous-step", "alone"])
def test_step_repeats_match_reference(setup, steps):
    """step p repeated 4096 times from the reference state, at four positions, scoring on, graphs replayed.  from-previous-step:
    each repeat runs step p - 1 first, so step p starts from the cutoff hints step p - 1 left, as in a decode.  alone:
    the repeats of step p start from its own hints"""
    m, toks, ref = setup
    m.set_scoring(True)
    try:
        report = {}
        for p in POSITIONS:
            n, first, flag = R.repeat_steps(m, ref, toks, p, REPEATS, steps=steps)
            report[p] = (n, first)
            assert flag == 0, (p, flag)
        print(f"steps={steps}: bad repeats (count, first) per position {report}")
        assert all(n == 0 for n, _ in report.values()), report
    finally:
        m.set_scoring(False)


def test_step_repeats_without_hint(setup):
    """the same repeats with the cutoff hint off (and with it the L2 prefetch that reads it) -- the knob that removed
    the divergence before the fix"""
    from effort_b200 import ops
    m, toks, ref = setup
    ctx = ops.default_context()
    try:
        ctx.setOption("hint", 0)
        m.set_scoring(False)  # drops the captured graphs: they hold the hint pointers
        m.set_scoring(True)
        report = {p: R.repeat_steps(m, ref, toks, p, REPEATS // 4)[:2] for p in POSITIONS}
        print(f"hint off: bad repeats (count, first) per position {report}")
        assert all(n == 0 for n, _ in report.values()), report
    finally:
        ctx.setOption("hint", 1)
        m.set_scoring(False)


def test_step_repeats_with_prefetch(setup):
    """the repeats with the L2 prefetch on: its warps load the hint early in the launch, and before the fix this made
    mixed hints inside a CTA the rule rather than the exception"""
    from effort_b200 import ops
    m, toks, ref = setup
    ctx = ops.default_context()
    try:
        ctx.setOption("prefetch", 1)
        m.set_scoring(False)  # drops the captured graphs: they hold the prefetch flag
        m.set_scoring(True)
        report = {p: R.repeat_steps(m, ref, toks, p, REPEATS // 4)[:2] for p in POSITIONS}
        print(f"prefetch on: bad repeats (count, first) per position {report}")
        assert all(n == 0 for n, _ in report.values()), report
    finally:
        ctx.setOption("prefetch", 0)
        m.set_scoring(False)


LAUNCH_REPEATS = 2048


@pytest.mark.parametrize("prefetch", [0, 1])
def test_launch_groups_with_a_stale_hint(setup, prefetch):
    """each launch group of the chain on a real step's inputs (layer 1 after step 2047): [q,k,v] with rmsNorm on load,
    wo accumulating, [w1,w3] with rmsNorm on load, w2 with silu on load.  The output with the hint off is the reference.
    Then each group is repeated with its matrices' hints set 8x above or below their own cutoffs (the search's bracket
    misses; CTA 0 rewrites the hint while the other CTAs read it), accumulating into the same prior each time: every
    repeat must give the reference bytes"""
    from effort_b200 import ops
    m, toks, ref = setup
    ctx = ops.default_context()
    wq, wk, wv, wo, w1, w2, w3, attn_norm, ffn_norm = m.layers[1][:9]
    m.set_scoring(False)
    m.rewind(m.cfg.max_seq - 1)
    m.step(toks[-1:], R.EFFORT)
    h, attn = m.buffer("HIDDEN"), m.buffer("ATTN")
    z = lambda w: torch.zeros(w.outSize, dtype=torch.float32, device="cuda")  # noqa: E731
    x1, x3 = z(w1), z(w3)
    groups = {
        "qkv": [dict(v=h, by=w, out=z(w), norm=attn_norm, effort=R.EFFORT, accumulate=True) for w in (wq, wk, wv)],
        "wo": [dict(v=attn, by=wo, out=h.clone(), effort=R.EFFORT, accumulate=True)],
        "w1w3": [dict(v=h, by=w, out=o, norm=ffn_norm, effort=R.EFFORT, accumulate=True) for w, o in ((w1, x1), (w3, x3))],
        "w2": [dict(v=x1, x3=x3, by=w2, out=h.clone(), effort=R.EFFORT, accumulate=True)],
    }
    report = {}
    try:
        ctx.setOption("prefetch", prefetch)
        for name, calls in groups.items():
            priors = [c["out"].clone() for c in calls]

            def launch():
                for c, pr in zip(calls, priors):
                    c["out"].copy_(pr)
                ops.fusedMulBatch(calls)
            ctx.setOption("hint", 0)
            launch()
            want = [c["out"].clone() for c in calls]
            ctx.setOption("hint", 1)
            launch()  # leaves each matrix's own cutoff in its hint
            hints = [c["by"].hint() for c in calls]
            own = [t.clone() for t in hints]
            bad = torch.zeros((), dtype=torch.int32, device="cuda")
            for i in range(LAUNCH_REPEATS):
                for t, o in zip(hints, own):
                    t.copy_(o * (8.0 if i % 2 == 0 else 0.125))
                launch()
                for c, w in zip(calls, want):
                    bad += (c["out"].view(torch.int32) != w.view(torch.int32)).any().to(torch.int32)
            report[name] = int(bad)
            if name == "w1w3":  # w2 reads what this group produced, as in the chain
                for c, w in zip(calls, want):
                    c["out"].copy_(w)
        print(f"prefetch={prefetch}: launches that differ from the hint-off bytes {report}")
        assert ctx.errorFlag() == 0
        assert all(n == 0 for n in report.values()), report
    finally:
        ctx.setOption("hint", 1)
        ctx.setOption("prefetch", 0)


def test_step_repeats_plain_stream_order():
    """EFFORT_PDL=0 (read once per process, so in a subprocess): the chain in plain stream order repeats its steps too"""
    env = dict(os.environ, EFFORT_PDL="0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "chain_repro.py"), "--repeats", "512",
                        "--positions", ",".join(map(str, POSITIONS))], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    import json
    out = json.loads(r.stdout.strip().splitlines()[-1])
    print(out)
    assert out["pdl"] is False  # what the library itself reports
    assert all(v["bad"] == 0 and v["err_flag"] == 0 for v in out["positions"].values()), out


def test_rewind_limits(setup):
    from effort_b200._lib import EffortError
    m, toks, ref = setup
    assert m._L.effort_model_rewind(None, 0, None) == EINVAL
    for pos in (-1, m.cfg.max_seq, m.cfg.max_seq + 5):
        with pytest.raises(EffortError):
            m.rewind(pos)
    # rewinding to 0 is a reset; the last position is allowed and a step there fills the cache
    m.set_scoring(False)
    m.rewind(m.cfg.max_seq - 1)
    m.step(toks[-1:], R.EFFORT)
    with pytest.raises(EffortError):
        m.step(toks[-1:], R.EFFORT)
    m.rewind(0)
    m.step(toks[:1], R.EFFORT)
    torch.cuda.synchronize()
    assert bool((ref.views.logits == ref.logits[0]).all())
    assert int(m.buffer("POS")[0]) == 1
