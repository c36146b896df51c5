"""GPU: the device scorer (csrc/score.cuh, DESIGN.md section 4.7) against its CPU model (tests/score_model.py), inside
every decode path of the model, with greedy decoding and sampling left untouched, and the tools built on it."""
import ctypes as C
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests import score_model as M

pytestmark = pytest.mark.gpu

EINVAL = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hook(logits_np, targets):
    """records through the C-ABI hook (one launch, one CTA per target) as numpy (argmax, rank, logprob)"""
    import torch
    from effort_b200 import ops
    a, r, lp = ops.score(torch.from_numpy(np.ascontiguousarray(logits_np, np.float32)).cuda(),
                         torch.tensor(np.asarray(targets, np.int64), dtype=torch.int32, device="cuda"))
    return a.cpu().numpy(), r.cpu().numpy(), lp.cpu().numpy()


def _case(V, seed, inf=False):
    """random logits, half of them on a coarse grid, a maximum repeated three times, NaN and -inf entries; +inf with inf"""
    rng = np.random.default_rng(seed)
    l = (rng.standard_normal(V) * 2).astype(np.float32)
    h = rng.random(V) < 0.5
    l[h] = np.round(l[h] * 2) / 2
    if V >= 16:
        l[rng.choice(V, 3, replace=False)] = np.float32(l.max() + 0.5)
        l[rng.choice(V, max(2, V // 100), replace=False)] = np.nan
        l[rng.choice(V, max(2, V // 200), replace=False)] = -np.inf
        l[rng.choice(V, 4, replace=False)] = np.float32(-0.0)
    if inf:
        l[rng.choice(V, min(2, V), replace=False)] = np.inf
    return l


def _targets(l, rng, n=4096):
    V = len(l)
    mx = np.nanmax(np.where(np.isnan(l), -np.inf, l))
    special = np.concatenate([np.flatnonzero(l == mx), np.flatnonzero(np.isnan(l))[:64], np.flatnonzero(np.isinf(l))[:64],
                              np.flatnonzero(l == 0)[:16], [-1, V, V + 100, -7]])
    return np.concatenate([special, rng.integers(0, V, n - len(special))]).astype(np.int64)


@pytest.mark.parametrize("V", [1, 1000, 32000, 131072])
def test_hook_matches_model(V):
    rng = np.random.default_rng(V)
    worst = 0.0
    for seed, inf in ((1, False), (2, False), (3, True)):
        l = _case(V, seed + V, inf)
        t = _targets(l, rng)
        worst = max(worst, M.check(l, t, *_hook(l, t)))
    print(f"V={V}: max |logprob - float64| / bar = {worst:.3f}")


def test_degenerate_logits():
    F = np.float32
    for l in (np.full(100, np.nan, F), np.full(100, -np.inf, F), np.array([np.nan, -np.inf, 3.0, np.inf, np.inf], F),
              np.array([5.0], F), np.array([-0.0, 0.0, -0.0, -1.0], F), np.array([np.nan, -np.inf, -np.inf, np.nan], F)):
        t = np.concatenate([np.arange(len(l)), [-1, len(l)]])
        M.check(l, t, *_hook(l, t))


# ---- the model ---------------------------------------------------------------------------------------------------
def _small(flags=0, vocab=2048, max_seq=64):
    from effort_b200.model import DecodeModel, MistralConfig
    return DecodeModel.random_init(MistralConfig(n_layers=2, vocab=vocab, max_seq=max_seq), seed=7, weight_flags=flags)


@pytest.fixture(scope="module")
def small_model():
    return _small()


def _records_view(m):
    """a live int32 [max_seq, 3] view of the model's device records"""
    import torch
    from effort_b200.model import _tensor_from_ptr
    return _tensor_from_ptr(m._L.effort_model_scores(m._h), 3 * m.cfg.max_seq, torch.int32).view(m.cfg.max_seq, 3)


TOKENS = [1, 17, 400, None, 999, None, 5, 3]


def _check_steps(m, tokens, targets, effort=0.5):
    """step `tokens` from a reset with scoring on (None = self-fed) and check each step's record: the greedy argmax, and
    rank and logprob byte-identical to the hook on a copy of the step's logits; later records untouched"""
    import torch
    from effort_b200 import ops
    recs = _records_view(m)
    recs.fill_(0x5A5A5A5A)
    torch.cuda.synchronize()
    m.set_score_targets(torch.tensor(targets, dtype=torch.int32, device="cuda"))
    m.reset()
    out = []
    for p, t in enumerate(tokens):
        m.step(None if t is None else torch.tensor([t], dtype=torch.int32, device="cuda"), effort)
        torch.cuda.synchronize()
        rec = recs.clone()
        a, r, lp = ops.score(m.logits(), torch.tensor([targets[p] if p < len(targets) else -1], dtype=torch.int32,
                                                      device="cuda"))
        assert int(rec[p, 0]) == m.next_token() == int(a[0]), (p, rec[p].tolist(), m.next_token())
        assert int(rec[p, 1]) == int(r[0]), (p, int(rec[p, 1]), int(r[0]))
        assert rec[p, 2].item() == lp.view(torch.int32)[0].item(), p     # logprob bits
        assert bool((rec[p + 1:] == 0x5A5A5A5A).all()), p
        out.append(rec[p].tolist())
    return out


def _targets_for(m, n):
    V = m.cfg.vocab
    t = [(37 * p + 11) % V for p in range(n)]
    t[2], t[5] = -1, V + 3                          # no target
    return t


@pytest.mark.parametrize("use_graph,chain", [(False, 2), (True, 2), (True, 1)])
def test_every_step_scores_its_logits(small_model, use_graph, chain):
    m = small_model
    try:
        m.set_graphs(use_graph)
        m.set_chain(chain)
        m.set_scoring(True)
        _check_steps(m, TOKENS, _targets_for(m, len(TOKENS)))
        _check_steps(m, TOKENS, [3] * len(TOKENS))   # new targets, same captured graphs
    finally:
        m.set_scoring(False)
        m.set_chain(2)


def test_fused_glue_path():
    from effort_b200 import ops
    m = _small(ops.INPUT_MAJOR)
    ctx = ops.default_context()
    try:
        ctx.setOption("engine", 1)
        m.set_chain(1)
        m.set_fused_glue(True)
        m.set_scoring(True)
        for use_graph in (False, True):
            m.set_graphs(use_graph)
            _check_steps(m, TOKENS, _targets_for(m, len(TOKENS)))
    finally:
        ctx.setOption("engine", 2)


def test_moe_and_q4_paths():
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=1024, max_seq=32)
    for m in (DecodeModel.random_init_moe(cfg, n_experts=4, seed=9), DecodeModel.random_init_q4(cfg, seed=5)):
        m.set_scoring(True)
        for use_graph in (False, True):
            m.set_graphs(use_graph)
            _check_steps(m, TOKENS, _targets_for(m, len(TOKENS)))
        del m


def _run(m, tokens, effort=0.25):
    import torch
    out = []
    m.reset()
    for t in tokens:
        m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort)
        torch.cuda.synchronize()
        out.append((m.logits().cpu().numpy().tobytes(), m.next_token()))
    return out


def _launches_per_step(m):
    import torch
    from effort_b200 import ops
    m.reset()
    tok = torch.tensor([3], dtype=torch.int32, device="cuda")
    for _ in range(3):
        m.step(tok, 0.25)                            # eager, capture, replay
    torch.cuda.synchronize()
    n0 = ops.launchCount()
    m.step(tok, 0.25)
    torch.cuda.synchronize()
    return ops.launchCount() - n0


def test_greedy_untouched():
    import torch
    m = _small()
    m.set_graphs(True)
    toks = [1, 17, 400, 999, 5, 33]
    never = _run(m, toks)                            # a model that never scored
    m.set_score_targets(torch.tensor(toks[1:], dtype=torch.int32, device="cuda"))
    m.set_scoring(True)
    scored = _run(m, toks)
    m.set_scoring(False)
    cleared = _run(m, toks)
    assert never == scored == cleared
    off = _launches_per_step(m)
    m.set_scoring(True)
    on = _launches_per_step(m)
    m.set_scoring(False)
    assert on == off + 1, (off, on)


def test_with_a_sampler(small_model):
    import torch
    m = small_model
    m.set_graphs(True)
    prompt = [1, 17, 400]
    try:
        m.set_sampler(0.8, 50, 0.9, seed=21)
        plain = m.generate(prompt, 24)
        m.set_scoring(True)
        m.set_score_targets(None)
        m.reset()
        drawn, greedy = [], []
        for p in range(len(prompt) + 23):
            m.step(torch.tensor([prompt[p]], dtype=torch.int32, device="cuda") if p < len(prompt) else None, 0.25)
            torch.cuda.synchronize()
            if p >= len(prompt) - 1:
                drawn.append(m.next_token())
            greedy.append(M.argmax(m.logits().cpu().numpy()))
        assert drawn == plain
        a, r, lp = m.scores()
        n = len(greedy)
        assert a[:n].tolist() == greedy
        assert (r[:n] == -1).all() and torch.isnan(lp[:n]).all()   # no targets set
    finally:
        m.set_sampler(None)
        m.set_scoring(False)


def test_score_every_position_up_to_max_seq():
    """score() at every position up to max_seq, each record checked at 33 positions against the model on that step's
    logits, and two more score() runs over all max_seq positions byte-identical to each other and to the step-by-step
    records."""
    import torch
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=32000, max_seq=2048)
    m = DecodeModel.random_init(cfg, seed=11)
    rng = np.random.default_rng(5)
    seq = rng.integers(0, cfg.vocab, cfg.max_seq).tolist()
    pred, lp, rank = m.score(seq, 0.25)
    assert pred.shape == (2048,) and lp.shape == (2047,) and rank.shape == (2047,)
    assert m._scoring is False
    # step by step: each record against the model on that step's logits
    m.set_scoring(True)
    m.set_score_targets(torch.tensor(seq[1:], dtype=torch.int32, device="cuda"))
    m.reset()
    recs = _records_view(m)
    toks = torch.tensor(seq, dtype=torch.int32, device="cuda")
    worst = 0.0
    for p in range(cfg.max_seq):
        m.step(toks[p:p + 1], 0.25)
        if p % 64 == 0 or p == cfg.max_seq - 1:
            torch.cuda.synchronize()
            l = m.logits().cpu().numpy()
            t = [seq[p + 1]] if p + 1 < len(seq) else [-1]
            rec = recs[p].cpu()
            worst = max(worst, M.check(l, t, [int(rec[0])], [int(rec[1])], rec[2:3].view(torch.float32).numpy()))
    torch.cuda.synchronize()
    a, r, l = m.scores()
    assert int(r[2047]) == -1 and torch.isnan(l[2047])
    print(f"score(): 2048 positions, max |logprob - float64| / bar at 33 of them = {worst:.3f}")
    # every position: two score() runs and the step-by-step records agree byte for byte
    n = cfg.max_seq
    p1, l1, r1 = m.score(seq[:n], 0.25)
    p2, l2, r2 = m.score(seq[:n], 0.25)
    assert torch.equal(p1, p2) and torch.equal(r1, r2) and torch.equal(l1.view(torch.int32), l2.view(torch.int32))
    assert torch.equal(p1, pred[:n]) and torch.equal(r1, rank[:n - 1]) and torch.equal(l1.view(torch.int32), lp[:n - 1].view(torch.int32))
    assert torch.equal(a[:n].cpu(), p1) and torch.equal(r[:n - 1].cpu(), r1)
    # new targets between graph replays take effect without recapture
    m.set_scoring(True)
    m.set_score_targets(torch.tensor([int(p1[0])], dtype=torch.int32, device="cuda"))
    m.reset()
    m.step(toks[0:1], 0.25)
    torch.cuda.synchronize()
    assert int(recs[0, 1]) == 0 and int(recs[1, 1]) == int(r1[1])   # record 0 rewritten, record 1 untouched
    m.set_scoring(False)
    with pytest.raises(ValueError):
        m.score(seq + [1], 0.25)
    with pytest.raises(ValueError):
        m.score([], 0.25)


def test_choose_follows_limit_logits(small_model):
    m = small_model
    m.set_graphs(True)
    prompt = [5, 77, 300, 12]
    rng = np.random.default_rng(9)
    for effort in (1.0, 0.25):
        m.choose(prompt, [0], effort)
        l = m.logits().cpu().numpy()
        order = M.ranks(l, np.arange(m.cfg.vocab))
        by_rank = np.argsort(order)
        top3, far = by_rank[:3].tolist(), by_rank[500:504].tolist()
        cases = [(far + [top3[2]], 16, 4), (far + [top3[2], top3[0]], 16, 5), (far, 16, None), (far, 600, 0),
                 ([top3[1], top3[1]], 16, 0), ([-1, m.cfg.vocab, top3[0]], 16, 2), ([-1], 16, None),
                 (rng.integers(0, m.cfg.vocab, 8).tolist(), 16, "host")]
        for cand, top, want in cases:
            if want == "host":   # the reference's loop over the top-`top` list, first candidate found
                hit = [j for i in range(top) for j, c in enumerate(cand) if c == by_rank[i]]
                want = hit[0] if hit else None
            assert m.choose(prompt, cand, effort, top) == want, (effort, cand, top, want)


def test_invalid_arguments(small_model):
    import torch
    from effort_b200 import _lib, ops
    L = _lib.load()
    ctx = ops.default_context()
    lg = torch.zeros(16, dtype=torch.float32, device="cuda")
    tg = torch.zeros(4, dtype=torch.int32, device="cuda")
    out = torch.zeros(12, dtype=torch.int32, device="cuda")
    h = small_model._h
    assert L.effort_score(ctx._h, lg.data_ptr(), 16, tg.data_ptr(), 4, out.data_ptr(), None) == 0
    for args in ((None, lg.data_ptr(), 16, tg.data_ptr(), 4, out.data_ptr()), (ctx._h, None, 16, tg.data_ptr(), 4, out.data_ptr()),
                 (ctx._h, lg.data_ptr(), 16, None, 4, out.data_ptr()), (ctx._h, lg.data_ptr(), 16, tg.data_ptr(), 4, None),
                 (ctx._h, lg.data_ptr(), 0, tg.data_ptr(), 4, out.data_ptr()), (ctx._h, lg.data_ptr(), -1, tg.data_ptr(), 4, out.data_ptr()),
                 (ctx._h, lg.data_ptr(), 16, tg.data_ptr(), 0, out.data_ptr()), (ctx._h, lg.data_ptr(), 16, tg.data_ptr(), -2, out.data_ptr())):
        assert L.effort_score(*args, None) == EINVAL, args
    assert L.effort_model_set_scoring(None, 1) == EINVAL
    assert L.effort_model_set_score_targets(h, tg.data_ptr(), -1, None) == EINVAL
    assert L.effort_model_set_score_targets(h, tg.data_ptr(), small_model.cfg.max_seq + 1, None) == EINVAL
    assert L.effort_model_set_score_targets(h, None, 3, None) == EINVAL
    assert L.effort_model_set_score_targets(None, tg.data_ptr(), 3, None) == EINVAL
    assert L.effort_model_set_score_targets(h, None, 0, None) == 0
    assert L.effort_model_scores(None) is None
    with pytest.raises(_lib.EffortError):
        ops.score(lg, tg.long())
    with pytest.raises(_lib.EffortError):
        ops.score(lg, tg[:0])
    with pytest.raises(ValueError):
        small_model.choose([], [1])
    torch.cuda.synchronize()


# ---- tensor parallel (>= 2 GPUs) -----------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tp_worker(rank, world, port):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig, init_comm
    init_comm(ops.default_context(), rank, world)
    cfg = MistralConfig(n_layers=2, vocab=4096, max_seq=64)
    seq = [1, 17, 400, 999, 5, 33, 2, 4000]
    m = DecodeModel.random_init(cfg, seed=7, tp_rank=rank, tp_size=world)
    pred, lp, rk = m.score(seq, 0.5)
    mine = torch.cat([pred.double(), lp.double(), rk.double()]).cuda()
    every = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(every, mine)
    ok = int(all(torch.equal(e, mine) for e in every))
    if rank == 0:   # the unsharded model, on the logits the ranks all-gathered
        del m
        full = DecodeModel.random_init(cfg, seed=7)
        p1, l1, r1 = full.score(seq, 0.5)
        ok &= int(torch.equal(p1, pred) and torch.equal(r1, rk) and bool(torch.allclose(l1, lp, atol=1e-4)))
    flag = torch.tensor([ok], dtype=torch.int32, device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)          # every rank fails together
    dist.destroy_process_group()
    assert int(flag.item()) == 1


@pytest.mark.timeout(300)
def test_tensor_parallel_ranks_write_the_same_records():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.spawn(_tp_worker, args=(2, _free_port()), nprocs=2, join=True)


# ---- tools -----------------------------------------------------------------------------------------------------------
def _tool(name, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", name), *args], capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_token_match_tool():
    out = _tool("token_match.py", "--layers", "2", "--vocab", "1024", "--tokens", "40", "--prompt-len", "8",
                "--efforts", "1.0,0.5,0.1")
    assert out["positions"] == 48 and [r["effort"] for r in out["results"]] == [1.0, 0.5, 0.1]
    first = out["results"][0]   # effort 1.0 repeats the control, and the continuation is its own greedy choice
    assert first["match_pct"] == 100.0 and first["rank0_share"] == 1.0 and first["mean_logprob"] <= 0
    assert all(0 <= r["match_pct"] <= 100 and 0 <= r["rank0_share"] <= 1 for r in out["results"])
    assert "gpu" in out and "power_limit_w" in out


def test_score_cost_tool():
    out = _tool("score_cost.py", "--layers", "2", "--vocab", "1024", "--steps", "16", "--warmup", "4", "--rounds", "1",
                "--calls", "20")
    assert len(out["us_per_token"]["greedy"]) == len(out["us_per_token"]["scoring"]) == 1
    assert out["hook_us_per_call_v32000"] > 0 and "gpu" in out and "power_limit_w" in out
