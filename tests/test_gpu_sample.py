"""GPU: the device sampler (csrc/sample.cuh, DESIGN.md section 4.6) against its CPU model (tests/sampler_model.py),
inside every decode path of the model, and with greedy decoding left untouched."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
from scipy import stats

from tests import sampler_model as S

pytestmark = pytest.mark.gpu

EINVAL = -1


def _logits(V, seed, ties=False, nans=False):
    rng = np.random.default_rng(seed)
    l = (rng.standard_normal(V) * 2).astype(np.float32)
    if ties:      # half the vocabulary on a coarse grid: long runs of equal logits, also at the top
        h = rng.random(V) < 0.5
        l[h] = np.round(l[h] * 2) / 2
    if nans and V > 4:
        l[rng.choice(V, max(1, V // 100), replace=False)] = np.nan
        l[rng.choice(V, max(1, V // 200), replace=False)] = -np.inf
        l[1] = np.nan
    return l


def _hook_draws(logits_np, T, K, P, seed, positions):
    """device draws for each position through the C-ABI hook (one launch each, into one device buffer)"""
    import torch
    from effort_b200 import _lib, ops
    ctx = ops.default_context()
    lg = torch.from_numpy(logits_np).cuda()
    out = torch.empty(len(positions), dtype=torch.int32, device="cuda")
    prm = _lib.Sampler(T, K, P, seed)
    sp = ops._stream_ptr()
    for j, p in enumerate(positions):
        _lib.check(ctx._L.effort_sample(ctx._h, lg.data_ptr(), lg.numel(), C.byref(prm), int(p), out[j:j + 1].data_ptr(), sp),
                   "effort_sample")
    return out.cpu().numpy().astype(np.int64)


CASES = [  # (T, K, P, ties, nans)
    (1.0, 0, 1.0, False, False),
    (0.8, 50, 0.9, False, False),
    (1.5, 0, 0.7, True, False),
    (0.6, 7, 1.0, True, True),
    (1.0, 300, 0.95, True, True),
    (2.0, 1, 1.0, True, False),
]


@pytest.mark.parametrize("V", [1, 1000, 32000, 131072])
def test_hook_matches_model(V):
    positions = np.arange(2048)
    seed = 0x1234_5678_9ABC
    report = []
    for ci, (T, K, P, ties, nans) in enumerate(CASES):
        l = _logits(V, 100 + ci, ties, nans)
        got = _hook_draws(l, T, K, P, seed + ci, positions)
        prep = S.prepare(l, T, K, P)
        want = S.draw(prep, seed + ci, positions)
        bad = got != want
        near = S.near_boundary(prep, seed + ci, positions)
        assert not np.any(bad & ~near), (V, T, K, P, np.flatnonzero(bad & ~near)[:8])
        assert bad.sum() <= len(positions) // 100, (V, T, K, P, int(bad.sum()))
        report.append(int(bad.sum()))
    print(f"V={V}: draws differing from the model within 1e-6 of a boundary, per case: {report}")
    # a near-uniform weight (T = 1e4) leaves every member of S_k drawable: S_k itself is exact, no exception
    l = _logits(V, 7, ties=True, nans=True)
    for K in (1, 10, 1000):
        prep = S.prepare(l, 1e4, K, 1.0)
        got = _hook_draws(l, 1e4, K, 1.0, 99, positions)
        assert set(got.tolist()) <= set(prep.sk.tolist()) if prep.greedy is None else set(got.tolist()) == {prep.greedy}


def test_degenerate_logits():
    import torch
    from effort_b200 import ops
    cases = [(np.full(100, np.nan, np.float32), 0), (np.full(100, -np.inf, np.float32), 0),
             (np.array([np.nan, -np.inf, 3.0, np.inf, np.inf], np.float32), 3), (np.array([5.0], np.float32), 0)]
    for l, want in cases:
        for pos in (0, 1, 77):
            assert int(ops.sample(torch.from_numpy(l).cuda(), 0.7, 0, 0.9, seed=3, position=pos).item()) == want


def test_distribution_chi_square():
    l = _logits(64, 5) / 2
    T, K, P = 0.9, 40, 0.95
    n = 20000
    got = _hook_draws(l, T, K, P, 2024, np.arange(n))
    prep = S.prepare(l, T, K, P)
    keep = np.zeros(64, bool)
    keep[prep.kept] = True
    assert not np.any(~keep[got])                       # nothing outside S, ever
    p = np.where(keep, np.exp((l.astype(np.float64) - l.max()) / T), 0.0)
    p /= p.sum()                                        # the float64 distribution over S
    counts = np.bincount(got, minlength=64)[keep]
    exp = p[keep] * n
    big = exp >= 5
    obs, exp = np.append(counts[big], counts[~big].sum()), np.append(exp[big], exp[~big].sum())
    keepx = exp > 0
    pv = stats.chisquare(obs[keepx], exp[keepx]).pvalue
    print(f"chi-square p = {pv:.3f} over {int(keep.sum())} tokens")
    assert pv > 1e-4


# ---- the model ---------------------------------------------------------------------------------------------------
def _small(flags=0):
    from effort_b200.model import DecodeModel, MistralConfig
    return DecodeModel.random_init(MistralConfig(n_layers=2, vocab=2048, max_seq=64), seed=7, weight_flags=flags)


@pytest.fixture(scope="module")
def small_model():
    return _small()


def _check_steps(m, prm, steps, start=0):
    """step `steps` tokens (None = self-fed) and compare next_token() with the hook on the step's logits"""
    import torch
    from effort_b200 import ops
    for k, t in enumerate(steps):
        m.step(None if t is None else torch.tensor([t], dtype=torch.int32, device="cuda"), 0.5)
        got = m.next_token()
        want = int(ops.sample(m.logits(), *prm, position=start + k + 1).item())
        assert got == want, (start + k + 1, got, want)


PRM = (0.9, 40, 0.95, 5)
TOKENS = [1, 17, 400, None, 999, None, 5]


@pytest.mark.parametrize("use_graph,chain", [(False, 2), (True, 2), (True, 1)])
def test_every_step_draws_from_its_logits(small_model, use_graph, chain):
    m = small_model
    try:
        m.set_graphs(use_graph)
        m.set_chain(chain)
        m.set_sampler(*PRM)
        m.reset()
        _check_steps(m, PRM, TOKENS)
        new = (1.3, 0, 0.8, 77)                          # new parameters, same captured graph
        m.set_sampler(*new)
        _check_steps(m, new, [None, 3, None], start=len(TOKENS))
    finally:
        m.set_sampler(None)
        m.set_chain(2)


def test_fused_glue_path():
    from effort_b200 import ops
    m = _small(ops.INPUT_MAJOR)
    ctx = ops.default_context()
    try:
        ctx.setOption("engine", 1)
        m.set_chain(1)
        m.set_fused_glue(True)
        for use_graph in (False, True):
            m.set_graphs(use_graph)
            m.set_sampler(*PRM)
            m.reset()
            _check_steps(m, PRM, TOKENS)
    finally:
        ctx.setOption("engine", 2)


def test_moe_and_q4_paths():
    from effort_b200.model import DecodeModel, MistralConfig
    cfg = MistralConfig(n_layers=2, vocab=1024, max_seq=32)
    for m in (DecodeModel.random_init_moe(cfg, n_experts=4, seed=9), DecodeModel.random_init_q4(cfg, seed=5)):
        for use_graph in (False, True):
            m.set_graphs(use_graph)
            m.set_sampler(*PRM)
            m.reset()
            _check_steps(m, PRM, TOKENS)
        del m


def _run(m, tokens, effort=0.25):
    import torch
    from effort_b200 import ops
    out = []
    for t in tokens:
        m.step(torch.tensor([t], dtype=torch.int32, device="cuda"), effort)
        torch.cuda.synchronize()
        out.append((m.logits().cpu().numpy().tobytes(), m.next_token()))
    return out


def test_greedy_untouched():
    import torch
    from effort_b200 import ops
    m = _small()
    m.set_graphs(True)
    toks = [1, 17, 400, 999, 5, 33]
    m.reset()
    never = _run(m, toks)                                # a model that never had a sampler
    m.set_sampler(*PRM)
    m.reset()
    sampled = _run(m, toks)
    m.set_sampler(None)
    m.reset()
    cleared = _run(m, toks)
    assert never == cleared
    assert [a[0] for a in sampled] == [a[0] for a in never]   # the sampler only writes `next`
    # one more launch per step, nothing else
    per = {}
    for prm in (None, PRM):
        m.set_sampler(*(prm or (None,)))
        m.reset()
        tok = torch.tensor([3], dtype=torch.int32, device="cuda")
        for _ in range(3):
            m.step(tok, 0.25)                            # eager, capture, replay
        torch.cuda.synchronize()
        n0 = ops.launchCount()
        m.step(tok, 0.25)
        torch.cuda.synchronize()
        per[prm is not None] = ops.launchCount() - n0
    assert per[True] == per[False] + 1, per
    # top_k = 1 is greedy
    m.set_sampler(None)
    greedy = m.generate([1, 17], 16)
    m.set_sampler(1.0, top_k=1, seed=4)
    assert m.generate([1, 17], 16) == greedy
    m.set_sampler(None)


def test_generate_is_reproducible(small_model):
    m = small_model
    m.set_graphs(True)
    m.set_chain(2)
    try:
        m.set_sampler(0.8, 50, 0.9, seed=1234)
        a = m.generate([1, 17, 400], 32, effort=0.25)
        m.reset()
        assert m.generate([1, 17, 400], 32, effort=0.25) == a
        assert len(a) == 32 and all(0 <= t < m.cfg.vocab for t in a)
        m.set_sampler(1.5, seed=99)
        assert m.generate([1, 17, 400], 32, effort=0.25) != a
        with pytest.raises(ValueError):
            m.generate([1] * 40, 26)                     # 40 + 26 - 1 > max_seq = 64
        assert len(m.generate([1] * 40, 25)) == 25
    finally:
        m.set_sampler(None)


def test_invalid_arguments(small_model):
    import torch
    from effort_b200 import _lib, ops
    L = _lib.load()
    ctx = ops.default_context()
    lg = torch.zeros(16, dtype=torch.float32, device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    good = _lib.Sampler(1.0, 0, 1.0, 0)
    assert L.effort_sample(ctx._h, lg.data_ptr(), 16, C.byref(good), 0, tok.data_ptr(), None) == 0
    bad = [(float("nan"), 0, 1.0), (-1.0, 0, 1.0), (0.0, 0, 1.0), (float("inf"), 0, 1.0), (1.0, -1, 1.0),
           (1.0, 0, 0.0), (1.0, 0, -0.5), (1.0, 0, 1.5), (1.0, 0, float("nan"))]
    for T, K, P in bad:
        prm = _lib.Sampler(T, K, P, 0)
        assert L.effort_sample(ctx._h, lg.data_ptr(), 16, C.byref(prm), 0, tok.data_ptr(), None) == EINVAL, (T, K, P)
        assert L.effort_model_set_sampler(small_model._h, C.byref(prm)) == EINVAL, (T, K, P)
    for n in (0, -3):
        assert L.effort_sample(ctx._h, lg.data_ptr(), n, C.byref(good), 0, tok.data_ptr(), None) == EINVAL
    assert L.effort_model_set_sampler(small_model._h, None) == 0
    with pytest.raises(_lib.EffortError):
        ops.sample(lg, 0.0)
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
    m = DecodeModel.random_init(MistralConfig(n_layers=2, vocab=4096, max_seq=64), seed=7, tp_rank=rank, tp_size=world)
    m.set_sampler(*PRM)
    m.reset()
    ok = 1
    for k, t in enumerate(TOKENS):
        m.step(None if t is None else torch.tensor([t], dtype=torch.int32, device="cuda"), 0.5)
        mine = torch.tensor([m.next_token()], dtype=torch.int64, device="cuda")
        hook = int(ops.sample(m.logits(), *PRM, position=k + 1).item())   # the all-gathered, unsharded logits
        every = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(every, mine)
        ok &= int(all(int(e.item()) == int(mine.item()) for e in every) and int(mine.item()) == hook)
    flag = torch.tensor([ok], dtype=torch.int32, device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)          # every rank fails together
    dist.destroy_process_group()
    assert int(flag.item()) == 1


@pytest.mark.timeout(300)
def test_tensor_parallel_ranks_draw_the_same_token():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.spawn(_tp_worker, args=(2, _free_port()), nprocs=2, join=True)
