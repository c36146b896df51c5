"""CPU checks of the scoring rule's model (tests/score_model.py, DESIGN.md section 4.7): exact argmax and rank on ties,
signed zeros, NaN and infinities, and evidence from an fp32 restatement of the kernel that the logprob bar is reachable."""
import numpy as np
import pytest

from tests import score_model as M

NAN, INF = np.float32(np.nan), np.float32(np.inf)


def _brute_rank(l, t):
    k = M.keys(l).astype(np.int64)
    return int(np.sum(k > k[t]) + np.sum(k[:t] == k[t]))


def test_keys_order_like_floats():
    x = np.array([-INF, -3.5, -1e-40, -0.0, 0.0, 1e-40, 2.0, INF], np.float32)
    k = M.keys(x).astype(np.int64)
    assert np.all(np.diff(k[[0, 1, 2, 3, 5, 6, 7]]) > 0) and k[3] == k[4]
    assert M.keys(np.array([NAN], np.float32))[0] == 0 < k[0]


def test_ties_at_the_top_and_at_the_target():
    l = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 3.0], np.float32)
    assert M.argmax(l) == 1
    assert list(M.ranks(l, range(6))) == [5, 0, 3, 1, 4, 2]
    lp = M.logprobs(l, [1, 3, 5])
    assert lp[0] == lp[1] == lp[2] == -np.log(3 + 2 * np.exp(-1.0) + np.exp(-2.0))


def test_signed_zeros_tie():
    l = np.array([-1.0, -0.0, 0.0, -0.0], np.float32)
    assert M.argmax(l) == 1
    assert list(M.ranks(l, range(4))) == [3, 0, 1, 2]
    lp = M.logprobs(l, [1, 2, 3])
    assert lp[0] == lp[1] == lp[2]


def test_nan_and_infinite_targets():
    l = np.array([NAN, -INF, 1.0, NAN, 0.5, -INF], np.float32)
    assert M.argmax(l) == 2
    assert list(M.ranks(l, range(6))) == [4, 2, 0, 5, 1, 3]
    lp = M.logprobs(l, range(6))
    assert lp[0] == lp[3] == lp[1] == lp[5] == -np.inf
    assert np.isclose(lp[2], -np.log(1 + np.exp(-0.5)))


@pytest.mark.parametrize("l,am", [
    (np.full(7, NAN), 0),
    (np.full(7, -INF), 0),
    (np.array([NAN, -INF, -INF], np.float32), 1),
    (np.array([1.0, INF, 2.0, INF, NAN], np.float32), 1),
])
def test_no_finite_maximum(l, am):
    V = len(l)
    assert M.argmax(l) == am
    assert list(M.ranks(l, range(V))) == [_brute_rank(l, t) for t in range(V)]
    assert np.all(np.isnan(M.logprobs(l, range(V))))


def test_one_token():
    l = np.array([-7.25], np.float32)
    assert M.argmax(l) == 0 and list(M.ranks(l, [0])) == [0] and M.logprobs(l, [0])[0] == 0.0
    assert M.emulate_logprob(l, 0) == 0.0


def test_out_of_range_targets():
    l = np.array([0.5, 1.5, -2.0], np.float32)
    t = [-1, 3, 103, -100, 1]
    assert list(M.ranks(l, t)) == [-1, -1, -1, -1, 0]
    lp = M.logprobs(l, t)
    assert np.all(np.isnan(lp[:4])) and np.isfinite(lp[4])


def test_rank_matches_the_definition_on_coarse_ties():
    rng = np.random.default_rng(3)
    l = (np.round(rng.standard_normal(500) * 2) / 2).astype(np.float32)
    l[rng.choice(500, 20, replace=False)] = NAN
    l[rng.choice(500, 5, replace=False)] = -0.0
    assert list(M.ranks(l, range(500))) == [_brute_rank(l, t) for t in range(500)]
    assert sorted(M.ranks(l, range(500))) == list(range(500))     # a permutation: every rank once


@pytest.mark.parametrize("V", [32000, 131072])
def test_fp32_formula_meets_the_bar(V):
    """the kernel's fp32 arithmetic in its summation order stays well inside the bar (evidence, not a measurement)"""
    rng = np.random.default_rng(V)
    l = (rng.standard_normal(V) * 2).astype(np.float32)
    l[rng.choice(V, 50, replace=False)] = NAN
    l[rng.choice(V, 50, replace=False)] = -INF
    l[: V // 4] = np.round(l[: V // 4] * 4) / 4
    targets = np.concatenate([rng.choice(V, 96, replace=False), [int(np.nanargmax(l))]])
    targets = targets[np.isfinite(l[targets])]
    want = M.logprobs(l, targets)
    got = np.array([M.emulate_logprob(l, int(t)) for t in targets], np.float64)
    ratio = np.abs(got - want) / M.bar(l, targets)
    print(f"V={V}: emulated fp32 logprob, max |err| / bar = {ratio.max():.3f}")
    assert ratio.max() <= 0.5
