"""The sampling rule of DESIGN.md section 4.6 as a CPU model (tests/sampler_model.py): Philox against the Random123
known-answer vectors, the greedy limits of top-k and top-p, NaN / infinity handling, exact set sizes under ties, and
the distribution of the draws.  The GPU tests pin the kernel to this model."""
import numpy as np
import pytest
from scipy import stats

from tests import sampler_model as S


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, want):
    assert tuple(int(w) for w in S.philox4x32_10(counter, key)) == want


def test_philox_word0_uses_position_and_both_seed_halves():
    x = S.philox_word0(np.arange(4), 0)
    assert int(x[0]) == 0x6627E8D5 and len(set(int(v) for v in x)) == 4
    assert int(S.philox_word0([7], 1)[0]) != int(S.philox_word0([7], 1 << 32)[0])


def _logits(V, seed):
    return np.random.default_rng(seed).standard_normal(V).astype(np.float32) * 3


def test_top_k_1_and_tiny_top_p_are_greedy_with_lowest_index_on_ties():
    l = _logits(1000, 1)
    l[[17, 400, 999]] = l.max() + 1          # a three-way tie for the maximum
    for kw in ({"top_k": 1}, {"top_p": 1e-9}, {"top_k": 5, "top_p": 1e-9}):
        prep = S.prepare(l, 1.0, **kw)
        assert list(prep.kept) == [17]
        assert set(S.draw(prep, 3, np.arange(200))) == {17}


def test_nan_never_drawn_and_degenerate_vectors():
    l = np.array([np.nan, 1.0, np.nan, 1.0, -np.inf], np.float32)
    got = S.draw(S.prepare(l, 1.0), 5, np.arange(500))
    assert set(got) == {1, 3}
    assert S.sample(np.full(8, np.nan, np.float32), 1.0) == 0
    assert S.sample(np.full(8, -np.inf, np.float32), 1.0) == 0
    assert S.sample(np.array([np.nan, -np.inf, -np.inf], np.float32), 1.0) == 0
    l = np.array([0.0, np.inf, 3.0, np.inf, np.nan], np.float32)
    assert S.sample(l, 1.0, seed=9, position=4) == 1      # +inf maximum: greedy's lowest index
    # a NaN inside S_k (it sorts last) carries no weight
    assert set(S.draw(S.prepare(np.array([np.nan, 2.0], np.float32), 1.0, top_k=2), 1, np.arange(100))) == {1}


def test_set_sizes_under_ties():
    l = np.array([1, 3, 3, 2, 3, 3, 0, 2], np.float32)
    assert list(S.order(l)) == [1, 2, 4, 5, 3, 7, 0, 6]
    for K in range(1, 9):
        prep = S.prepare(l, 1e4, top_k=K)          # T = 1e4: near-uniform weights, every member kept
        assert len(prep.sk) == K and sorted(prep.kept) == sorted(S.order(l)[:K])
    assert len(S.prepare(l, 1.0, top_k=0).sk) == 8 and len(S.prepare(l, 1.0, top_k=100).sk) == 8
    # +0 and -0 are equal logits: tie cut by index
    z = np.array([-0.0, 0.0, -0.0], np.float32)
    assert list(S.order(z)) == [0, 1, 2]
    assert list(S.prepare(z, 1.0, top_k=2).kept) == [0, 1]
    # top-p keeps the shortest prefix reaching ceil(P * Qk): equal weights -> exactly ceil(P * n) tokens
    e = np.zeros(8, np.float32)
    for P, n in ((0.125, 1), (0.126, 2), (0.5, 4), (0.51, 5), (1.0, 8)):
        assert len(S.prepare(e, 1.0, top_p=P).kept) == n, P


def test_draw_is_a_function_of_seed_and_position():
    prep = S.prepare(_logits(32000, 2), 0.8, 50, 0.9)
    a = S.draw(prep, 11, np.arange(64))
    assert np.array_equal(a, S.draw(prep, 11, np.arange(64)))
    assert not np.array_equal(a, S.draw(prep, 12, np.arange(64)))
    assert set(a) <= set(prep.kept) and len(prep.kept) <= 50


@pytest.mark.parametrize("T,K,P", [(1.0, 0, 1.0), (0.7, 20, 1.0), (1.3, 0, 0.8), (0.9, 40, 0.95)])
def test_chi_square_against_float64_distribution(T, K, P):
    l = _logits(64, 3) / 3
    p = S.probabilities(l, T, K, P)
    want = np.exp((l.astype(np.float64) - l.max()) / T)
    keep = p > 0
    want = np.where(keep, want, 0) / want[keep].sum()
    assert np.allclose(p, want, rtol=1e-6, atol=1e-9)       # the integer weights are the float64 distribution
    n = 20000
    counts = np.bincount(S.draw(S.prepare(l, T, K, P), 1234, np.arange(n)), minlength=64)
    assert counts[~keep].sum() == 0
    exp = want[keep] * n
    big = exp >= 5
    obs = np.append(counts[keep][big], counts[keep][~big].sum())
    exp = np.append(exp[big], exp[~big].sum())
    obs, exp = obs[exp > 0], exp[exp > 0]
    assert stats.chisquare(obs, exp).pvalue > 1e-4
