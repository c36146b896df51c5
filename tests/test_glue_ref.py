"""CPU: the float64 restatements of the glue kernels (tests/glue_ref.py) that tests/test_gpu_glue.py checks the decode
kernels against -- the rope check and rotation recovery, the attention restatement against the decode restatement's,
and the greedy and top-2 tie rules."""
import numpy as np
import pytest

from tests import glue_ref as G
from tests.ref_decode import attention, rope


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


@pytest.mark.parametrize("n_kv", [1, 8])
def test_recovery_returns_injected_rotations(n_kv):
    rng = np.random.default_rng(n_kv)
    xk = rng.standard_normal(n_kv * 128)
    rot = np.exp(1j * rng.uniform(-np.pi, np.pi, 64))
    krow = G.rotate(xk, rot).reshape(-1)
    got = G.recover_rotation(xk, krow)
    assert np.max(np.abs(got - rot)) < 1e-12
    # the best-conditioned head is used: a head whose pair is near zero does not spoil the recovery
    if n_kv > 1:
        xk2 = xk.reshape(n_kv, 128).copy()
        xk2[0, :64] = 1e-30
        xk2[0, 64:] = 0.0
        got = G.recover_rotation(xk2, G.rotate(xk2, rot).reshape(-1))
        assert np.max(np.abs(got - rot)) < 1e-12


@pytest.mark.parametrize("theta", [1e6, 1e4])
def test_rope_check_accepts_fp32_rope_and_rejects_a_wrong_position(theta):
    """ref_decode.rope takes the angle in fp32 as the kernel does: it passes the check at every position up to 2047,
    and a key roped at a neighbouring position, or with the other theta, fails it."""
    rng = np.random.default_rng(3)
    xk = rng.standard_normal(8 * 128).astype(np.float32)
    worst_norm, worst_ratio = 0.0, 0.0
    for pos in list(range(0, 40)) + list(range(40, 2048, 37)) + [2047]:
        n, r = G.rope_check(xk, rope(xk, pos, theta), pos, theta)
        worst_norm, worst_ratio = max(worst_norm, n), max(worst_ratio, r)
    assert worst_norm < 4 * 2.0 ** -24, worst_norm
    assert worst_ratio <= 1.0, worst_ratio
    for pos in (1, 100, 2047):
        assert G.rope_check(xk, rope(xk, pos - 1, theta), pos, theta)[1] > 1.0
        assert G.rope_check(xk, rope(xk, pos, 1e10 / theta), pos, theta)[1] > 1.0
    # a rotation keeps the norm; a scaled key does not
    assert G.rope_check(xk, 1.0001 * rope(xk, 5, theta), 5, theta)[0] > 1e-5


@pytest.mark.parametrize("n_kv,T", [(8, 1), (8, 40), (1, 17), (32, 5)])
def test_attention_matches_decode_restatement(n_kv, T):
    """glue_ref.attention (float64) against the decode restatement's fp32 attention (RefModel) on random caches"""
    rng = np.random.default_rng(T * 100 + n_kv)
    q = rng.standard_normal((32, 128)).astype(np.float32)
    K = rng.standard_normal((T, n_kv, 128)).astype(np.float32) * np.float32(0.3)
    V = rng.standard_normal((T, n_kv, 128)).astype(np.float32)
    want = attention(q, K, V)
    got = G.attention(q, K, V)
    for h in range(32):
        assert _rel(want[h], got[h]) < 1e-5, h


def test_attention_step_ropes_the_query_with_the_keys_rotation():
    """attention_step recovers the rotation from the cached key row: with q and k roped by the fp32 restatement at
    position pos, it equals attention on rope(q, pos)"""
    rng = np.random.default_rng(11)
    n_kv, pos, theta = 8, 1234, 1e6
    xq = rng.standard_normal(32 * 128).astype(np.float32)
    xk = rng.standard_normal(n_kv * 128).astype(np.float32)
    K = (rng.standard_normal((pos + 1, n_kv, 128)) * 0.05).astype(np.float32)
    V = rng.standard_normal((pos + 1, n_kv, 128)).astype(np.float32)
    K[pos] = rope(xk, pos, theta).reshape(n_kv, 128)
    want = G.attention(rope(xq, pos, theta).reshape(32, 128), K, V)
    got = G.attention_step(xq, xk, K, V, pos)
    assert _rel(got, want) < 1e-6
    # a query roped one position off is detectably different
    off = G.attention(rope(xq, pos - 1, theta).reshape(32, 128), K, V)
    assert _rel(off, want) > 1e-3


def test_greedy_tie_and_nan_rule():
    nan, inf = np.nan, np.inf
    assert G.greedy(np.array([1, 3, 3, 2], np.float32)) == 1
    assert G.greedy(np.array([nan, 3, nan, 3], np.float32)) == 1
    assert G.greedy(np.array([3, nan, 4], np.float32)) == 2
    assert G.greedy(np.array([nan, nan], np.float32)) == 0
    assert G.greedy(np.array([-inf, -inf], np.float32)) == 0
    assert G.greedy(np.array([nan, -inf], np.float32)) == 1
    assert G.greedy(np.array([1, inf, nan, inf], np.float32)) == 1
    assert G.greedy(np.array([0.0, -0.0], np.float32)) == 0
    assert G.greedy(np.array([-0.0, 0.0], np.float32)) == 0


def test_gate_top2_tie_rule():
    assert G.gate_top2([1.0, 2.0, 2.0, 0.0])[0] == (1, 2)
    assert G.gate_top2([2.0, 1.0, 2.0])[0] == (0, 2)
    assert G.gate_top2([0.0, 1.0, 0.5, 1.0, 1.0])[0] == (1, 3)
    (i0, i1), (v0, v1) = G.gate_top2([0.0, 3.0, 1.0])
    assert (i0, i1) == (1, 2)
    assert abs(v0 - np.exp(3) / (np.exp(3) + np.exp(1))) < 1e-15 and abs(v0 + v1 - 1) < 1e-15
