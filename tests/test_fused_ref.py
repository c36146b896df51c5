"""CPU: the premises the bit-exact tier of tests/test_gpu_fused.py rests on (tests/fused_ref.py)."""
import numpy as np

from tests import fused_ref as F
from tests.ref_decode import rmsnorm_mul


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def test_norm_grid_sum_is_order_independent():
    """Every fp32 partial sum of squares of a grid vector is exact: sequential, reversed, pairwise, and the kernels'
    shapes (16 consecutive values per thread then a butterfly over 32 lanes and a sum over 8 warps; a stride-512 walk)
    give the float64 sum, so the denominator has the same bits whichever order the kernel takes."""
    for seed in range(8):
        h = F.grid_h(seed)
        sq = h * h                                   # exact: k^2 * 2^-16 with k^2 < 2^24
        want = np.float32(np.sum(h.astype(np.float64) ** 2))
        assert float(want) == float(np.sum(sq.astype(np.float64)))
        sums = []
        acc = np.float32(0)
        for x in sq:
            acc = np.float32(acc + x)
        sums.append(acc)
        acc = np.float32(0)
        for x in sq[::-1]:
            acc = np.float32(acc + x)
        sums.append(acc)
        sums.append(np.sum(sq, dtype=np.float32))    # numpy's pairwise order
        per_thread = sq.reshape(256, 16).cumsum(axis=1, dtype=np.float32)[:, -1]
        lanes = per_thread.reshape(8, 32)
        for o in (16, 8, 4, 2, 1):                   # xor butterfly
            lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(np.float32)
        sums.append(np.float32(lanes[:, 0].cumsum(dtype=np.float32)[-1]))
        strided = sq.reshape(8, 512).cumsum(axis=0, dtype=np.float32)[-1]
        sums.append(np.float32(strided.reshape(16, 32).sum(axis=1, dtype=np.float32).cumsum(dtype=np.float32)[-1]))
        assert all(_bits(s) == _bits(want) for s in sums), (seed, sums, want)
        d = F.norm_denom(h)
        w = (1.0 + 0.1 * np.random.default_rng(seed).standard_normal(4096)).astype(np.float16)
        assert np.array_equal(_bits(F.norm_input(h, w)), _bits(rmsnorm_mul(h, w)))
        assert np.float32(d) > 0


def test_div_by_is_ieee_division():
    """div_by (reciprocal, then one FMA correction) returns the correctly rounded quotient: on every entry of grid
    vectors over their own denominators, on random pairs, and on significands near all-ones."""
    rng = np.random.default_rng(3)
    for seed in range(2):
        h = F.grid_h(100 + seed)
        d = F.norm_denom(h)
        for x in h[:1024]:
            assert _bits(F.div_by(x, d)) == _bits(np.float32(x) / d), (x, d)
    xs = (rng.standard_normal(3000) * 10.0 ** rng.integers(-6, 6, 3000)).astype(np.float32)
    ds = (np.abs(rng.standard_normal(3000)) * 10.0 ** rng.integers(-3, 3, 3000) + 1e-3).astype(np.float32)
    ones = np.float32(2.0) - np.float32(2.0 ** -23) * rng.integers(1, 64, 500).astype(np.float32)
    xs = np.concatenate([xs, ones, ones * np.float32(3.0)])
    ds = np.concatenate([ds, ones[::-1], ones])
    for x, d in zip(xs, ds):
        assert _bits(F.div_by(x, d)) == _bits(np.float32(x) / np.float32(d)), (x, d)


def test_div_by_exact_fma_emulation():
    """the exact rounding helper behind div_by: a single rounding of the exact value, ties to even"""
    assert F.f32_round(F.Fraction(1) + F.Fraction(1, 2 ** 24)) == np.float32(1.0)        # tie -> even
    assert F.f32_round(F.Fraction(1) + F.Fraction(3, 2 ** 24)) == np.float32(1.0 + 2.0 ** -22)
    assert F.f32_round(F.Fraction(-5, 3)) == np.float32(-5.0) / np.float32(3.0)
    a = np.float32(1.0 + 2.0 ** -12)
    assert F.fmaf(a, a, np.float32(-1.0)) == np.float32(2.0 ** -11 + 2.0 ** -24)         # exact, unlike a*a - 1
    assert np.float32(a * a) - np.float32(1.0) == np.float32(2.0 ** -11)


def test_silu_grid_is_exact_for_any_faithful_expf():
    """x1 >= 18: 1 + expf(-x1) rounds to exactly 1 even with expf off by 2 ulps, so the product is fl(x1 * x3).
    x1 <= -90: e^90 exceeds FLT_MAX by a factor of 3.5, so expf overflows and the product is +-0, never selected."""
    x1 = F.grid_x1(5, 14336)
    x3 = np.random.default_rng(6).standard_normal(14336).astype(np.float32)
    pos = x1 >= 18
    assert pos.any() and (~pos).any() and np.all(x1[~pos] <= -90)
    e = np.exp(-x1[pos])
    for n in (-2, -1, 0, 1, 2):
        en = np.array([F.ulp_step(x, n) for x in e[:2000]], np.float32)
        assert np.all(np.float32(1.0) + en == np.float32(1.0))
    assert np.float32(1.0) + np.float32(np.exp(np.float64(-18.0))) == np.float32(1.0)
    got = F.silu_input(x1, x3)
    assert np.array_equal(_bits(got[pos]), _bits(x1[pos] * x3[pos]))
    assert np.exp(np.float64(90.0)) > 3.5 * float(np.finfo(np.float32).max)
    with np.errstate(over="ignore"):
        assert np.isinf(np.exp(np.float32(90.0)))
    assert np.all(got[~pos] == 0.0)
    from oracle import oracle as O
    stats = np.full((16 * 14336, 4), 0.5, np.float16)
    assert O.prepare_dispatch(np.where(pos, 0.0, got).astype(np.float32), stats, 0.0, 14336, 256, 16 * 14336).shape[0] == 0


def test_restatements_match_ref_decode():
    """the silu restatement is ref_decode's on realistic inputs; the norm one takes an explicit denominator"""
    rng = np.random.default_rng(8)
    x1, x3 = rng.standard_normal(14336).astype(np.float32), rng.standard_normal(14336).astype(np.float32)
    want = (x3 * x1 / (1.0 + np.exp(-x1))).astype(np.float32)
    assert np.array_equal(_bits(F.silu_input(x1, x3)), _bits(want))
    h = (rng.standard_normal(4096) * 3).astype(np.float32)
    w = (1.0 + 0.1 * rng.standard_normal(4096)).astype(np.float16)
    d = F.norm_denom(h)
    assert np.array_equal(_bits(F.norm_input(h, w)), _bits(rmsnorm_mul(h, w)))
    assert np.array_equal(_bits(F.norm_input(h, w, denom=F.ulp_step(d, 0))), _bits(rmsnorm_mul(h, w)))
    assert F.ulp_step(d, 2) > F.ulp_step(d, 1) > d > F.ulp_step(d, -1) > F.ulp_step(d, -2)
