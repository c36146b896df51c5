"""Restatements of the glue the fused decode chain applies on load (effort_fused_mul_batch), and the inputs on which that
glue is bit-exact whatever order the kernel sums in.  Test infrastructure only.

  norm:  x = (h / d) * w in fp32, d = sqrtf(sum(h^2) / 4096 + eps)       (ref_decode.rmsnorm_mul, aux.metal:113-152)
  silu:  x = x3 * x1 / (1 + expf(-x1)) in fp32                           (silu32b, matrix.metal:25-34)

On a norm grid vector (every h_i = k_i * 2^-8 with sum k_i^2 < 2^24) every fp32 partial sum of squares is exact, so d has
the same bits in any summation order.  On a silu grid (every x1 >= 18 or <= -90) the product is fl(x1 * x3) or +-0 for
any expf within a few ulps.  tests/test_fused_ref.py pins both premises, and the kernel's division (div_by in
bucket_mul_v4.cuh) against IEEE division."""
from fractions import Fraction

import numpy as np

DIM = 4096
GRID_STEP = 2.0 ** -8


def grid_h(seed: int, n: int = DIM) -> np.ndarray:
    """A make_v-like residual stream on the norm grid: k_i ~ N(0, 30^2) with 1 % of entries x4, sum k_i^2 < 2^24."""
    rng = np.random.default_rng(seed)
    k = np.rint(rng.standard_normal(n) * 30.0)
    idx = rng.choice(n, size=max(1, n // 100), replace=False)
    k[idx] *= 4
    k += 0.0  # no -0: div_by(-0, d) is +0
    assert float(np.sum(k * k)) < 2.0 ** 24
    return (k * GRID_STEP).astype(np.float32)


def grid_x1(seed: int, n: int) -> np.ndarray:
    """x1 on the silu grid: 80 % in [18, ...), 20 % in (..., -90]."""
    rng = np.random.default_rng(seed)
    mag = np.abs(rng.standard_normal(n)) * 8.0
    pos = rng.random(n) < 0.8
    return np.where(pos, 18.0 + mag, -90.0 - mag).astype(np.float32)


def norm_denom(h, eps=1e-5) -> np.float32:
    """sqrtf(fp32(sum h^2) / 4096 + eps), the sum taken in float64 (exact on the norm grid)."""
    h = np.asarray(h, np.float32)
    ss = np.float32(np.sum(h.astype(np.float64) ** 2))
    return np.float32(np.sqrt(np.float32(ss / np.float32(h.size) + np.float32(eps))))


def norm_input(h, w, eps=1e-5, denom=None) -> np.ndarray:
    """(h / d) * w in fp32 with IEEE division; d = norm_denom(h, eps) unless given."""
    d = norm_denom(h, eps) if denom is None else np.float32(denom)
    return ((np.asarray(h, np.float32) / d) * np.asarray(w).astype(np.float32)).astype(np.float32)


def silu_input(x1, x3) -> np.ndarray:
    x1, x3 = np.asarray(x1, np.float32), np.asarray(x3, np.float32)
    with np.errstate(over="ignore"):
        return (x3 * x1 / (np.float32(1.0) + np.exp(-x1))).astype(np.float32)


def ulp_step(x: np.float32, n: int) -> np.float32:
    """x moved by n fp32 ulps (n < 0: down)."""
    x = np.float32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, np.float32(np.inf if n > 0 else -np.inf), dtype=np.float32)
    return x


def f32_round(q: Fraction) -> np.float32:
    """The exact rational q rounded once to fp32 (nearest, ties to even; normal range only)."""
    if q == 0:
        return np.float32(0.0)
    s, a = (-1, -q) if q < 0 else (1, q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    assert -126 <= e <= 127, "normal range only"
    m = a / Fraction(2) ** (e - 23)          # in [2^23, 2^24)
    n, r = divmod(m.numerator, m.denominator)
    if 2 * r > m.denominator or (2 * r == m.denominator and n & 1):
        n += 1
    return np.float32(s * float(Fraction(n) * Fraction(2) ** (e - 23)))


def fmaf(a, b, c) -> np.float32:
    return f32_round(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def div_by(x, d) -> np.float32:
    """bucket_mul_v4.cuh div_by: r = rn(1/d); q = x*r; q += (x - q*d)*r with two FMAs."""
    x, d = np.float32(x), np.float32(d)
    r = np.float32(np.float32(1.0) / d)
    q = np.float32(x * r)
    return fmaf(fmaf(-q, d, x), r, q)
