"""A numpy / Python-int restatement of the device sampler's rule (DESIGN.md section 4.6, csrc/sample.cuh).

Everything after the weights is integer arithmetic, so this model and the kernel agree bit for bit except where the
device's expf and the host's exp differ in the last ulp.  `prepare` does the position-independent part (order, top-k,
weights, top-p); `draw` is the Philox draw for one or many positions."""
import math

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC'11).  counter: 4 words, key: 2 words (numpy uint64 arrays or ints).
    Vectorised over numpy arrays; returns the 4 output words."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) for c in counter)
    k0, k1 = (np.asarray(k, np.uint64) for k in key)
    m0, m1, w0, w1, mask = (np.uint64(x) for x in (M0, M1, W0, W1, MASK32))
    for r in range(10):
        if r:
            k0, k1 = (k0 + w0) & mask, (k1 + w1) & mask
        p0, p1 = m0 * c0, m1 * c2                     # < 2^64: no overflow
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & mask
    return c0, c1, c2, c3


def philox_word0(position, seed):
    """word 0 of Philox4x32-10 with counter (position, 0, 0, 0) and key (seed & 0xffffffff, seed >> 32)"""
    pos = np.asarray(position, np.uint64)
    z = np.zeros_like(pos)
    return philox4x32_10((pos, z, z, z), (np.uint64(seed & MASK32), np.uint64(seed >> 32)))[0]


def weights(logits, temperature):
    """q_i = floor(expf((l_i - m) / T) * 2^32) as uint64 (NaN -> 0).  fp32 subtraction and IEEE division; the exp
    is the correctly rounded fp32 value (float64 exp, rounded once)."""
    l = np.asarray(logits, np.float32)
    fin = l[~np.isnan(l)]
    m = np.float32(fin.max())
    with np.errstate(invalid="ignore", over="ignore"):
        z = (l - m) / np.float32(temperature)
        w = np.exp(z.astype(np.float64)).astype(np.float32)
    w = np.where(np.isnan(l), np.float32(0), w)
    return np.floor(w.astype(np.float64) * 2.0 ** 32).astype(np.uint64)


def order(logits):
    """token indices in sampling order: larger logit first, equal logits (+0 == -0) by lower index, NaN last"""
    l = np.asarray(logits, np.float32).astype(np.float64)
    l = np.where(np.isnan(l), -np.inf, l) + 0.0          # +0.0 turns -0 into +0
    nan_last = np.isnan(np.asarray(logits, np.float32))
    return np.lexsort((np.arange(len(l)), -l, nan_last))


class Prepared:
    """the position-independent part of one draw: `kept` = S in index order, `cum` = its inclusive prefix sums of q,
    `greedy` = the token when no draw happens (non-finite maximum), `sk` / `sk_cum` = S_k in sampling order and its
    prefix sums, `need` = the top-p target"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def prepare(logits, temperature, top_k=0, top_p=1.0):
    l = np.asarray(logits, np.float32)
    V = len(l)
    valid = ~np.isnan(l)
    if not valid.any() or l[valid].max() == -np.inf:
        return Prepared(greedy=0)
    if l[valid].max() == np.inf:
        return Prepared(greedy=int(np.flatnonzero(l == np.inf)[0]))
    ordr = order(l)
    K = V if top_k == 0 or top_k >= V else top_k
    sk = ordr[:K]
    q = weights(l, temperature)
    sk_cum = np.cumsum(q[sk], dtype=np.uint64)
    Qk = int(sk_cum[-1])
    need = math.ceil(float(np.float32(top_p)) * float(Qk))
    n_keep = int(np.searchsorted(sk_cum, np.uint64(need), side="left")) + 1   # shortest prefix with sum >= need
    kept = np.sort(sk[:n_keep])
    cum = np.cumsum(q[kept], dtype=np.uint64)
    return Prepared(greedy=None, kept=kept, cum=cum, Q=int(cum[-1]), q=q, sk=sk, sk_cum=sk_cum, Qk=Qk, need=need)


def targets(Q, x):
    """(x * Q) >> 32 for 32-bit x and Q < 2^64, without overflowing uint64"""
    x = np.asarray(x, np.uint64)
    Q = int(Q)
    hi, lo = np.uint64(Q >> 32), np.uint64(Q & MASK32)
    return x * hi + ((x * lo) >> np.uint64(32))


def draw(prep, seed, positions):
    """tokens for each position (numpy int64 array)"""
    positions = np.atleast_1d(np.asarray(positions, np.uint64))
    if prep.greedy is not None:
        return np.full(len(positions), prep.greedy, np.int64)
    t = targets(prep.Q, philox_word0(positions, seed))
    return prep.kept[np.searchsorted(prep.cum, t, side="right")].astype(np.int64)


def sample(logits, temperature, top_k=0, top_p=1.0, seed=0, position=0):
    return int(draw(prepare(logits, temperature, top_k, top_p), seed, [position])[0])


def near_boundary(prep, seed, positions, rel=1e-6):
    """per position: True where an ulp of expf could change the draw -- the target lies within rel*Q of a prefix
    boundary of S, or `need` lies within rel*Qk of a prefix boundary of S_k"""
    positions = np.atleast_1d(np.asarray(positions, np.uint64))
    if prep.greedy is not None:
        return np.zeros(len(positions), bool)
    need_close = bool(np.any(np.abs(prep.sk_cum.astype(np.float64) - prep.need) <= rel * prep.Qk))
    t = targets(prep.Q, philox_word0(positions, seed)).astype(np.float64)
    cum = prep.cum.astype(np.float64)
    i = np.searchsorted(cum, t)
    lo = np.abs(t - cum[np.clip(i - 1, 0, len(cum) - 1)])
    hi = np.abs(cum[np.clip(i, 0, len(cum) - 1)] - t)
    return need_close | (np.minimum(lo, hi) <= rel * prep.Q)


def probabilities(logits, temperature, top_k=0, top_p=1.0):
    """float64 distribution the draw follows: q_i / Q over S (0 elsewhere)"""
    prep = prepare(logits, temperature, top_k, top_p)
    p = np.zeros(len(logits))
    if prep.greedy is not None:
        p[prep.greedy] = 1.0
        return p
    p[prep.kept] = prep.q[prep.kept].astype(np.float64) / prep.Q
    return p
