"""CPU model of the device scorer (csrc/score.cuh, DESIGN.md section 4.7): per target token t against logits l[0..V),
the greedy argmax and the rank exactly, and the log-probability in float64 with the bar the fp32 kernel must meet.
`emulate_logprob` restates the kernel's fp32 formula and summation order, as evidence that the bar is reachable."""
import numpy as np

THREADS = 1024


def keys(logits):
    """the sampler's order-preserving uint32 keys: a > b <=> key(a) > key(b); -0 == +0; NaN -> 0, below -inf"""
    l = np.asarray(logits, np.float32)
    b = np.where(l == 0, np.float32(0), l).view(np.uint32)
    k = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return np.where(np.isnan(l), np.uint32(0), k)


def argmax(logits):
    """the greedy token: the lowest index of the maximum; NaN never wins; all NaN -> 0"""
    k = keys(logits).astype(np.int64)
    return int(np.argmax(k))   # np.argmax returns the first maximum; the key order is the greedy order


def ranks(logits, targets):
    """#{i : key_i > key_t} + #{i < t : key_i == key_t} per target (the position of t in the sampler's order);
    -1 for targets outside [0, V)"""
    k = keys(logits).astype(np.int64)
    V = len(k)
    order = np.lexsort((np.arange(V), -k))        # larger key first, equal keys by lower index
    pos = np.empty(V, np.int64)
    pos[order] = np.arange(V)
    t = np.asarray(targets, np.int64)
    ok = (t >= 0) & (t < V)
    return np.where(ok, pos[np.where(ok, t, 0)], -1)


def _max(l):
    fin = l[~np.isnan(l)]
    return fin.max() if len(fin) else -np.inf


def logprobs(logits, targets):
    """float64 log_softmax over the non-NaN logits at each target: -inf for a NaN or -inf target, NaN for no target or
    a maximum that is not finite"""
    l = np.asarray(logits, np.float32).astype(np.float64)
    t = np.asarray(targets, np.int64)
    V = len(l)
    ok = (t >= 0) & (t < V)
    m = _max(l)
    if not np.isfinite(m):
        return np.full(len(t), np.nan)
    logS = np.log(np.sum(np.exp(l[~np.isnan(l)] - m)))
    lt = l[np.where(ok, t, 0)]
    lp = np.where(np.isnan(lt) | (lt == -np.inf), -np.inf, (lt - m) - logS)
    return np.where(ok, lp, np.nan)


def bar(logits, targets):
    """|logprob - float64| <= 4e-6 + 2^-22 * |l_t - m|: the fp32 subtraction gives the relative term; one logf ulp at
    S <= V plus the fp32 sum's rounding the absolute one"""
    l = np.asarray(logits, np.float32).astype(np.float64)
    t = np.clip(np.asarray(targets, np.int64), 0, len(l) - 1)
    with np.errstate(invalid="ignore"):
        return 4e-6 + 2.0 ** -22 * np.abs(l[t] - _max(l))


def emulate_logprob(logits, t):
    """the kernel's fp32 formula for one in-range target: per-thread strided sums of expf(l_i - m) over 1024 threads
    (expf taken as the correctly rounded fp32 exp), a butterfly over each warp's 32 lanes, the 32 warp sums in order,
    then (l_t - m) - logf(S)"""
    l = np.asarray(logits, np.float32)
    V = len(l)
    m = np.float32(_max(l))
    rows = -(-V // THREADS)
    pad = np.full(rows * THREADS, np.nan, np.float32)
    pad[:V] = l
    with np.errstate(invalid="ignore"):
        e = np.exp((pad - m).astype(np.float64)).astype(np.float32)   # pad - m is the fp32 subtraction
    e = np.where(np.isnan(pad), np.float32(0), e).reshape(rows, THREADS)
    s = np.zeros(THREADS, np.float32)
    for r in range(rows):
        s = s + e[r]                                  # adding +0 for NaN / padding leaves a sum unchanged
    s = s.reshape(32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lane ^ o]
    S = np.float32(0)
    for w in range(32):
        S = np.float32(S + s[w, 0])
    return np.float32(np.float32(l[t] - m) - np.float32(np.log(np.float64(S))))


def check(logits, targets, argmax_got, rank_got, logprob_got):
    """assert one batch of device records against the model; returns the largest |logprob - float64| / bar"""
    targets = np.asarray(targets, np.int64)
    a = np.asarray(argmax_got, np.int64)
    r = np.asarray(rank_got, np.int64)
    lp = np.asarray(logprob_got, np.float64)
    want_a = argmax(logits)
    assert np.all(a == want_a), (np.flatnonzero(a != want_a)[:8], want_a)
    want_r = ranks(logits, targets)
    bad = np.flatnonzero(r != want_r)
    assert len(bad) == 0, (targets[bad[:8]], r[bad[:8]], want_r[bad[:8]])
    want = logprobs(logits, targets)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(lp), nan), targets[np.isnan(lp) != nan][:8]
    inf = np.isinf(want)
    assert np.array_equal(lp[inf], want[inf]), targets[inf][:8]
    fin = ~nan & ~inf
    if not fin.any():
        return 0.0
    err = np.abs(lp[fin] - want[fin]) / bar(logits, targets[fin])
    assert err.max() <= 1.0, (targets[fin][np.argmax(err)], float(err.max()))
    return float(err.max())
