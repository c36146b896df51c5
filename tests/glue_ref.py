"""Float64 restatements of the decode loop's glue kernels (effort_b200/csrc/decode.cuh) for checking each kernel on the
inputs it actually consumed: the q/k/v GEMV outputs, the caches, the residual and the gate input that the decode step
left on the device (DecodeModel.buffer).  No upstream GEMV noise enters such a comparison, so the bars can be tight at
any effort, depth and position.  Test infrastructure only."""
import numpy as np

from tests.ref_decode import rmsnorm_mul

HD = 128
HALF = HD // 2


def _pairs(x):
    """[..., 128] -> the rotate-half pairs (x_j, x_{j+64}) as complex128 [..., 64]"""
    x = np.asarray(x, np.float64).reshape(-1, HD)
    return x[:, :HALF] + 1j * x[:, HALF:]


def _unpairs(z):
    return np.concatenate([z.real, z.imag], axis=-1)


def rope_freq(theta):
    """the exact frequencies theta^(-j/64), j < 64 (model.swift:693-717), in float64"""
    return np.power(np.float64(theta), -np.arange(HALF, dtype=np.float64) / HALF)


def rope_check(xk, krow, pos, theta):
    """The cached key row `krow` [n_kv*128] against the GEMV output `xk` it was roped from.  The kernel takes the angle
    in fp32 (powf for the frequency, then pos*freq rounded), so against the exact float64 angle its error grows with
    pos*freq_j: up to ~4 ulps of the angle, about 1e-4 rad at pos 2047.  Returns
      norm_err:    max over pairs of | |(k_j, k_j+64)| - |(x_j, x_j+64)| | / |(x_j, x_j+64)|  (a rotation keeps the norm),
      angle_ratio: max over pairs of |recovered angle - pos*freq_j| (mod 2 pi) / (2^-20 * pos * freq_j + 1e-6),
    where pairs with a norm below 1e-20 (too small to carry an angle) are skipped.  A rope that is right gives
    norm_err of a few fp32 ulps and angle_ratio <= 1."""
    a, b = _pairs(xk), _pairs(krow)
    na, nb = np.abs(a), np.abs(b)
    ok = na > 1e-20
    norm_err = float(np.max(np.abs(nb - na)[ok] / na[ok], initial=0.0))
    exact = pos * rope_freq(theta)
    got = np.angle(b * np.conj(a))
    err = np.abs(np.angle(np.exp(1j * (got - exact))))   # wrapped to [0, pi]
    bound = 2.0 ** -20 * exact + 1e-6
    angle_ratio = float(np.max((err / bound)[ok], initial=0.0))
    return norm_err, angle_ratio


def recover_rotation(xk, krow):
    """The rotation (cos, sin) per pair j that the kernel applied to this step's key, as complex128 [64]: krow / xk
    pairwise, taken from the KV head with the largest |(x_j, x_j+64)| (the best-conditioned quotient)."""
    a, b = _pairs(xk), _pairs(krow)
    best = np.argmax(np.abs(a), axis=0)
    cols = np.arange(HALF)
    return b[best, cols] / a[best, cols]


def rotate(x, rot):
    """rotate-half rope of x [n*128] with the per-pair rotation rot (complex [64]), in float64 -> [n, 128]"""
    return _unpairs(_pairs(x) * rot)


def attention(q, K, V):
    """Attention of one token in float64: q [n_heads, 128] (roped), K / V [T, n_kv, 128] (the cache rows 0..pos);
    head h reads KV head h // (n_heads / n_kv).  scores = q.k / sqrt(128), softmax = exp(s) / sum(exp(s)) WITHOUT max
    subtraction (aux.metal:185-199), out = sum_t p_t v_t.  Returns [n_heads, 128]."""
    q = np.asarray(q, np.float64)
    K = np.ascontiguousarray(np.asarray(K).transpose(1, 0, 2), np.float64)   # [n_kv, T, 128]
    V = np.ascontiguousarray(np.asarray(V).transpose(1, 0, 2), np.float64)
    n_heads, n_kv = q.shape[0], K.shape[0]
    qg = q.reshape(n_kv, n_heads // n_kv, HD)
    p = np.exp(qg @ K.transpose(0, 2, 1) / np.sqrt(HD))                      # [n_kv, rep, T]
    p /= p.sum(axis=-1, keepdims=True)
    return (p @ V).reshape(n_heads, HD)


def attention_step(xq, xk, K, V, pos):
    """The attention kernel's output at position `pos` restated on the GPU's own inputs: the query is roped with the
    rotation recovered from this step's cached key row K[pos] (so the fp32 angle error of the kernel cancels: q and k
    of one pair share its cos/sin), then attention over the cache rows 0..pos."""
    n_kv = K.shape[1]
    rot = recover_rotation(xk, K[pos].reshape(n_kv * HD))
    return attention(rotate(xq, rot), K[: pos + 1], V[: pos + 1])


def final_norm_fp16(h, w, eps=1e-5):
    """fp16(rmsNorm(h) * w) as float64: the lm_head's / gate's input (helpers/mps.swift:19 casts v to fp16)"""
    return rmsnorm_mul(np.asarray(h, np.float32), np.asarray(w), eps).astype(np.float16).astype(np.float64)


def greedy(logits):
    """The greedy token: the lowest index among the maximal non-NaN logits; token 0 when every logit is NaN"""
    x = np.asarray(logits)
    ok = ~np.isnan(x)
    if not ok.any():
        return 0
    return int(np.flatnonzero(ok & (x == x[ok].max()))[0])


def gate_logits(h_keep, ffn_norm, gate, eps=1e-5):
    """The MoE gate logits in float64: gate [n_experts, dim] fp16 @ fp16(rmsNorm(h_keep) * ffn_norm)"""
    return np.asarray(gate).astype(np.float64) @ final_norm_fp16(h_keep, ffn_norm, eps)


def gate_top2(logits):
    """The two largest gate logits, the lower expert first on ties, and their softmax exp(x) / sum(exp(x))
    (mpsTopK(2) + gateVals.softmax(), runNetwork.swift:185-189).  Returns ((i0, i1), (v0, v1))."""
    order = sorted(range(len(logits)), key=lambda e: (-float(logits[e]), e))[:2]
    e = np.exp(np.asarray(logits, np.float64)[order])
    return tuple(order), tuple(e / e.sum())
