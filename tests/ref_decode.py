"""CPU restatement of one decode step (runNetwork.swift:113-209) on top of the oracle's bucketMul.
Test infrastructure only.  Glue ops follow aux.metal / matrix.metal (cited inline)."""
import numpy as np

from oracle import oracle as O


def rmsnorm_mul(x, w, eps=1e-5):
    """rmsNorm32fast (aux.metal:113-152) then mulVec32by16 (aux.metal:269)."""
    x = x.astype(np.float32)
    ss = np.float32(np.sum(x.astype(np.float64) ** 2))
    denom = np.sqrt(np.float32(ss / np.float32(x.size) + np.float32(eps)))
    return ((x / denom) * w.astype(np.float32)).astype(np.float32)


def rope(x, pos, theta=1e6, hd=128):
    """rope_mx (aux.metal:218-231) with freqs = (1/theta)^(j/64) (model.swift:693-717)."""
    x = x.reshape(-1, hd).astype(np.float32)
    j = np.arange(hd // 2)
    freq = np.power(np.float32(1.0 / theta), (j / np.float32(hd // 2)).astype(np.float32)).astype(np.float32)
    ang = (np.float32(pos) * freq).astype(np.float32)
    c, s = np.cos(ang), np.sin(ang)
    out = np.empty_like(x)
    out[:, : hd // 2] = x[:, : hd // 2] * c - x[:, hd // 2:] * s
    out[:, hd // 2:] = x[:, hd // 2:] * c + x[:, : hd // 2] * s
    return out.reshape(-1)


def attention(q, K, V):
    """calcScores + softmax + sumScores for one token in fp32: q [n_heads, hd] (roped), K / V [T, n_kv, hd]; head h reads
    KV head h // (n_heads / n_kv).  Returns [n_heads, hd]."""
    n_heads, hd = q.shape
    rep = n_heads // K.shape[1]
    out = np.empty((n_heads, hd), np.float32)
    for hh in range(n_heads):
        sc = (K[:, hh // rep, :] @ q[hh]) / np.float32(np.sqrt(hd))   # dotSetScore2 aux.metal:445
        p = np.exp(sc.astype(np.float32))                             # softmax without max (aux.metal:185-199)
        p = p / p.sum()
        out[hh] = p @ V[:, hh // rep, :]                              # sumScores32 aux.metal:379-393
    return out


class RefModel:
    """weights: list of layers, each dict name -> dict(buckets, stats, probes, in, out) + 'attn_norm','ffn_norm'."""

    def __init__(self, layers, norm, out_core, emb, n_heads=32, n_kv=8, hd=128, fast=False):
        self.layers, self.norm, self.out_core, self.emb = layers, norm, out_core, emb
        self.fast = fast   # the OpenMP port (fp32, chunked sum order) instead of the sequential oracle
        self.n_heads, self.n_kv, self.hd = n_heads, n_kv, hd
        self.kc = [[] for _ in layers]
        self.vc = [[] for _ in layers]
        self.pos = 0

    def _mul(self, v, w, effort, exp_no=0):
        if w.get("n_experts", 1) > 1:   # expNo selects the expert's rows / probes (bucketMul.metal:49,143)
            if self.fast:
                return O.bucket_mul_mt(v, w["buckets"], w["stats"], w["probes"], w["in"], w["out"], effort, exp_no=exp_no)[0]
            r = O.bucket_mul(v, w["buckets"], w["stats"], w["probes"], w["in"], w["out"], effort, exp_no=exp_no)
            return r["out32"]
        return self._mul1(v, w, effort)

    def _mul1(self, v, w, effort):
        # expertMul routing (expertMul.swift:20-38): Q4 with buckets -> zero + bucketMulQ4 + outliers; Q4 without ->
        # dense basicMul on `core`; FP16 -> bucketMul
        kind = w.get("kind", "fp16")
        if kind == "q4":
            return O.bucket_mul_q4(v, w["buckets"], w["stats"], w["probes"], w["outliers"], w["in"], w["out"], effort)["out32"]
        if kind == "core":
            return O.basic_mul(v, w["core"], cast_v=True)[0]
        if self.fast:
            out, _ = O.bucket_mul_mt(v, w["buckets"], w["stats"], w["probes"], w["in"], w["out"], effort)
            return out
        r = O.bucket_mul(v, w["buckets"], w["stats"], w["probes"], w["in"], w["out"], effort)
        return r["out32"]

    def step(self, token, effort):
        h = self.emb[token].astype(np.float32)
        for li, L in enumerate(self.layers):
            hn = rmsnorm_mul(h, L["attn_norm"])
            xq, xk, xv = self._mul(hn, L["wq"], effort), self._mul(hn, L["wk"], effort), self._mul(hn, L["wv"], effort)
            q = rope(xq, self.pos).reshape(self.n_heads, self.hd)
            k = rope(xk, self.pos).reshape(self.n_kv, self.hd)
            self.kc[li].append(k)
            self.vc[li].append(xv.reshape(self.n_kv, self.hd).copy())
            out = attention(q, np.stack(self.kc[li]), np.stack(self.vc[li]))
            h = h + self._mul(out.reshape(-1), L["wo"], effort)
            fx = rmsnorm_mul(h, L["ffn_norm"])
            if "gate" in L:   # runNetwork.swift:185-200
                gl, _ = O.basic_mul(fx, L["gate"], cast_v=True)
                order = sorted(range(len(gl)), key=lambda e: (-float(gl[e]), e))[:2]      # mpsTopK(2), ties: lower index
                gv = np.exp(gl[order].astype(np.float32))
                gv = gv / gv.sum()                                                         # gateVals.softmax()
                for e, g in zip(order, gv):
                    x1, x3 = self._mul(fx, L["w1"], effort, e), self._mul(fx, L["w3"], effort, e)
                    x2 = (x3 * x1 / (1.0 + np.exp(-x1))).astype(np.float32)
                    h = h + np.float32(g) * self._mul(x2, L["w2"], effort, e)
                continue
            x1, x3 = self._mul(fx, L["w1"], effort), self._mul(fx, L["w3"], effort)
            x2 = (x3 * x1 / (1.0 + np.exp(-x1))).astype(np.float32)               # silu32b matrix.metal:25-34
            h = h + self._mul(x2, L["w2"], effort)
        on = rmsnorm_mul(h, self.norm)
        if self.fast:
            logits = O.basic_mul_fast(np.float16(on).astype(np.float32), self.out_core)
        else:
            logits, _ = O.basic_mul(on, self.out_core, cast_v=True)                # runNetwork.swift:209
        self.pos += 1
        return logits
