"""Host-side mirror of the reference's operator interface for the bucketMul path.

Same names, argument meaning and error behaviour as the Swift free functions, so that the parity tests
read like the reference's own call sites (runNetwork.swift:132-134, benchmarks/benchmark.swift:175):

    expertMul(v=h_norm, by=layer.wq, out=xq, effort=0.25)           expertMul.swift:20
    bucketMul(v=..., by=..., expNo=..., out=..., effort=...)        bucketMul.swift:11
    bucketMulQ4(...)                                                bucketMulQ4.swift:11
    basicMul(v=..., by=core, out=...)                               helpers/mps.swift:14
    bucketize(w) -> {"buckets", "bucket.stats", "probes"}           convert.swift:209

torch is used only as the owner of device memory and streams; every operator is one call into the C-ABI
(include/effort_b200.h).  Nothing here computes on the CPU and nothing falls back to PyTorch math.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import EffortError, MulArgs, Sampler, check

KIND_FP16, KIND_Q4 = 0, 1
NO_REPACK = 1
SLICE_MAJOR = 2
INPUT_MAJOR = 4
CUTOFF_SELECT, CUTOFF_BISECT = 0, 1


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise EffortError(f"{name} must be a CUDA tensor (no CPU path exists)")
    if t.dtype != dtype:
        raise EffortError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise EffortError(f"{name} must be contiguous")


class Context:
    """Per-stream scratch; replaces the BucketMul.shared singleton (bucketMul.swift:18-32)."""

    def __init__(self, device: Optional[int] = None):
        L = _lib.load()
        if not torch.cuda.is_available():
            raise EffortError("effort_b200 needs a CUDA device: there is no CPU fallback")
        dev = torch.cuda.current_device() if device is None else device
        h = C.c_void_p()
        check(L.effort_ctx_create(dev, C.byref(h)), "effort_ctx_create")
        self._h, self._L, self.device = h, L, dev

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._L.effort_ctx_destroy(self._h)
                self._h = None
        except Exception:
            pass


    def setCutoffMode(self, mode):
        """'select' (default: exact order statistic, ~1 us) or 'bisect' (the reference's findCutoff32 loop bit for bit)."""
        m = {"select": CUTOFF_SELECT, "bisect": CUTOFF_BISECT}.get(mode, mode)
        check(self._L.effort_ctx_set_cutoff_mode(self._h, int(m)), "effort_ctx_set_cutoff_mode")

    def setOption(self, name: str, value: int):
        """A/B knobs of the fused operator: 'engine' (2|1), 'stage' (0 cp.async | 1 cp.async.bulk), 'dynamic' (1|0)."""
        check(self._L.effort_ctx_set_option(self._h, name.encode(), int(value)), f"effort_ctx_set_option({name})")

    def errorFlag(self) -> int:
        f = C.c_uint(0)
        check(self._L.effort_ctx_error_flag(self._h, C.byref(f), _stream_ptr()), "effort_ctx_error_flag")
        return int(f.value)


_default_ctx: dict[int, Context] = {}


def default_context() -> Context:
    d = torch.cuda.current_device()
    if d not in _default_ctx:
        _default_ctx[d] = Context(d)
    return _default_ctx[d]


class ExpertWeights:
    """loader.swift:46-167.  Holds the caller's tensors (reference layout) alive and the native handle."""

    def __init__(self, buckets=None, stats=None, probes=None, outliers=None, core=None, *, inDim: int,
                 outDim: int, numExperts: int = 1, percentLoad: Optional[int] = None, kind: int = KIND_FP16,
                 flags: int = 0):
        L = _lib.load()
        self.inSize, self.outSize, self.numExperts, self.kind = inDim, outDim, numExperts, kind
        self.percentLoad = percentLoad if percentLoad is not None else (16 if kind == KIND_FP16 else 8)
        self.buckets, self.stats, self.probes, self.outliers, self.core = buckets, stats, probes, outliers, core
        self.bucketsLoaded = buckets is not None  # loader.swift:88,105
        if buckets is not None:
            _need(buckets, torch.float16, "buckets")
            _need(probes, torch.float16, "probes")
            _need(stats, torch.float16 if kind == KIND_FP16 else torch.float32, "stats")
            bsz = 16 if kind == KIND_FP16 else 32
            rows = numExperts * inDim * self.percentLoad
            if buckets.numel() != rows * (outDim // bsz):
                raise EffortError(f"buckets has {buckets.numel()} elements, expected {rows}x{outDim // bsz}")
            if stats.numel() != rows * (4 if kind == KIND_FP16 else 2):
                raise EffortError("stats shape mismatch")
            if probes.numel() != numExperts * 4096:
                raise EffortError("probes implemented for 4096 only (bucketMul.swift:36)")
        if outliers is not None:
            _need(outliers, torch.float32, "outliers")
        if core is not None:
            _need(core, torch.float16, "core")
        h = C.c_void_p()
        check(L.effort_weights_create(_ptr(buckets), _ptr(stats), _ptr(probes), _ptr(outliers),
                                      0 if outliers is None else outliers.shape[0], _ptr(core), inDim, outDim,
                                      numExperts, self.percentLoad, kind, flags, _stream_ptr(), C.byref(h)),
              "effort_weights_create")
        self._h, self._L = h, L

    def release_reference_layout(self):
        """Drop the caller-layout tensors (the handle owns a repacked copy + probes).  Afterwards only the fast
        path may be used: the calcDispatch/mul test hooks read the reference layout."""
        if self.buckets is not None and self.owned_bytes > 0:
            self.buckets = self.stats = self.probes = None

    @property
    def expertSize(self) -> int:  # loader.swift:50
        return self.percentLoad * self.inSize

    @property
    def owned_bytes(self) -> int:
        return int(self._L.effort_weights_owned_bytes(self._h))

    def hint(self) -> Optional[torch.Tensor]:
        """A live device view of the matrix's cutoff hints [n_experts] (effort_weights_hint, a test hook), or None."""
        ptr = self._L.effort_weights_hint(self._h)
        if not ptr:
            return None
        from .model import _tensor_from_ptr
        return _tensor_from_ptr(ptr, self.numExperts)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._L.effort_weights_destroy(self._h)
                self._h = None
        except Exception:
            pass


def _check_vec(v: torch.Tensor, n: int, name: str):
    _need(v, torch.float32, name)
    if v.numel() != n:
        raise EffortError(f"{name} has {v.numel()} elements, expected {n}")


def bucketMul(v, by: ExpertWeights, expNo=None, out=None, effort: float = 0.25, ctx: Optional[Context] = None):
    """bucketMul.swift:11.  v: VectorFloat[in], out: VectorFloat[out] (overwritten), expNo: device uint32 scalar."""
    ctx = ctx or default_context()
    _check_vec(v, by.inSize, "v")
    _check_vec(out, by.outSize, "out")
    check(ctx._L.effort_bucket_mul(ctx._h, v.data_ptr(), by._h, _ptr(expNo), out.data_ptr(), float(effort),
                                   _stream_ptr()), "bucketMul")
    return out


def bucketMulQ4(v, by: ExpertWeights, expNo=None, out=None, effort: float = 0.25, ctx: Optional[Context] = None):
    """bucketMulQ4.swift:11 (accumulates into `out`; expertMul zeroes it first)."""
    ctx = ctx or default_context()
    _check_vec(v, by.inSize, "v")
    _check_vec(out, by.outSize, "out")
    check(ctx._L.effort_bucket_mul_q4(ctx._h, v.data_ptr(), by._h, _ptr(expNo), out.data_ptr(), float(effort),
                                      _stream_ptr()), "bucketMulQ4")
    return out


def expertMul(v, by: ExpertWeights, expNo=None, out=None, effort: float = 0.25, ctx: Optional[Context] = None):
    """expertMul.swift:20-38."""
    ctx = ctx or default_context()
    _check_vec(v, by.inSize, "v")
    _check_vec(out, by.outSize, "out")
    check(ctx._L.effort_expert_mul(ctx._h, v.data_ptr(), by._h, _ptr(expNo), out.data_ptr(), float(effort),
                                   _stream_ptr()), "expertMul")
    return out


def expertMulBatch(calls: Sequence[tuple], ctx: Optional[Context] = None):
    """calls: [(v, by, expNo, out, effort[, vCutoff]), ...] independent expertMuls enqueued as one launch group.
    vCutoff (tensor-parallel row shards only): the first 4096 entries of the full input vector."""
    ctx = ctx or default_context()
    arr = (MulArgs * len(calls))()
    for k, call in enumerate(calls):
        v, by, expNo, out, effort = call[:5]
        v_cut = call[5] if len(call) > 5 else None
        _check_vec(v, by.inSize, "v")
        _check_vec(out, by.outSize, "out")
        if v_cut is not None:
            _need(v_cut, torch.float32, "vCutoff")
            if v_cut.numel() < 4096:
                raise EffortError("vCutoff must hold the first 4096 entries of the full input vector")
        arr[k] = MulArgs(v.data_ptr(), by._h, _ptr(expNo), out.data_ptr(), float(effort), _ptr(v_cut))
    check(ctx._L.effort_expert_mul_batch(ctx._h, arr, len(calls), _stream_ptr()), "expertMulBatch")


def basicMul(v, by: torch.Tensor, out, ctx: Optional[Context] = None):
    """helpers/mps.swift:14-47: dense fp16 [out,in] GEMV, v cast to fp16, fp32 result."""
    ctx = ctx or default_context()
    _need(by, torch.float16, "weights")
    rows, cols = by.shape
    _check_vec(v, cols, "v")
    _check_vec(out, rows, "out")
    check(ctx._L.effort_basic_mul(ctx._h, v.data_ptr(), by.data_ptr(), rows, cols, out.data_ptr(), _stream_ptr()),
          "basicMul")
    return out


# ---- test hooks (BucketMul.calcDispatch / mul, bucketMul.swift:34,69) ------------------------------------
def findCutoff(v, by: ExpertWeights, expNo=None, effort: float = 0.25, ctx: Optional[Context] = None):
    ctx = ctx or default_context()
    check(ctx._L.effort_find_cutoff(ctx._h, v.data_ptr(), by._h, _ptr(expNo), float(effort), _stream_ptr()),
          "findCutoff")
    c, loops = C.c_float(0), C.c_int(0)
    check(ctx._L.effort_read_dispatch(ctx._h, None, 0, None, None, C.byref(c), C.byref(loops), _stream_ptr()),
          "read")
    return float(c.value), int(loops.value)


def calcDispatch(v, by: ExpertWeights, expNo=None, effort: float = 0.25, ctx: Optional[Context] = None):
    ctx = ctx or default_context()
    _check_vec(v, by.inSize, "v")
    check(ctx._L.effort_calc_dispatch(ctx._h, v.data_ptr(), by._h, _ptr(expNo), float(effort), _stream_ptr()),
          "calcDispatch")


def readDispatch(by: ExpertWeights, ctx: Optional[Context] = None):
    """Returns dict(dispatch [padded,2] float32 numpy, n_selected, padded_size, cutoff, loops)."""
    import numpy as np
    ctx = ctx or default_context()
    cap = by.expertSize + 2048
    buf = np.zeros((cap, 2), dtype=np.float32)
    n, p, c, loops = C.c_uint32(0), C.c_uint32(0), C.c_float(0), C.c_int(0)
    check(ctx._L.effort_read_dispatch(ctx._h, buf.ctypes.data, cap, C.byref(n), C.byref(p), C.byref(c),
                                      C.byref(loops), _stream_ptr()), "readDispatch")
    return {"dispatch": buf[: p.value], "n_selected": n.value, "padded_size": p.value, "cutoff": float(c.value),
            "loops": loops.value}


def mul(by: ExpertWeights, out, ctx: Optional[Context] = None):
    ctx = ctx or default_context()
    _check_vec(out, by.outSize, "out")
    check(ctx._L.effort_mul(ctx._h, by._h, out.data_ptr(), _stream_ptr()), "mul")
    return out


def lastCutoff(ctx: Optional[Context] = None) -> float:
    """The cutoff the last fused operator (batch slot 0) on this context used."""
    ctx = ctx or default_context()
    c = C.c_float(0)
    check(ctx._L.effort_read_dispatch(ctx._h, None, 0, None, None, C.byref(c), None, _stream_ptr()), "read")
    return float(c.value)


def lastSelected(ctx: Optional[Context] = None) -> int:
    ctx = ctx or default_context()
    n = C.c_uint32(0)
    check(ctx._L.effort_last_selected(ctx._h, C.byref(n), _stream_ptr()), "lastSelected")
    return int(n.value)


def fusedMulBatch(calls: Sequence[dict], ctx: Optional[Context] = None):
    """One launch group of the fused decode chain (effort_fused_mul_batch).  Each call is a dict with
    v, by, out, effort and optionally norm (fp16 [in]: input = rmsNorm(v) * norm), eps (1e-5), x3 (input = silu(v) * x3),
    expNo (device uint32 scalar), scale (device f32 scalar: out (+)= scale * W(input)) and accumulate (False: overwrite)."""
    ctx = ctx or default_context()
    arr = (_lib.FusedArgs * len(calls))()
    for k, c in enumerate(calls):
        by, v, out = c["by"], c["v"], c["out"]
        _check_vec(v, by.inSize, "v")
        _check_vec(out, by.outSize, "out")
        x3, norm, scale = c.get("x3"), c.get("norm"), c.get("scale")
        if x3 is not None:
            _check_vec(x3, by.inSize, "x3")
        if norm is not None:
            _need(norm, torch.float16, "norm")
        if scale is not None:
            _need(scale, torch.float32, "scale")
        arr[k] = _lib.FusedArgs(v.data_ptr(), _ptr(x3), _ptr(norm), float(c.get("eps", 1e-5)), by._h, _ptr(c.get("expNo")),
                                _ptr(scale), out.data_ptr(), float(c["effort"]), 1 if c.get("accumulate") else 0)
    check(ctx._L.effort_fused_mul_batch(ctx._h, arr, len(calls), _stream_ptr()), "fusedMulBatch")


def lastProblem(slot: int = 0, ctx: Optional[Context] = None) -> tuple[float, int]:
    """(cutoff, selected rows) of batch slot `slot` of the last fused launch group on this context."""
    ctx = ctx or default_context()
    c, n = C.c_float(0), C.c_uint32(0)
    check(ctx._L.effort_last_problem(ctx._h, int(slot), C.byref(c), C.byref(n), _stream_ptr()), "lastProblem")
    return float(c.value), int(n.value)


def bucket_mul_multi(V: torch.Tensor, w: ExpertWeights, effort: float = 0.25, ctx: Optional[Context] = None):
    """The prefill's multi-token GEMV (effort_bucket_mul_multi): V [T][in] float32 on the device, T <= 16.  Returns
    (out [T][out], cutoffs [T] float32, counts [T] int32): each token's output, select-rule cutoff and selected-row count."""
    ctx = ctx or default_context()
    _need(V, torch.float32, "V")
    if V.dim() != 2 or V.shape[1] != w.inSize:
        raise ValueError(f"V must be [T][{w.inSize}], got {tuple(V.shape)}")
    T = V.shape[0]
    out = torch.empty(T, w.outSize, dtype=torch.float32, device=V.device)
    cut = torch.empty(T, dtype=torch.float32, device=V.device)
    cnt = torch.empty(T, dtype=torch.int32, device=V.device)
    check(ctx._L.effort_bucket_mul_multi(ctx._h, V.data_ptr(), T, w._h, out.data_ptr(), float(effort), cut.data_ptr(),
                                         cnt.data_ptr(), _stream_ptr()), "bucket_mul_multi")
    return out, cut, cnt


def sample(logits: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0, seed: int = 0, position: int = 0,
           ctx: Optional[Context] = None) -> torch.Tensor:
    """One draw from logits [V] f32 on the device (the rule of DESIGN.md section 4.6): temperature, top-k (0 = no limit),
    top-p (1 = no limit), Philox counter `position` under `seed`.  Returns a device int32 tensor [1]; no host sync."""
    ctx = ctx or default_context()
    _need(logits, torch.float32, "logits")
    out = torch.empty(1, dtype=torch.int32, device=logits.device)
    prm = Sampler(float(temperature), int(top_k), float(top_p), int(seed))
    check(ctx._L.effort_sample(ctx._h, logits.data_ptr(), logits.numel(), C.byref(prm), int(position), out.data_ptr(),
                               _stream_ptr()), "sample")
    return out


def score_columns(records: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """effort_score_t records held as int32 [n, 3] -> (argmax, rank, logprob) column views (logprob as float32)."""
    return records[:, 0], records[:, 1], records[:, 2].view(torch.float32)


def score(logits: torch.Tensor, targets: torch.Tensor, ctx: Optional[Context] = None):
    """Score each target token against logits [V] f32 on the device (the rule of DESIGN.md section 4.7), one record per
    target (device int32 [n]; outside [0, V) = no target).  Returns (argmax, ranks, logprobs), device tensors [n] (int32,
    int32, float32); argmax is the greedy token in every record.  No host sync."""
    ctx = ctx or default_context()
    _need(logits, torch.float32, "logits")
    _need(targets, torch.int32, "targets")
    rec = torch.empty((targets.numel(), 3), dtype=torch.int32, device=logits.device)
    check(ctx._L.effort_score(ctx._h, logits.data_ptr(), logits.numel(), targets.data_ptr(), targets.numel(), rec.data_ptr(),
                              _stream_ptr()), "score")
    return score_columns(rec)


def pdl_enabled() -> bool:
    """whether kernels are launched with programmatic dependent launch (EFFORT_PDL, read once per process)"""
    return bool(_lib.load().effort_pdl_enabled())


def launchCount() -> int:
    return int(_lib.load().effort_launch_count())


# ---- convert ------------------------------------------------------------------------------------------
def bucketize(w: torch.Tensor) -> dict:
    """convert.swift:209-260 (FP16): w [out,in] f16 cuda -> {'buckets','bucket.stats','probes'} (reference layout)."""
    L = _lib.load()
    _need(w, torch.float16, "w")
    out_dim, in_dim = w.shape
    dev = w.device
    buckets = torch.empty((in_dim * 16, out_dim // 16), dtype=torch.float16, device=dev)
    stats = torch.empty((in_dim * 16, 4), dtype=torch.float16, device=dev)
    probes = torch.empty((4096,), dtype=torch.float16, device=dev)
    check(L.effort_bucketize(w.data_ptr(), out_dim, in_dim, buckets.data_ptr(), stats.data_ptr(), probes.data_ptr(),
                             _stream_ptr()), "bucketize")
    return {"buckets": buckets, "bucket.stats": stats, "probes": probes}
