#!/usr/bin/env python
"""bench.py -- BASELINE.json's metric on BASELINE.json's config.

    python bench.py --gpus N --steps K --warmup W            (ours; under torchrun for N > 1)
    python bench.py --impl reference --gpus N --steps K ...  (CPU arm: the oracle port on the host cores)

Workload (config.workload): Mistral-7B FP16 single-stream decode (BASELINE.json configs[1]): 32 layers x
7 bucketMul GEMVs (4096->4096 x2, 4096->1024 x2, 4096->14336 x2, 14336->4096) + rmsnorm / rope / attention /
silu / residual + the dense 4096->32000 lm_head, random-initialised weights (no checkpoints offline), one
token per step from a fixed seeded token sequence.  A step = one token.  value = tokens/s at --effort (default 0.25, the
north-star operating point); the same run also reports effort 1.0 and 0.5 in `efforts`.

Timing: W warm-up tokens (>= 3), then exactly K tokens between CUDA events on the launching stream with a
barrier + synchronize on both sides, max over ranks.  Every token streams the selected rows of 14 GB of
distinct weights (>> 50 MB L2), so no L2 flush is needed between iterations (config.l2).

--dump-outputs DIR writes what the timed decode hands its caller after the last timed step: the logits
(DIR/logits.npy, float32 [vocab]) and the next token (DIR/next_token.npy, float64 [1]).  Weights and the first
tokens are seeded, so runs with the same arguments decode the same inputs, and the default kernels sum in a fixed
order, so they compute the same bits.  Two different builds that sum in different orders still drift apart at low
effort (rows move across the cutoff and the change grows through the 32 layers): compare their dumps with a tolerance
that fits the effort.

Besides the contract keys the line carries (rank 0, N = 1; each can be switched off, none touches the timed region):
  quality   per-token logit cos-sim of the effort-e decode against a DENSE decode of the same tokens (every projection
            through basicMul on the kept fp16 `core`; method: benchmarks/benchmark.swift:159-177, bar 0.99:
            playground.swift:41), for the N(0, 0.02^2) weights of the headline run and for a heavy-tailed init
  q4        BASELINE configs[2]: the Q4 model (bucketMulQ4 on wq/w1/w2/w3, dense wk/wv/wo) at effort 0.5
  sweep     BASELINE configs[4]: raw bucketMul GEMVs 4096 x {4096, 11008, 14336} x effort 1.0 .. 0.1
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "Mistral-7B decode tok/s @ effort"
SHAPES_PER_LAYER = [(4096, 4096), (4096, 1024), (4096, 1024), (4096, 4096), (4096, 14336), (4096, 14336), (14336, 4096)]
DENSE_LM_HEAD_BYTES = 32000 * 4096 * 2
BUCKET_BYTES_PER_TOKEN = 32 * sum(2 * i * o for i, o in SHAPES_PER_LAYER)  # 13.958 GB
Q4_BUCKETED = ("wq", "w1", "w2", "w3")                                      # q4_convert.py:53,59


def peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (HBM3, 3.35 TB/s), not a measured peak"


# ---------------------------------------------------------------------------------------------------------
# CPU arm: the reference has no CPU implementation (Swift+Metal only) -> the oracle port, all host threads
# ---------------------------------------------------------------------------------------------------------
def cpu_layer_sample(effort: float, reps: int = 5, seed: int = 1234):
    """One transformer layer's 7 GEMVs on the host cores (oracle port, OpenMP, the reference's bisection cutoff).
    Returns seconds per layer for the bucketMul port at `effort` and for the dense fp16 GEMV (basicMul,
    matrix.metal:150-162 -- the dense CPU baseline north_star asks for): MEDIAN of `reps` repetitions after one warm-up,
    min/max reported.  Thread count: the boxes expose 64-128 logical CPUs but SMT / cgroup quotas make "all of them"
    slower than fewer, so the count is chosen ONCE among {all, 1/2, 1/4} of the CPUs the process may run on by the median
    of three dense 4096->14336 GEMVs each (round 1 picked it from a single timed probe and landed on a 12x slower count
    on one box), then stays fixed and is reported as `cores`.  (Binding threads with OMP_PROC_BIND was tried: 400x slower
    inside these containers.)"""
    import numpy as np
    from oracle import oracle as O
    from tests.util import make_v, make_w
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    O.set_cutoff_mode("bisect")
    by_shape, dense = {}, {}
    for k, (i, o) in enumerate(sorted(set(SHAPES_PER_LAYER))):
        w = make_w(o, i, seed + k)
        dense[(i, o)] = w
        by_shape[(i, o)] = O.bucketize(w)
    vs = {i: make_v(i, 42) for i in (4096, 14336)}
    outs = {o: np.empty(o, np.float32) for o in (4096, 1024, 14336)}
    scr = {i: np.empty(2 * 16 * i, np.float32) for i in (4096, 14336)}

    def run_bucket():
        for (i, o) in SHAPES_PER_LAYER:
            r = by_shape[(i, o)]
            O.bucket_mul_mt(vs[i], r["buckets"], r["bucket.stats"], r["probes"], i, o, effort, outs[o], scr[i])

    def run_dense():
        for (i, o) in SHAPES_PER_LAYER:
            O.basic_mul_fast(vs[i], dense[(i, o)], outs[o])

    best_t, best_dt = 1, float("inf")
    probe_w, probe_out = dense[(4096, 14336)], outs[14336]
    for nt in sorted({avail, max(1, avail // 2), max(1, avail // 4)}, reverse=True):
        O.set_threads(nt)
        O.basic_mul_fast(vs[4096], probe_w, probe_out)   # warm this thread count
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            O.basic_mul_fast(vs[4096], probe_w, probe_out)
            ts.append(time.perf_counter() - t0)
        dt = sorted(ts)[1]
        if dt < best_dt:
            best_t, best_dt = nt, dt
    O.set_threads(best_t)
    res = {"threads": O.num_threads(), "reps": reps, "cpus_available": avail}
    for name, fn in (("bucketmul", run_bucket), ("dense", run_dense)):
        fn()  # warm-up (page faults, thread pool)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        ts.sort()
        res[name + "_s"] = ts[len(ts) // 2]
        res[name + "_min_s"], res[name + "_max_s"] = ts[0], ts[-1]
    res["sample"] = f"1 layer (7 GEMVs, 436 MB of buckets) x32 = 1 token, median of {reps} reps after 1 warm-up; lm_head excluded"
    return res


def cpu_record(r):
    return {"value": 1.0 / (r["bucketmul_s"] * 32), "unit": "tok/s", "cores": r["threads"], "kind": "port", "sample": r["sample"],
            "min": 1.0 / (r["bucketmul_max_s"] * 32), "max": 1.0 / (r["bucketmul_min_s"] * 32),
            "dense_gemv_tok_s": 1.0 / (r["dense_s"] * 32),
            "dense_gemv_min": 1.0 / (r["dense_max_s"] * 32), "dense_gemv_max": 1.0 / (r["dense_min_s"] * 32)}


def run_reference(args, rank, world):
    if rank != 0:
        return
    steps = max(1, args.steps)
    r = cpu_layer_sample(args.effort, reps=5)
    cb = cpu_record(r)
    tok_s = cb["value"]
    line = {
        "impl": "reference", "metric": f"{METRIC} {args.effort}", "value": tok_s, "unit": "tok/s", "n_gpus": args.gpus,
        "steps": steps, "warmup": args.warmup, "ms_per_step": r["bucketmul_s"] * 32 * 1e3, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "fp16 weights, f32 accumulate", "data": "synthetic",
        "config": workload_config(args, 1),
        "cpu_baseline": cb,
        "cpu_dense_gemv": {"value": cb["dense_gemv_tok_s"], "unit": "tok/s", "cores": r["threads"], "min": cb["dense_gemv_min"],
                           "max": cb["dense_gemv_max"],
                           "what": "dense fp16 GEMV (basicMul, matrix.metal:150-162) on the same layer sample"},
        "e2e": {"value": tok_s, "unit": "tok/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "note": "reference is Swift+Metal (no CPU path, not buildable here): CPU arm = oracle/ port of bucketMul, OpenMP",
    }
    print(json.dumps(line), flush=True)


def workload_config(args, world):
    return {"workload": "Mistral-7B FP16 single-stream decode, random-init, 32 layers, 1 token/step (BASELINE configs[1])",
            "effort": args.effort, "context": f"positions {args.warmup}..{args.warmup + args.steps}",
            "parallelism": "single GPU" if world == 1 else (
                f"{world} independent replicas" if getattr(args, "replicas", False) else
                f"tp{world}: q/k/v/w1/w3 column-sharded, wo/w2 row-sharded; per row-parallel GEMV one all-gather (cutoff "
                f"input) + one all-reduce as one-shot NVLink peer-memory kernels fused with silu*mul / residual+rmsNorm "
                f"(EFFORT_P2P=0: NCCL), vocab-sharded lm_head"),
            "l2": "14 GB of distinct weights per token >> 50 MB L2: no flush needed"}


# ---------------------------------------------------------------------------------------------------------
# ours
# ---------------------------------------------------------------------------------------------------------
def student_t_w(nu: float = 3.0, scale: float = 0.02):
    """Heavy-tailed synthetic init: every weight ~ scale * t_nu / sqrt(nu / (nu - 2)) (Student-t, unit variance before the
    scale): same variance as the Gaussian init, a few weights per bucket carry most of the mass -- the regime real
    transformer weights are in and the one the bucket order exploits."""
    import torch

    def fn(out_dim, in_dim, gen):
        z = torch.randn((out_dim, in_dim), generator=gen, device="cuda", dtype=torch.float32)
        # chi-square(nu) as a sum of nu squared normals (nu integer)
        c = torch.zeros((out_dim, in_dim), device="cuda", dtype=torch.float32)
        for _ in range(int(nu)):
            c += torch.randn((out_dim, in_dim), generator=gen, device="cuda", dtype=torch.float32) ** 2
        t = z / torch.sqrt(c / nu)
        return (t * (scale / (nu / (nu - 2.0)) ** 0.5)).half()
    return fn


def decode_quality(model_factory, dense_factory, effort, n_tokens):
    """Logit cos-sim, token by token, of the effort-e decode vs a dense decode fed the SAME tokens."""
    import numpy as np
    import torch
    from oracle import oracle as O
    m = model_factory()
    m.reset()
    toks, logits_e = [1], []
    buf = np.zeros(m.cfg.vocab, np.float32)
    nxt = m.step_host(1, effort, buf)
    logits_e.append(buf.copy())
    for _ in range(n_tokens - 1):
        toks.append(nxt)
        nxt = m.step_host(nxt, effort, buf)
        logits_e.append(buf.copy())
    d = dense_factory(m)
    d.reset()
    cs = []
    for t, le in zip(toks, logits_e):
        d.step_host(t, 1.0, buf)
        cs.append(O.cossim(le, buf))
    del d
    torch.cuda.empty_cache()
    return {"min": float(min(cs)), "mean": float(sum(cs) / len(cs)), "tokens": len(cs)}


def dense_twin(model):
    """Every projection as a Q4-kind ExpertWeights WITHOUT buckets: expertMul routes those to basicMul on `core`
    (expertMul.swift:26-31) -- the dense fp16 decode the quality is measured against."""
    from effort_b200 import ops
    from effort_b200.model import DecodeModel
    d = DecodeModel(model.cfg, model.ctx)
    for i, L in enumerate(model.layers):
        ews = [ops.ExpertWeights(core=w, inDim=w.shape[1], outDim=w.shape[0], kind=ops.KIND_Q4) for w in model.dense[i]]
        d.set_layer(i, *ews, L[7], L[8])
    d.set_head(*model.head)
    return d


def gemv_sweep(stream, shapes, efforts, peak):
    """BASELINE configs[4]: raw bucketMul GEMVs, graph replay over rotating weight copies (> 2x L2)."""
    import torch
    from effort_b200 import ops
    from tools.sweep import make_v_gpu, rand_weights
    rows = []
    for (in_dim, out_dim) in shapes:
        mat_bytes = 2 * in_dim * out_dim
        copies = max(2, -(-(300 << 20) // mat_bytes))
        ws = [rand_weights(out_dim, in_dim, 100 + c)[0] for c in range(copies)]
        torch.cuda.empty_cache()
        v = make_v_gpu(in_dim)
        out = torch.empty(out_dim, dtype=torch.float32, device="cuda")
        iters = 3 * copies
        for eff in efforts:
            for k in range(copies):
                ops.bucketMul(v, ws[k], None, out, eff)
            torch.cuda.synchronize()
            nsel = ops.lastSelected()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                for k in range(iters):
                    ops.bucketMul(v, ws[k % copies], None, out, eff)
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 8
            e0.record(stream)
            for _ in range(reps):
                g.replay()
            e1.record(stream)
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (reps * iters)
            alg = eff * mat_bytes
            rows.append({"shape": f"{in_dim}x{out_dim}", "effort": eff, "us": round(us, 2), "GBs": round(alg / us / 1e3, 1),
                         "frac": round(alg / us / 1e3 / peak, 3), "selected_frac": round(nsel / (in_dim * 16), 4)})
        del ws
        torch.cuda.empty_cache()
    return rows


def run_ours(args, rank, local_rank, world):
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from effort_b200 import ops
    from effort_b200.model import DecodeModel, MistralConfig, init_comm
    from tools.clocks import ClockSampler

    tp = world > 1 and not args.replicas
    if tp:
        init_comm(ops.default_context(), rank, world)
    streams_total = 1 if tp else world   # independent token streams in the job
    stream = torch.cuda.Stream()
    want_quality = rank == 0 and world == 1 and not args.quick and not args.no_quality
    with torch.cuda.stream(stream):
        # the KV cache must hold every timed position (the C++ loop refuses steps past max_seq, like the reference's maxSeqLen)
        cfg = MistralConfig(n_layers=args.layers, max_seq=max(2048, args.steps + max(3, args.warmup) + 8))
        if tp:   # one model, column/row sharded over the ranks (same seed everywhere)
            model = DecodeModel.random_init(cfg, seed=1234, tp_rank=rank, tp_size=world)
        else:
            model = DecodeModel.random_init(cfg, seed=1234 + rank, keep_dense=want_quality)
        torch.cuda.synchronize()

        def barrier():
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()

        def decode_device(effort, n_warm, n_steps):
            # tokens from a fixed seeded sequence rather than the model's own argmax: every step then decodes the same
            # input in every run and build (one argmax flipped by fp32 reordering would change all later inputs); a
            # step copies its token on the device either way
            n_warm = max(3, n_warm)
            toks = torch.randint(0, cfg.vocab, (n_warm + n_steps,), generator=torch.Generator().manual_seed(4242),
                                 dtype=torch.int32).cuda()
            toks[0] = 1
            toks = [toks[i:i + 1] for i in range(n_warm + n_steps)]
            model.reset()
            for tok in toks[:n_warm]:
                model.step(tok, effort)
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = ops.launchCount()
            e0.record(stream)
            for tok in toks[n_warm:]:
                model.step(tok, effort)
            e1.record(stream)
            barrier()
            ms = e0.elapsed_time(e1)
            return ms, ops.launchCount() - l0

        # headline: device-resident decode at --effort
        with ClockSampler(index=local_rank, period=0.02) as cs:
            ms, launches = decode_device(args.effort, args.warmup, args.steps)
        clocks = cs.summary()
        if args.dump_outputs and rank == 0:
            import numpy as np
            os.makedirs(args.dump_outputs, exist_ok=True)
            np.save(os.path.join(args.dump_outputs, "logits.npy"), model.logits().cpu().numpy().astype(np.float32))
            np.save(os.path.join(args.dump_outputs, "next_token.npy"), np.array([model.next_token()], np.float64))
        t = torch.tensor([ms], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
        tok_s = args.steps * streams_total / (ms / 1e3)

        # end to end: host token in (pinned, H2D), next token + logits out (D2H) every step
        import numpy as np
        logits = np.zeros(model.cfg.vocab, np.float32)
        model.reset()
        nxt = model.step_host(1, args.effort, logits)
        for _ in range(max(3, args.warmup) - 1):
            nxt = model.step_host(nxt, args.effort, logits)
        barrier()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            nxt = model.step_host(nxt, args.effort, logits)
        barrier()
        e2e_s = time.perf_counter() - t0
        t = torch.tensor([e2e_s], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_tok_s = args.steps * streams_total / float(t.item())

        extras = {}
        if not args.quick:   # every rank takes part: the sharded step holds collectives, and decode_device barriers
            for eff in (1.0, 0.5):
                if abs(eff - args.effort) < 1e-9:
                    continue
                ms_e, _ = decode_device(eff, 3, max(8, args.steps // 4))
                extras[str(eff)] = max(8, args.steps // 4) / (ms_e / 1e3)
        extras[str(args.effort)] = tok_s / streams_total

        # tensor parallel: the sharded model must compute what the unsharded one does (rank 0 holds both).  Asserted at
        # effort 1.0, where only the fp32 summation order differs; the bench effort is recorded next to it without a bar:
        # on a random-init network a low-effort selection is knife-edge and ANY reordering compounds through 32 layers
        # (DESIGN.md section 2, "Depth and chaos") -- the 2-layer comparison with a bar lives in tests/test_gpu_tp.py.
        tp_check = None
        if tp and not args.quick:
            ref_model = DecodeModel.random_init(cfg, seed=1234) if rank == 0 else None
            tp_check = {"tokens": 4}
            ok = [True]
            for eff, key in ((1.0, "logit_cos_sim_vs_unsharded_effort_1.0"), (args.effort, f"logit_cos_sim_vs_unsharded_effort_{args.effort}")):
                model.reset()
                cs_tp = []
                tok = torch.tensor([1], dtype=torch.int32, device="cuda")
                if rank == 0:
                    ref_model.reset()
                for _ in range(4):
                    model.step(tok, eff)
                    torch.cuda.synchronize()
                    if rank == 0:
                        ref_model.step(tok, eff)
                        torch.cuda.synchronize()
                        a, b = model.logits().double(), ref_model.logits().double()
                        cs_tp.append(float((a @ b) / (a.norm() * b.norm())))
                        tok = torch.tensor([ref_model.next_token()], dtype=torch.int32, device="cuda")
                    tl = [int(tok.item())]
                    dist.broadcast_object_list(tl, src=0)
                    tok = torch.tensor(tl, dtype=torch.int32, device="cuda")
                tp_check[key] = cs_tp
                if rank == 0 and eff == 1.0:
                    ok[0] = min(cs_tp) > 0.9995
            dist.broadcast_object_list(ok, src=0)      # every rank leaves together: a lone assert would strand the peers
            if not ok[0]:
                if rank == 0:
                    print(json.dumps({"error": "tensor-parallel logits diverge from the unsharded model", "tp_check": tp_check}))
                dist.destroy_process_group()
                raise SystemExit(3)
            if rank == 0:
                del ref_model
                torch.cuda.empty_cache()
            model.reset()

        # roofline of the dominant operator: bucketMul 4096 -> 14336 (w1/w3; 50 % of the bucket bytes with w2)
        roof = None
        if rank == 0:
            peak, peak_src = peaks()
            w1s = [L[4] for L in model.layers]            # 32 distinct 117 MB matrices: every launch reads HBM
            r_in, r_out = w1s[0].inSize, w1s[0].outSize   # 4096 -> 14336 (/world under TP)
            v = torch.randn(r_in, device="cuda", dtype=torch.float32)
            out = torch.empty(r_out, device="cuda", dtype=torch.float32)
            for w in w1s[:4]:
                ops.bucketMul(v, w, None, out, args.effort)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                for w in w1s:
                    ops.bucketMul(v, w, None, out, args.effort)
            g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 10
            e0.record(stream)
            for _ in range(reps):
                g.replay()
            e1.record(stream)
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (reps * len(w1s))
            alg = args.effort * r_in * r_out * 2
            ach = alg / us / 1e3
            roof = {"bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                    "kernel": f"bucketMul {r_in}->{r_out}: one launch of the fused round-2 kernel (cutoff + selection + TMA-staged "
                              f"gather-MAC + reductions into out)",
                    "us_per_launch": us, "algorithmic_bytes": alg, "peak_source": peak_src}

        def guarded(fn):
            try:
                return fn()
            except Exception as e:  # an optional record must never cost the headline line
                return {"error": f"{type(e).__name__}: {e}"[:300]}

        quality = q4 = sweep = None
        if want_quality:
            def q_headline():
                return {str(e): decode_quality(lambda: model, dense_twin, e, min(args.steps, 8)) for e in (1.0, 0.5, args.effort)}
            quality = {"what": "per-token logit cos-sim, effort-e decode vs a dense fp16 decode (every projection through basicMul "
                               "on its core) of the same tokens, all 32 layers.  NOTE: a random-init network has no trained "
                               "redundancy -- the per-GEMV approximation error (see per_operator) compounds through 224 GEMVs; "
                               "the reference's >= 0.99 figure is for trained Mistral weights (docs/ryc), which are not available "
                               "offline",
                       "gaussian N(0, 0.02^2) (headline weights)": guarded(q_headline)}

            def q_per_op():
                # one layer's seven operators on heavy-tailed activations (tests/util.make_v): bucketMul vs basicMul
                from tests.util import make_v
                import numpy as _np
                from oracle import oracle as O
                rows = {}
                for name, w_e, w_d in zip(("wq", "wk", "wv", "wo", "w1", "w2", "w3"), model.layers[0][:7], model.dense[0]):
                    v = torch.from_numpy(make_v(w_e.inSize, 42)).cuda()
                    out = torch.empty(w_e.outSize, dtype=torch.float32, device="cuda")
                    ref = torch.empty_like(out)
                    ops.basicMul(v, w_d, ref)
                    r = {}
                    for e in (1.0, 0.5, args.effort):
                        ops.bucketMul(v, w_e, None, out, e)
                        r[str(e)] = round(O.cossim(out.cpu().numpy(), ref.cpu().numpy()), 5)
                    rows[name] = r
                return rows
            quality["per_operator (layer 0, cos-sim of bucketMul vs dense basicMul)"] = guarded(q_per_op)
            model.dense = None
            torch.cuda.empty_cache()

        if rank == 0 and world == 1 and not args.quick and not args.no_extras:
            peak, _ = peaks()
            # free the headline model first: the extra records build their own
            del model
            torch.cuda.empty_cache()

            def q_heavy():
                hm = DecodeModel.random_init(cfg, seed=77, keep_dense=True, weight_fn=student_t_w(3.0))
                r = {str(e): decode_quality(lambda: hm, dense_twin, e, min(args.steps, 8)) for e in (1.0, 0.5, args.effort)}
                del hm
                torch.cuda.empty_cache()
                return r
            if quality is not None:
                quality["student-t(nu=3) * 0.02/sqrt(3), same variance as the Gaussian init"] = guarded(q_heavy)

            def q4_record():
                qm = DecodeModel.random_init_q4(cfg, seed=4321)
                qm.reset()
                tok = torch.tensor([1], dtype=torch.int32, device="cuda")
                qm.step(tok, 0.5)
                for _ in range(4):
                    qm.step(None, 0.5)
                torch.cuda.synchronize()
                n = max(8, args.steps // 2)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(n):
                    qm.step(None, 0.5)
                e1.record(stream)
                torch.cuda.synchronize()
                tps = n / (e0.elapsed_time(e1) / 1e3)
                # Q4 roofline operator: bucketMulQ4 4096 -> 14336 (w1), effort * in * out * 0.5 bytes of nibbles
                w1s = [L[4] for L in qm.layers]
                v = torch.randn(4096, device="cuda", dtype=torch.float32)
                out = torch.empty(14336, device="cuda", dtype=torch.float32)
                g = torch.cuda.CUDAGraph()
                for w in w1s[:2]:
                    ops.expertMul(v, w, None, out, 0.5)
                torch.cuda.synchronize()
                with torch.cuda.graph(g, stream=stream):
                    for w in w1s:
                        ops.expertMul(v, w, None, out, 0.5)
                g.replay()
                torch.cuda.synchronize()
                e0.record(stream)
                for _ in range(5):
                    g.replay()
                e1.record(stream)
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / (5 * len(w1s))
                alg = 0.5 * 4096 * 14336 * 0.5
                bytes_tok = args.layers * (0.5 * 0.5 * (4096 * 4096 + 3 * 4096 * 14336) + 2 * (2 * 4096 * 1024 + 4096 * 4096)) + DENSE_LM_HEAD_BYTES
                del qm
                torch.cuda.empty_cache()
                return {"workload": "Mistral-7B Q4 single-stream decode (BASELINE configs[2]): bucketMulQ4 + outliers on wq/w1/w2/w3, "
                                    "dense fp16 core on wk/wv/wo (q4_convert.py:53), effort 0.5", "value": tps, "unit": "tok/s",
                        "roofline": {"kernel": "expertMul Q4 4096->14336 (fused kernel + calcOutliers)", "us_per_launch": us,
                                     "algorithmic_bytes": alg, "achieved": alg / us / 1e3, "unit": "GB/s", "frac": alg / us / 1e3 / peak,
                                     "note": "outlier records (16 B x 2 % of the weights = 18.8 MB) are streamed on top of the nibbles"},
                        "token_bytes": bytes_tok, "token_roofline_frac": tps / (peak * 1e9 / bytes_tok)}
            q4 = guarded(q4_record)

            def sweep_record():
                effs = [1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3, 0.25, 0.2, 0.1]
                return {"what": "raw bucketMul GEMV (BASELINE configs[4]), one fused launch per call, graph replay over weight "
                                "copies > 2x L2", "rows": gemv_sweep(stream, [(4096, 4096), (4096, 11008), (4096, 14336)], effs, peak)}
            sweep = guarded(sweep_record)

        cpu = None
        if rank == 0 and world == 1 and not args.no_cpu:  # CPU baseline on rank 0 at N=1 only
            cpu = cpu_record(cpu_layer_sample(args.effort, reps=5))

        if rank == 0:
            peak, _ = peaks()
            bytes_tok = args.effort * BUCKET_BYTES_PER_TOKEN * args.layers / 32 + DENSE_LM_HEAD_BYTES
            roof_tok_s = peak * 1e9 / bytes_tok * (world if tp else 1)   # TP: every rank streams 1/world of the bytes
            line = {
                "metric": f"{METRIC} {args.effort}", "value": tok_s, "unit": "tok/s", "n_gpus": world, "steps": args.steps,
                "warmup": max(3, args.warmup), "ms_per_step": ms / args.steps, "higher_is_better": True,
                "scaling": "strong" if (tp or world == 1) else "weak", "vs_baseline": None, "dtype": "fp16 weights, f32 accumulate",
                "data": "synthetic", "config": workload_config(args, world),
                "e2e": {"value": e2e_tok_s, "unit": "tok/s", "h2d_bytes_per_step": 4, "d2h_bytes_per_step": 4 + 4 * cfg.vocab},
                "gpu_launches": int(launches),
                "clocks": {"sm_mhz": clocks["sm_mhz"], "sm_max_mhz": clocks["sm_max_mhz"], "reasons": clocks["reasons"],
                           "gpu": clocks["gpu"], "power_limit_w": clocks["power_limit_w"]},
                "roofline": roof, "cpu_baseline": cpu, "efforts": extras,
                "token_roofline": {"bytes_per_token": bytes_tok, "tok_s_at_peak": roof_tok_s,
                                   "frac": (tok_s / streams_total) / roof_tok_s},
                "quality": quality, "q4": q4, "sweep": sweep, "tp_check": tp_check,
            }
            print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--effort", type=float, default=0.25)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--quick", action="store_true", help="headline only: no effort 1.0 / 0.5, quality, q4, sweep records")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-quality", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the heavy-tail quality, q4 and sweep records")
    ap.add_argument("--replicas", action="store_true", help="N>1: independent replicas instead of tensor parallelism")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's logits and next token as DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank, world)
    else:
        run_ours(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
