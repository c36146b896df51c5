"""Timeline of one isolated launch of the default fused kernel (bucket_mul_v4_kernel).  EFFORT_TRACE=1: per-CTA
global-timer stamps of the phases + SM-cycle stamps of CTA 0 (prologue steps, every chunk of pair 0, when each consumer
ran dry).  EFFORT_TRACE=2: the cycle stamps only -- the global-timer reads perturb the serial prologue."""
import argparse, ctypes as C, os, sys
import numpy as np
os.environ.setdefault("EFFORT_TRACE", "1")
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from effort_b200 import ops, _lib  # noqa: E402
from tools.sweep import rand_weights, make_v_gpu  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--shape", default="4096x14336")
ap.add_argument("--effort", type=float, default=0.25)
a = ap.parse_args()
in_dim, out_dim = (int(x) for x in a.shape.split("x"))
ws = [rand_weights(out_dim, in_dim, 100 + c)[0] for c in range(4)]
v = make_v_gpu(in_dim)
out = torch.empty(out_dim, dtype=torch.float32, device="cuda")
ctx = ops.default_context()
L = _lib.load()
L.effort_debug_read_trace.restype = C.c_int
L.effort_debug_read_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
L.effort_debug_read_unit_trace.restype = C.c_int
L.effort_debug_read_unit_trace.argtypes = [C.c_void_p, C.c_void_p]
for k in range(200):
    ops.bucketMul(v, ws[k % 4], None, out, a.effort)
torch.cuda.synchronize()
names = {0: "start", 1: "init done", 2: "v loaded", 3: "scored", 6: "cutoff", 8: "listed", 9: "streamed", 10: "reduced"}
for rep in range(3):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    ops.bucketMul(v, ws[rep % 4], None, out, a.effort)
    e.record()
    torch.cuda.synchronize()
    n_sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    buf = np.zeros((n_sms, 16), dtype=np.uint64)
    n = L.effort_debug_read_trace(ctx._h, buf.ctypes.data, n_sms)
    t = buf[:n].astype(np.int64)
    t = t[t[:, 0] > 0]
    if len(t) == 0:          # EFFORT_TRACE=2: cycle stamps only
        t = np.zeros((1, 16), dtype=np.int64)
    t0 = t[:, 0].min()
    print(f"{a.shape} effort {a.effort} rep {rep}: event total {s.elapsed_time(e)*1000:.1f} us; ctas {len(t)}; selected {ops.lastSelected()}")
    for k, nm in names.items():
        rel = (t[:, k] - t0) / 1000.0
        print(f"   {nm:10s} min {rel.min():7.2f}  median {np.median(rel):7.2f}  max {rel.max():7.2f} us")
    ub = np.zeros(648 + 48 + 16, dtype=np.uint64)
    if L.effort_debug_read_unit_trace(ctx._h, ub.ctypes.data) == 0 and rep == 2:
        base = int(ub[640])
        u = ub[:640].reshape(80, 8).astype(np.int64)
        cs = ub[696:710].astype(np.int64)
        lab = ["entry", "dependency wait over", "products scored", "select done", "cutoff broadcast", "masks", "records stored",
               "list barrier", "consumers done", "tiles reduced", "(v normalised", "constants", "loop top", "16 tests)"]
        print("   CTA 0 thread 0, SM cycles since kernel entry: " + "; ".join(f"{l} {int(c - cs[0])}" for l, c in zip(lab, cs) if c))
        fin = ub[648:696].astype(np.int64)
        print("   consumers of CTA 0: ran dry at cycle / rows / chunks:",
              "  ".join(f"{int(fin[w]) - base if fin[w] else -1}/{int(fin[16 + w])}/{int(fin[32 + w])}" for w in range(8)))
        print("   chunks of pair 0, CTA 0 -- SM cycles since the CTA started: rows | producer issued | consumer: starts waiting, "
              "barrier passed, records read, first piece done, all rows done, slot released")
        for k in range(80):
            if u[k, 0] == 0:
                break
            c = [int(u[k, j]) - base if u[k, j] else -1 for j in (0, 1, 2, 4, 5, 6, 7)]
            print(f"     chunk {k:2d}: {int(u[k,3]):2d} rows | {c[0]:6d} | {c[1]:6d} {c[2]:6d} {c[3]:6d} {c[4]:6d} {c[5]:6d} {c[6]:6d}")
