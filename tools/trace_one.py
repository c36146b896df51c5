"""Phase timeline of the fused kernel (EFFORT_TRACE=1): per-CTA globaltimer stamps."""
import argparse, ctypes as C, os, sys
import numpy as np
os.environ["EFFORT_TRACE"] = "1"
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
for k in range(200):
    ops.bucketMul(v, ws[k % 4], None, out, a.effort)
torch.cuda.synchronize()
names = ["start", "zeroed", "issued", "scored", "minmax", "phaseA", "cutoff", "masks", "listed", "streamed", "partial"]
for rep in range(3):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    ops.bucketMul(v, ws[rep % 4], None, out, a.effort)
    e.record()
    torch.cuda.synchronize()
    n_sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    buf = np.zeros((n_sms, 16), dtype=np.uint64)
    n = L.effort_debug_read_trace(ctx._h, buf.ctypes.data, n_sms)
    t = buf[:n, :11].astype(np.int64)
    loops = buf[:n, 11:13]
    sorted_t = buf[:n, 13].astype(np.int64)
    comp_t = buf[:n, 14].astype(np.int64)
    print("   replay iterations:", int(buf[0, 15]), " compacted at median",
          float(np.median((comp_t[comp_t > 0] - buf[:n, 0].astype(np.int64)[buf[:n, 0] > 0].min()) / 1000.0)) if (comp_t > 0).any() else None)
    t = t[t[:, 0] > 0]
    t0 = t[:, 0].min()
    rel = (t - t0) / 1000.0
    print(f"{a.shape} effort {a.effort} rep {rep}: event total {s.elapsed_time(e)*1000:.1f} us; ctas {len(t)}")
    print("   loops after phase A / total:", int(loops[0, 0]), int(loops[0, 1]),
          " rank-sorted at median", float(np.median((sorted_t[sorted_t > 0] - t0) / 1000.0)) if (sorted_t > 0).any() else None)
    for k, nm in enumerate(names):
        print(f"   {nm:9s} min {rel[:,k].min():7.2f}  median {np.median(rel[:,k]):7.2f}  max {rel[:,k].max():7.2f} us")
