"""Interleaved A/B timing (the GPU may be power-capped: sequential blocks of runs are not comparable).

Products and pre-packs at 8192^3.  LASER_B200_LIB selects another build of the library, so that two builds can be timed
alternately in one session."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, laser_b200 as L
torch.cuda.set_device(0); L.init()
n = 8192
a = torch.rand(n, n, device="cuda"); b = torch.rand(n, n, device="cuda"); c = torch.empty(n, n, device="cuda")
bt = b.t().contiguous()
pa = L.alloc_packed(L.gemm_prepackA_mem_required(n, n, n)); pb = L.alloc_packed(L.gemm_prepackB_mem_required(n, n, n))
L.gemm_prepackA(pa, n, n, n, a, n, 1); L.gemm_prepackB(pb, n, n, n, b, n, 1)
variants = {   # name: (call, calls per sample, a product?)
    "default row,row (split each call)": (lambda: L.gemm_strided(n, n, n, 1.0, a, n, 1, b, n, 1, 0.0, c, n, 1), 2, True),
    "default row,B^T (both K-major)": (lambda: L.gemm_strided(n, n, n, 1.0, a, n, 1, bt, 1, n, 0.0, c, n, 1), 2, True),
    "packedB": (lambda: L.gemm_packedB(n, n, n, 1.0, a, n, 1, pb, 0.0, c, n, 1), 2, True),
    "packed A+B": (lambda: L.gemm_packed(n, n, n, 1.0, pa, pb, 0.0, c, n, 1), 2, True),
    "x3": (lambda: L.gemm_strided(n, n, n, 1.0, a, n, 1, b, n, 1, 0.0, c, n, 1, path=L.PATH_TF32X3), 2, True),
    "x1": (lambda: L.gemm_strided(n, n, n, 1.0, a, n, 1, b, n, 1, 0.0, c, n, 1, path=L.PATH_TF32X1), 2, True),
    "prepackA, A row-major": (lambda: L.gemm_prepackA(pa, n, n, n, a, n, 1), 10, False),
    "prepackB, B column-major": (lambda: L.gemm_prepackB(pb, n, n, n, bt, 1, n), 10, False),
}
times = {k: [] for k in variants}
for f, _, _ in variants.values():
    f()
torch.cuda.synchronize()
for rnd in range(12):
    for k, (f, calls, _) in variants.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            f()
        e1.record(); torch.cuda.synchronize()
        times[k].append(e0.elapsed_time(e1) / calls)
print("library:", os.environ.get("LASER_B200_LIB") or L.lib_path())
for k, v in times.items():
    med = statistics.median(v)
    rate = "-> %.1f TFLOP/s (median)" % (2 * n**3 / med / 1e9) if variants[k][2] else ""
    print("%-36s median %.3f ms  min %.3f  %s" % (k, med, min(v), rate))
