"""Time and error of one fp32 tensor-core mode (f16x3 | tf32x3 | tf32x1) next to tf32x3 on one H100 -> one JSON line on stdout.

bench.py runs this in a CHILD process per mode (with a timeout) after all of its own measurements: the modes were written
after the round's GPU minutes were spent, so their first run on silicon must not be able to take the bench line down.
Also usable by hand:  python tools/two_piece_probe.py f16x3|tf32x3|tf32x1 [n] [steps]
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "f16x3"
    PATH = {"f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1}[name]
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 8192
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    L.init()
    dev = torch.device("cuda", 0)
    A = torch.empty(n * n, dtype=torch.float32, device=dev); B = torch.empty(n * n, dtype=torch.float32, device=dev)
    C = torch.empty(n * n, dtype=torch.float32, device=dev); Cd = torch.empty(n * n, dtype=torch.float32, device=dev)
    out = {"mode": name, "shape": [n, n, n]}
    # ---- error: against an fp64 product on a slab (2048 rows x 2048 columns x full K), both distributions
    m = min(n, 2048)
    for dist, (lo, hi) in (("P_U(0,1)", (0.0, 1.0)), ("S_U(-0.1,0.1)", (-0.1, 0.1))):
        L.fill_uniform_f32(A, n * n, 42, lo, hi); L.fill_uniform_f32(B, n * n, 43, lo, hi)
        C.fill_(float("nan")); Cd.fill_(float("nan"))
        L.gemm_strided(m, m, n, 1.0, A, n, 1, B, n, 1, 0.0, C, m, 1, path=PATH)
        assert L.last_path() == PATH
        L.gemm_strided(m, m, n, 1.0, A, n, 1, B, n, 1, 0.0, Cd, m, 1, path=L.PATH_TF32X3)
        torch.cuda.synchronize()
        exact = A.view(n, n)[:m, :].double() @ B.view(n, n)[:, :m].double()
        got = C[:m * m].view(m, m).double(); dflt = Cd[:m * m].view(m, m).double()
        e = {}
        for label, x in ((name, got), ("tf32x3", dflt)):
            d = (x - exact).abs()
            e[label] = {"max_rel": (d / exact.abs()).max().item(), "normwise": (torch.linalg.norm(x - exact) / torch.linalg.norm(exact)).item(),
                       "mean_relative_error": (d / exact.abs().clamp_min(1e-30)).mean().item()}
        out["error_vs_fp64_%s" % dist] = e
        del exact, got, dflt
    # ---- time at n^3 on the bench's distribution (S), device-resident, split pre-pass included
    f = lambda: L.gemm_strided(n, n, n, 1.0, A, n, 1, B, n, 1, 0.0, C, n, 1, path=PATH)
    ms = timed(f, steps, 3)
    L.profile_begin()
    for _ in range(3):
        f()
    prof = L.profile_end()
    msd = timed(lambda: L.gemm_strided(n, n, n, 1.0, A, n, 1, B, n, 1, 0.0, Cd, n, 1, path=L.PATH_TF32X3), steps, 3)
    flops = 2.0 * n * n * n
    out.update({"ms": ms, "tflops": flops / ms / 1e9, "kernel_ms": prof["gemm_ms"] / max(1, prof["gemm_launches"]),
                "prep_ms_per_step": prof["prep_ms"] / 3, "tf32x3_ms_same_process": msd,
                "speedup_vs_tf32x3": msd / ms})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
