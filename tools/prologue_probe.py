"""Prologue fusion at backward-pass shapes: the plain product, the fused call (RELU_GRAD, TANH_GRAD on the operand) and the
unfused sequence (a torch elementwise product writing dY', then the plain product), timed alternately after warm-up with
CUDA events; prep_ms / gemm_ms of each from laser_b200_profile_begin/end (separate, profiled runs); parity of fused vs
unfused.

    dX = dY' . W^T : A = dY (row-major, K-major), op on A, B = W^T (K-major)
    dW = X^T . dY' : A = X^T (MN-major), B = dY (row-major: the MN-major preparation), op on B

python tools/prologue_probe.py [--sizes 8192 4096] [--reps 10] [--out DIR]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[8192, 4096])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=".", help="directory for prologue_probe.json")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    dev = torch.cuda.get_device_name(0)
    results = {"device": dev, "cases": []}
    for n in a.sizes:
        M = N = K = n
        def f(numel, seed, lo, hi):
            t = torch.empty(numel, device="cuda")
            L.fill_uniform_f32(t, numel, seed, lo, hi)
            return t
        dY = {"dX": f(M * K, 1, -0.1, 0.1), "dW": f(K * N, 1, -0.1, 0.1)}
        aux = {("dX", "relu_grad"): f(M * K, 2, -1, 1), ("dX", "tanh_grad"): f(M * K, 3, -1, 1),
               ("dW", "relu_grad"): f(K * N, 2, -1, 1), ("dW", "tanh_grad"): f(K * N, 3, -1, 1)}
        W = f(N * K, 4, -0.1, 0.1)          # dX: B = W^T, W stored N x K row-major
        X = f(K * M, 5, -0.1, 0.1)          # dW: A = X^T, X stored K x M row-major
        buf = torch.empty(max(M * K, K * N), device="cuda")
        C = torch.empty(M * N, device="cuda")

        def plain(kind, g):
            if kind == "dX":
                L.gemm_strided(M, N, K, 1.0, g, K, 1, W, 1, K, 0.0, C, N, 1, path=L.PATH_F16X3)
            else:
                L.gemm_strided(M, N, K, 1.0, X, 1, M, g, N, 1, 0.0, C, N, 1, path=L.PATH_F16X3)

        def fused(kind, op):
            z = aux[(kind, op)]
            if kind == "dX":
                L.gemm_strided_fused(M, N, K, 1.0, dY[kind], K, 1, W, 1, K, 0.0, C, N, 1, path=L.PATH_F16X3, op_a=(op, z, K, 1))
            else:
                L.gemm_strided_fused(M, N, K, 1.0, X, 1, M, dY[kind], N, 1, 0.0, C, N, 1, path=L.PATH_F16X3, op_b=(op, z, N, 1))

        def unfused(kind, op):
            z, g = aux[(kind, op)], buf[:dY[kind].numel()]
            if op == "relu_grad":
                torch.mul(dY[kind], z > 0, out=g)
            else:
                torch.mul(dY[kind], 1 - z * z, out=g)
            plain(kind, g)

        for kind in ("dX", "dW"):
            variants = {"a_plain": lambda: plain(kind, dY[kind])}
            for op in ("relu_grad", "tanh_grad"):
                variants["b_fused_" + op] = (lambda op=op: fused(kind, op))
                variants["c_unfused_" + op] = (lambda op=op: unfused(kind, op))
            for fn in variants.values():
                for _ in range(a.warmup):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in variants}
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in variants]
            for _ in range(a.reps):                      # alternating: every rep runs every variant once
                for (name, fn), (e0, e1) in zip(variants.items(), ev):
                    e0.record(); fn(); e1.record()
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1))
            prof = {}
            for name, fn in variants.items():
                L.profile_begin(); fn(); prof[name] = L.profile_end()
            parity = {}
            for op in ("relu_grad", "tanh_grad"):
                fused(kind, op); ref_c = C.clone()
                unfused(kind, op); torch.cuda.synchronize()
                parity[op] = ((ref_c.double() - C.double()).norm() / C.double().norm()).item()
            case = {"n": n, "product": kind, "parity_fused_vs_unfused_normwise": parity, "variants": {}}
            for name in variants:
                case["variants"][name] = {"median_ms": statistics.median(times[name]), "min_ms": min(times[name]),
                                          "prep_ms": prof[name]["prep_ms"], "gemm_ms": prof[name]["gemm_ms"],
                                          "prep_launches": prof[name]["prep_launches"]}
            results["cases"].append(case)
            print("%s %d^3" % (kind, n))
            for name, v in case["variants"].items():
                print("  %-22s step %.3f ms (min %.3f)  prep %.3f ms (%d launches)  gemm %.3f ms" %
                      (name, v["median_ms"], v["min_ms"], v["prep_ms"], v["prep_launches"], v["gemm_ms"]))
            print("  parity fused vs unfused (normwise):", parity)
            sys.stdout.flush()
    with open(os.path.join(a.out, "prologue_probe.json"), "w") as fh:
        json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
