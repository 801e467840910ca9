"""Batch-reduced fused product against the three ways a caller could sum a batch's products without it, on the workloads the
entry is for: the filter gradient of a convolution over NCHW data, a plain sum of large products, and a backward product
with a derivative op whose aux tensor has its own batch stride.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  reduce  laser_b200_gemm_strided_batch_reduce_f32_fused_dev: the concatenation along K written by the operand preparation
  loop    one laser_b200_gemm_strided_f32_fused_dev call per problem, beta = 1 after the first
  cat     torch.cat of the operands (and of the aux) along K, then one fused call over the concatenation
  torch   torch.einsum in fp32 with TF32 off (torch.where for the op)
Also: the preparation / GEMM split of the reduce call from the library's profile brackets (a run of its own), launches per
call, whether the reduce C equals the cat C bit for bit, and the card name and power limit read in the same run.

python tools/batch_reduce_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402


def fill(numel, seed, lo=-1.0, hi=1.0):
    t = torch.empty(numel, device="cuda")
    L.fill_uniform_f32(t, numel, seed, lo, hi)
    return t


def at(t, off):
    return L.DevPtr(t.data_ptr() + 4 * off, "f32")


def filter_gradient():
    """dW = sum_n dY_n cols_n^T: dY_n [64][56*56] (NCHW), cols_n [576][3136] from the im2col of image n, read transposed"""
    n, cin, cout, hw, k = 32, 64, 64, 56, 3
    ishape, kshape = (n, cin, hw, hw), (cout, cin, k, k)
    P, Kc = hw * hw, cin * k * k
    x, dy = fill(n * cin * P, 1), fill(n * cout * P, 2, -0.1, 0.1)
    cols = torch.empty(n * Kc * P, device="cuda")
    L.im2col(cols, x, ishape, kshape, (1, 1), (1, 1), images=n)
    C = torch.empty(cout * Kc, device="cuda")
    dy3, cols3 = dy.view(n, cout, P), cols.view(n, Kc, P)

    def loop():
        for i in range(n):
            L.gemm_strided_fused(cout, Kc, P, 1.0, at(dy, i * cout * P), P, 1, at(cols, i * Kc * P), 1, P, 1.0 if i else 0.0, C, Kc, 1)

    def cat():
        A, B = torch.cat(list(dy3), 1), torch.cat(list(cols3), 1)   # [64][nP], and B^ transposed [576][nP]
        L.gemm_strided_fused(cout, Kc, n * P, 1.0, A, n * P, 1, B, 1, n * P, 0.0, C, Kc, 1)

    return ("filter gradient 3x3, 56^2, 64 -> 64, 32 images (64 x 576, nK = 32 x 3136)", dict(
        reduce=lambda: L.gemm_strided_batch_reduce_fused(n, cout, Kc, P, 1.0, dy, P, 1, cout * P, cols, 1, P, Kc * P, 0.0, C, Kc, 1),
        loop=loop, cat=cat, torch=lambda: torch.einsum("bmp,bqp->mq", dy3, cols3), C=C, flops=2.0 * n * cout * Kc * P))


def big_sum():
    """64 products of 512^3 summed, row-major"""
    b, m = 64, 512
    A, B, C = fill(b * m * m, 3), fill(b * m * m, 4), torch.empty(m * m, device="cuda")
    A3, B3 = A.view(b, m, m), B.view(b, m, m)

    def loop():
        for i in range(b):
            L.gemm_strided_fused(m, m, m, 1.0, at(A, i * m * m), m, 1, at(B, i * m * m), m, 1, 1.0 if i else 0.0, C, m, 1)

    def cat():   # B's problems stacked row-major already are B^; A^ needs the copy
        L.gemm_strided_fused(m, m, b * m, 1.0, torch.cat(list(A3), 1), b * m, 1, B, m, 1, 0.0, C, m, 1)

    return ("64 x 512^3 summed", dict(
        reduce=lambda: L.gemm_strided_batch_reduce_fused(b, m, m, m, 1.0, A, m, 1, m * m, B, m, 1, m * m, 0.0, C, m, 1),
        loop=loop, cat=cat, torch=lambda: torch.einsum("bmk,bkn->mn", A3, B3), C=C, flops=2.0 * b * m ** 3))


def relu_grad_sum():
    """sum_b (dY_b . relu'(Z_b)) X_b, 32 problems of 512 x 512 x 1024, Z with its own batch stride (padded by 64 floats)"""
    b, M, N, K = 32, 512, 512, 1024
    zs = M * K + 64
    dY, Z, X, C = fill(b * M * K, 5, -0.1, 0.1), fill(b * zs, 6), fill(b * K * N, 7), torch.empty(M * N, device="cuda")
    dY3, X3 = dY.view(b, M, K), X.view(b, K, N)
    Z3 = Z.view(b, zs)[:, :M * K].reshape(b, M, K)

    def loop():
        for i in range(b):
            L.gemm_strided_fused(M, N, K, 1.0, at(dY, i * M * K), K, 1, at(X, i * K * N), N, 1, 1.0 if i else 0.0, C, N, 1,
                                 op_a=("relu_grad", at(Z, i * zs), K, 1))

    def cat():
        L.gemm_strided_fused(M, N, b * K, 1.0, torch.cat(list(dY3), 1), b * K, 1, X, N, 1, 0.0, C, N, 1,
                             op_a=("relu_grad", torch.cat(list(Z3), 1), b * K, 1))

    return ("relu_grad on A with batched aux: 32 x 512 x 512 x 1024 summed", dict(
        reduce=lambda: L.gemm_strided_batch_reduce_fused(b, M, N, K, 1.0, dY, K, 1, M * K, X, N, 1, K * N, 0.0, C, N, 1,
                                                         op_a=("relu_grad", Z, K, 1, zs)),
        loop=loop, cat=cat, torch=lambda: torch.einsum("bmk,bkn->mn", torch.where(Z3 > 0, dY3, torch.zeros_like(dY3)), X3),
        C=C, flops=2.0 * b * M * N * K))


def workloads():
    """-> [(name, dict(reduce, loop, cat, torch: calls; C; flops))], each workload's tensors in its own scope"""
    return [filter_gradient(), big_sum(), relu_grad_sum()]


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=".", help="directory for batch_reduce_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "unavailable", "reps": a.reps,
           "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "cases": []}
    lines = ["card (name, power limit, max SM clock, SM clock): %s" % res["nvidia_smi"],
             "medians over %d alternating timed calls, CUDA events; default fp32 mode %s" % (a.reps, res["f32_mode"]), ""]
    arms = ("reduce", "loop", "cat", "torch")
    for name, w in workloads():
        for _ in range(a.warmup):
            for arm in arms:
                w[arm]()
        torch.cuda.synchronize()
        launches, path = {}, None
        for arm in ("reduce", "loop", "cat"):
            n0 = L.launch_count()
            w[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path = path or _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))   # the reduce call's
        w["cat"](); torch.cuda.synchronize()
        ref = w["C"].clone()
        w["reduce"](); torch.cuda.synchronize()
        identical = bool(torch.equal(w["C"].view(torch.int32), ref.view(torch.int32)))
        got = w["C"].clone()
        want = w["torch"]().reshape(-1)
        rel = ((got.double() - want.double()).norm() / want.double().norm()).item()
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm in arms:
                ms[arm].append(timed(w[arm]))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        L.profile_begin()
        for _ in range(a.reps):
            w["reduce"]()
        torch.cuda.synchronize()
        prof = L.profile_end()
        split = dict(prep_ms=prof["prep_ms"] / a.reps, gemm_ms=prof["gemm_ms"] / a.reps,
                     prep_launches=prof["prep_launches"] / a.reps, gemm_launches=prof["gemm_launches"] / a.reps)
        case = dict(name=name, path=path, ms=med, ms_all=ms, tflops={k: w["flops"] / v / 1e9 for k, v in med.items()},
                    launches=launches, reduce_equals_cat_bitwise=identical, normwise_vs_torch_fp32=rel, profile=split)
        res["cases"].append(case)
        lines.append("%s [%s]\n  reduce %8.3f ms  loop %8.3f ms  cat %8.3f ms  torch %8.3f ms | reduce: prep %.3f ms (%g launches) "
                     "+ GEMM %.3f ms (%g launches) | launches loop %d cat %d | reduce == cat bitwise %s | vs torch %.2e"
                     % (name, path, med["reduce"], med["loop"], med["cat"], med["torch"], split["prep_ms"], split["prep_launches"],
                        split["gemm_ms"], split["gemm_launches"], launches["loop"], launches["cat"], identical, rel))
        print(lines[-1], flush=True)
    with open(os.path.join(a.out, "batch_reduce_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "batch_reduce_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
