"""Batched fused product against the per-problem loop and torch, on the workloads that decide whether the batched entry
should replace the loop: many small problems, a backward product over a batch, a convolution image by image, and a batch
whose problems already fill the GPU on their own (the regression check).

Per workload, alternating after warm-up, medians over --reps timed steps (CUDA events around each call):
  batched  laser_b200_gemm_strided_batched_f32_fused_dev
  loop     laser_b200_gemm_strided_batched_f32_dev (one launch sequence per problem), or one _fused_dev call per problem
           where an op is involved
  torch    torch.bmm / torch.matmul in fp32 with TF32 off, plus an elementwise kernel for the op
Also: launches per call (laser_b200_launch_count), whether the batched C equals the loop's bit for bit, and the card name
and power limit read in the same run.

python tools/batched_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
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
from laser_b200 import gemm as G  # noqa: E402


def fill(numel, seed, lo=-1.0, hi=1.0):
    t = torch.empty(numel, device="cuda")
    L.fill_uniform_f32(t, numel, seed, lo, hi)
    return t


def loop_plain(batch, M, N, K, A, rsA, csA, bsA, B, rsB, csB, bsB, C, rsC, bsC):
    _capi.check(_capi.lib().laser_b200_gemm_strided_batched_f32_dev(batch, M, N, K, 1.0, A.data_ptr(), rsA, csA, bsA, B.data_ptr(),
                                                                rsB, csB, bsB, 0.0, C.data_ptr(), rsC, 1, bsC, L.PATH_AUTO,
                                                                G._current_stream()))


def workloads():
    """-> name, (batched call, loop call, torch call, C tensor, flops)"""
    out = []

    def plain(name, batch, M, N, K):
        A, B, C = fill(batch * M * K, 1), fill(batch * K * N, 2), torch.empty(batch * M * N, device="cuda")
        A3, B3 = A.view(batch, M, K), B.view(batch, K, N)
        return (name, dict(
            batched=lambda: L.gemm_strided_batched_fused(batch, M, N, K, 1.0, A, K, 1, M * K, B, N, 1, K * N, 0.0, C, N, 1, M * N),
            loop=lambda: loop_plain(batch, M, N, K, A, K, 1, M * K, B, N, 1, K * N, C, N, M * N),
            torch=lambda: torch.bmm(A3, B3), C=C, flops=2.0 * batch * M * N * K))

    out.append(plain("64 x 512^3 row-major", 64, 512, 512, 512))
    out.append(plain("256 x 256^3", 256, 256, 256, 256))

    def backward(name, batch, M, N, K):
        """dX_b = (dY_b . relu'(Z_b)) W^T, W (N x K row-major) shared"""
        dY, Z, W = fill(batch * M * K, 3, -0.1, 0.1), fill(batch * M * K, 4), fill(N * K, 5, -0.1, 0.1)
        C = torch.empty(batch * M * N, device="cuda")

        def loop():
            for b in range(batch):
                L.gemm_strided_fused(M, N, K, 1.0, L.DevPtr(dY.data_ptr() + 4 * b * M * K, "f32"), K, 1, W, 1, K, 0.0,
                                     L.DevPtr(C.data_ptr() + 4 * b * M * N, "f32"), N, 1,
                                     op_a=("relu_grad", L.DevPtr(Z.data_ptr() + 4 * b * M * K, "f32"), K, 1))
        return (name, dict(
            batched=lambda: L.gemm_strided_batched_fused(batch, M, N, K, 1.0, dY, K, 1, M * K, W, 1, K, 0, 0.0, C, N, 1, M * N,
                                                         op_a=("relu_grad", Z, K, 1, M * K)),
            loop=loop,
            torch=lambda: torch.matmul(torch.where(Z > 0, dY, torch.zeros_like(dY)).view(batch, M, K), W.view(N, K).t()),
            C=C, flops=2.0 * batch * M * N * K))

    def conv(name, batch, M, K, N):
        """shared filters (M x K) times each image's im2col matrix (K x N, N-major)"""
        F, X, C = fill(M * K, 6), fill(batch * K * N, 7), torch.empty(batch * M * N, device="cuda")
        return (name, dict(
            batched=lambda: L.gemm_strided_batched_fused(batch, M, N, K, 1.0, F, K, 1, 0, X, N, 1, K * N, 0.0, C, N, 1, M * N),
            loop=lambda: loop_plain(batch, M, N, K, F, K, 1, 0, X, N, 1, K * N, C, N, M * N),
            torch=lambda: torch.matmul(F.view(M, K), X.view(batch, K, N)), C=C, flops=2.0 * batch * M * N * K))

    out.append(backward("32 x (dY . relu'(Z)) W^T, 512 x 1024 x 1024, W shared", 32, 512, 1024, 1024))
    out.append(conv("conv: 32 images, filters 64 x 576 shared, 576 x 3136 per image", 32, 64, 576, 3136))
    out.append(plain("8 x 2048^3", 8, 2048, 2048, 2048))
    return out


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
    ap.add_argument("--out", default=".", help="directory for batched_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "unavailable", "reps": a.reps,
           "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "cases": []}
    lines = ["card: %s" % res["nvidia_smi"], "medians over %d alternating timed calls, CUDA events; default fp32 mode %s"
             % (a.reps, res["f32_mode"]), ""]
    for name, w in workloads():
        arms = ("batched", "loop", "torch")
        for _ in range(a.warmup):
            for arm in arms:
                w[arm]()
        torch.cuda.synchronize()
        launches = {}
        for arm in ("batched", "loop"):
            n0 = L.launch_count()
            w[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
        w["loop"](); torch.cuda.synchronize()
        ref = w["C"].clone()
        w["batched"](); torch.cuda.synchronize()
        identical = bool(torch.equal(w["C"].view(torch.int32), ref.view(torch.int32)))
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm in arms:
                ms[arm].append(timed(w[arm]))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        case = dict(name=name, ms=med, ms_all=ms, tflops={k: w["flops"] / v / 1e9 for k, v in med.items()}, launches=launches,
                    batched_equals_loop_bitwise=identical, path=_capi.PATH_NAMES.get(L.last_path(), str(L.last_path())))
        res["cases"].append(case)
        lines.append("%-62s batched %8.3f ms  loop %8.3f ms  torch %8.3f ms | launches batched %d loop %d | bit-identical %s"
                     % (name, med["batched"], med["loop"], med["torch"], launches["batched"], launches["loop"], identical))
        print(lines[-1], flush=True)
    with open(os.path.join(a.out, "batched_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "batched_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
