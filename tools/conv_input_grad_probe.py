"""Fused convolution input gradient against the unfused route and torch, on the convolution layers of tools/conv_probe.py
(32 images each) and the reference's conv bench geometry.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  fused    laser_b200_conv2d_input_grad_f32_fused_dev: W' rotated once per call, B's transposed windows prepared straight
           from grad_output, the images of a chunk in one GEMM launch
  unfused  the batched fused product dcols_n = W^T * dY_n into an im2col-shaped [n][c_in * kH * kW][outH * outW] buffer, then
           torch.nn.functional.fold (the col2im scatter-add; both steps in the time)
  torch    torch.nn.grad.conv2d_input in fp32, cuDNN TF32 off
Both library arms run on PATH_AUTO.  Also: launches per call; the fused call's preparation and GEMM milliseconds
(laser_b200_profile_begin / _end, a run of its own); the per-kernel device time of the window pass and the filter rotation
from torch.profiler (another run of its own); the share of B's taps that are structural zeros (1 - 1 / (sH * sW) away from
the edges: what a strided layer multiplies and prepares for nothing); the normwise difference of each library arm to torch; and
the card name, power limit and SM clock read in the same run.

python tools/conv_input_grad_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402

WORKLOADS = [   # name, ishape, kshape, padding, strides
    ("3x3 56^2 64->64, 32 images", (32, 64, 56, 56), (64, 64, 3, 3), (1, 1), (1, 1)),
    ("3x3 28^2 128->128, 32 images", (32, 128, 28, 28), (128, 128, 3, 3), (1, 1), (1, 1)),
    ("3x3 14^2 256->256, 32 images", (32, 256, 14, 14), (256, 256, 3, 3), (1, 1), (1, 1)),
    ("3x3 stride 2 56^2 64->128, 32 images", (32, 64, 56, 56), (128, 64, 3, 3), (1, 1), (2, 2)),
    ("1x1 56^2 256->64, 32 images", (32, 256, 56, 56), (64, 256, 1, 1), (0, 0), (1, 1)),
    ("reference bench 224^2 3->20 3x3, 16 images", (16, 3, 224, 224), (20, 3, 3, 3), (0, 0), (1, 1)),
]


def fill(numel, seed, lo=-1.0, hi=1.0):
    t = torch.empty(numel, device="cuda")
    L.fill_uniform_f32(t, numel, seed, lo, hi)
    return t


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def zero_taps(H, W, kshape, padding, strides, oh, ow):
    """share of B's n * H * W x c_out * kH * kW taps that are structural zeros (between, before or past grad_output's pixels)"""
    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        return ((d >= 0) & (d % s == 0) & (d // s < out)).sum()
    kH, kW = kshape[2:]
    return 1.0 - axis(H, kH, padding[0], strides[0], oh) * axis(W, kW, padding[1], strides[1], ow) / float(H * kH * W * kW)


def workload(ishape, kshape, padding, strides):
    n, C, H, W = ishape
    cout, _, kH, kW = kshape
    _, _, oh, ow = L.conv2d_out_shape(ishape, kshape, padding, strides)
    P, Kc = oh * ow, C * kH * kW
    w, dy = fill(cout * Kc, 1), fill(n * cout * P, 2, -0.1, 0.1)
    dcols = torch.empty(n * Kc * P, device="cuda")
    dx_f = torch.empty(n * C * H * W, device="cuda")
    w4, dy4 = w.view(kshape), dy.view(n, cout, oh, ow)
    out = {}

    def fused():
        L.conv2d_input_grad_fused(dx_f, ishape, dy, w, kshape, padding, strides)

    def unfused():
        L.gemm_strided_batched_fused(n, Kc, P, cout, 1.0, w, 1, Kc, 0, dy, P, 1, cout * P, 0.0, dcols, P, 1, Kc * P)
        out["unfused"] = torch.nn.functional.fold(dcols.view(n, Kc, P), (H, W), (kH, kW), padding=padding, stride=strides)

    def tch():
        return torch.nn.grad.conv2d_input(ishape, w4, dy4, stride=strides, padding=padding)

    return dict(fused=fused, unfused=unfused, torch=tch, dx_f=dx_f, out=out, flops=2.0 * C * cout * kH * kW * n * H * W,
                zero_taps=zero_taps(H, W, kshape, padding, strides, oh, ow))


def kernel_times(fn, reps):
    """{kernel name: device ms per call} of `fn` from torch.profiler"""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = collections.defaultdict(float)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            out[e.key] += t / 1000.0 / reps
    return dict(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=".", help="directory for conv_input_grad_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "unavailable", "reps": a.reps,
           "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "cases": []}
    lines = ["card (name, power limit, max SM clock, SM clock): %s" % res["nvidia_smi"],
             "medians over %d alternating timed calls, CUDA events; default fp32 mode %s; TFLOP/s over the dense product "
             "2 * c_in * c_out * kH * kW * n * H * W" % (a.reps, res["f32_mode"]), ""]
    arms = ("fused", "unfused", "torch")
    for name, ishape, kshape, padding, strides in WORKLOADS:
        w = workload(ishape, kshape, padding, strides)
        for _ in range(a.warmup):
            for arm in arms:
                w[arm]()
        torch.cuda.synchronize()
        launches, path = {}, None
        for arm in ("fused", "unfused"):
            n0 = L.launch_count()
            w[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path = path or _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))   # the fused call's
        want = w["torch"]().reshape(-1).double()
        rel = {arm: ((x.reshape(-1).double() - want).norm() / want.norm()).item()
               for arm, x in (("fused", w["dx_f"]), ("unfused", w["out"]["unfused"]))}
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm in arms:
                ms[arm].append(timed(w[arm]))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        L.profile_begin()
        for _ in range(a.reps):
            w["fused"]()
        torch.cuda.synchronize()
        prof = L.profile_end()
        split = dict(prep_ms=prof["prep_ms"] / a.reps, gemm_ms=prof["gemm_ms"] / a.reps,
                     prep_launches=prof["prep_launches"] / a.reps, gemm_launches=prof["gemm_launches"] / a.reps)
        kt = kernel_times(w["fused"], a.reps)
        rows_ms = sum(v for k, v in kt.items() if "im2col_rows_kernel" in k)
        rot_ms = sum(v for k, v in kt.items() if "copy_strided_kernel" in k)
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, path=path, ms=med, ms_all=ms,
                    tflops={k: w["flops"] / v / 1e9 for k, v in med.items()}, launches=launches, profile=split, kernel_ms=kt,
                    window_rows_ms=rows_ms, rotation_ms=rot_ms, structural_zero_taps=w["zero_taps"], normwise_vs_torch_fp32=rel)
        res["cases"].append(case)
        lines.append("%s [%s]\n  fused %8.3f ms  unfused %8.3f ms  torch %8.3f ms | TFLOP/s fused %.1f torch %.1f | fused: prep "
                     "%.3f ms (%g launches; window rows %.3f ms, rotation %.3f ms) + GEMM %.3f ms (%g launches) | launches "
                     "unfused %d | structural-zero taps %.0f%% | vs torch fused %.2e unfused %.2e"
                     % (name, path, med["fused"], med["unfused"], med["torch"], case["tflops"]["fused"], case["tflops"]["torch"],
                        split["prep_ms"], split["prep_launches"], rows_ms, rot_ms, split["gemm_ms"], split["gemm_launches"],
                        launches["unfused"], 100 * w["zero_taps"], rel["fused"], rel["unfused"]))
        print(lines[-1], flush=True)
        del w
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "conv_input_grad_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_input_grad_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
