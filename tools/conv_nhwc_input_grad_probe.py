"""Channels-last convolution input gradient against the routes a user has without it, on the workloads of
tools/conv_nhwc_filter_grad_probe.py.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call), every library arm on
PATH_AUTO, the filters given as torch's channels_last weight [c_out][kH][kW][c_in] (the filter matrix read with strides (1, K)):
  nhwc     laser_b200_conv2d_nhwc_input_grad_f32_fused_dev on the NHWC gradients
  nchw     laser_b200_conv2d_input_grad_f32_fused_dev on NCHW copies of the same data (made before the timing)
  convert  the conversion route, timed whole: nhwc2nchw of dY, the filters permuted to [c_out][c_in][kH][kW] (torch), the
           NCHW entry, nchw2nhwc of dX
  torch    torch.nn.grad.conv2d_input on channels_last tensors in fp32, cuDNN TF32 off
Also: launches per call; the nhwc call's preparation and GEMM milliseconds (laser_b200_profile_begin / _end, a run of its own);
the per-kernel device time of the window passes (im2col_rows_kernel) of the nhwc and nchw calls (torch.profiler, another run of
its own); how far the nhwc and convert results lie apart next to their distance from torch; and the card name, power limit and
SM clocks read in the same run.

python tools/conv_nhwc_input_grad_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402

WORKLOADS = [   # name, ishape, kshape, padding, strides (tools/conv_nhwc_filter_grad_probe.py's)
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


def workload(ishape, kshape, padding, strides):
    n, C, H, W = ishape
    cout, _, kH, kW = kshape
    _, _, oh, ow = L.conv2d_out_shape(ishape, kshape, padding, strides)
    K = C * kH * kW
    w = fill(cout * K, 1)                                                          # [c_out][kH][kW][c_in]
    dy = fill(n * oh * ow * cout, 2, -0.1, 0.1)                                    # NHWC
    w_nchw = w.view(cout, kH, kW, C).permute(0, 3, 1, 2).contiguous()
    dy_nchw = torch.empty_like(dy)
    L.nhwc2nchw(dy_nchw, dy, n, cout, oh, ow)
    dyc, dx_tmp = torch.empty_like(dy), torch.empty(n * C * H * W, device="cuda")  # the conversion route's own buffers
    dx_h, dx_n, dx_c = (torch.empty(n * H * W * C, device="cuda") for _ in range(3))
    w4 = w.view(cout, kH, kW, C).permute(0, 3, 1, 2)                               # channels_last views
    dy4 = dy.view(n, oh, ow, cout).permute(0, 3, 1, 2)
    wmat = w.view(cout, K).t()

    def nhwc():
        L.conv2d_nhwc_input_grad_fused(dx_h, ishape, dy, wmat, kshape, padding, strides)

    def nchw():
        L.conv2d_input_grad_fused(dx_n, ishape, dy_nchw, w_nchw, kshape, padding, strides)

    def convert():
        L.nhwc2nchw(dyc, dy, n, cout, oh, ow)
        wc = w4.contiguous()
        L.conv2d_input_grad_fused(dx_tmp, ishape, dyc, wc, kshape, padding, strides)
        L.nchw2nhwc(dx_c, dx_tmp, n, C, H, W)

    def tch():
        return torch.nn.grad.conv2d_input(ishape, w4, dy4, stride=strides, padding=padding)

    return dict(nhwc=nhwc, nchw=nchw, convert=convert, torch=tch, dx_h=dx_h, dx_c=dx_c, flops=2.0 * n * H * W * C * cout * kH * kW)


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
    ap.add_argument("--out", default=".", help="directory for conv_nhwc_input_grad_probe.json / .txt")
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
    arms = ("nhwc", "nchw", "convert", "torch")
    for name, ishape, kshape, padding, strides in WORKLOADS:
        w = workload(ishape, kshape, padding, strides)
        for _ in range(a.warmup):
            for arm in arms:
                w[arm]()
        torch.cuda.synchronize()
        launches, path = {}, None
        for arm in ("nhwc", "nchw", "convert"):
            n0 = L.launch_count()
            w[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path = path or _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))   # the nhwc call's
        want = w["torch"]().permute(0, 2, 3, 1).reshape(-1).double()
        got, conv = w["dx_h"].double(), w["dx_c"].double()
        rel = {"nhwc_vs_torch": ((got - want).norm() / want.norm()).item(),
               "convert_vs_torch": ((conv - want).norm() / want.norm()).item(),
               "nhwc_vs_convert": ((got - conv).norm() / want.norm()).item(),
               "nhwc_vs_convert_max_over_max": ((got - conv).abs().max() / want.abs().max()).item()}
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm in arms:
                ms[arm].append(timed(w[arm]))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        L.profile_begin()
        for _ in range(a.reps):
            w["nhwc"]()
        torch.cuda.synchronize()
        prof = L.profile_end()
        split = dict(prep_ms=prof["prep_ms"] / a.reps, gemm_ms=prof["gemm_ms"] / a.reps,
                     prep_launches=prof["prep_launches"] / a.reps, gemm_launches=prof["gemm_launches"] / a.reps)
        kt = kernel_times(w["nhwc"], a.reps)
        kt_nchw = kernel_times(w["nchw"], a.reps)
        win_ms = sum(v for k, v in kt.items() if "im2col_rows_kernel" in k)
        win_nchw_ms = sum(v for k, v in kt_nchw.items() if "im2col_rows_kernel" in k)
        copy_ms = sum(v for k, v in kt.items() if "copy_strided_kernel" in k)
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, path=path, ms=med, ms_all=ms,
                    tflops={k: w["flops"] / v / 1e9 for k, v in med.items()}, launches=launches, profile=split,
                    kernel_ms=kt, kernel_ms_nchw=kt_nchw, window_rows_ms=win_ms, window_rows_nchw_ms=win_nchw_ms,
                    filter_copy_ms=copy_ms, normwise=rel)
        res["cases"].append(case)
        lines.append("%s [%s]\n  nhwc %8.3f ms  nchw %8.3f ms  convert %8.3f ms  torch %8.3f ms | nhwc: prep %.3f ms (%g launches; "
                     "window rows %.3f ms, nchw window rows %.3f ms, W'^T copy %.3f ms) + GEMM %.3f ms (%g launches) | "
                     "launches nhwc %d nchw %d convert %d | ||nhwc - convert|| / ||torch|| %.2e, max %.2e (nhwc vs torch %.2e, "
                     "convert vs torch %.2e)"
                     % (name, path, med["nhwc"], med["nchw"], med["convert"], med["torch"], split["prep_ms"], split["prep_launches"],
                        win_ms, win_nchw_ms, copy_ms, split["gemm_ms"], split["gemm_launches"], launches["nhwc"], launches["nchw"],
                        launches["convert"], rel["nhwc_vs_convert"], rel["nhwc_vs_convert_max_over_max"], rel["nhwc_vs_torch"],
                        rel["convert_vs_torch"]))
        print(lines[-1], flush=True)
        del w
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "conv_nhwc_input_grad_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_nhwc_input_grad_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
