"""Fused convolution filter gradient against today's two-step way and torch, on the convolution layers of tools/conv_probe.py
(32 images each) and the reference's conv bench geometry.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  fused   laser_b200_conv2d_filter_grad_f32_fused_dev: B's tap rows prepared straight from the images, no im2col matrix
  im2col  laser_b200_im2col_f32_dev into a caller-owned workspace, then laser_b200_gemm_strided_batch_reduce_f32_fused_dev over
          the matrices read transposed (the im2col step included in the time)
  torch   torch.nn.grad.conv2d_weight in fp32, cuDNN TF32 off
Both library arms run on PATH_AUTO (they resolve to the same path).  Also: launches per call; the fused call's preparation and
GEMM milliseconds (laser_b200_profile_begin / _end, a run of its own); the per-kernel device time of the preparation from
torch.profiler (another run of its own); the preparation's bytes-needed rate (grad_output read and its pieces written, the
images read once, the tap rows written once, over the preparation time); whether the fused dW equals the im2col arm's bit for
bit; and the card name, power limit and SM clock read in the same run.

python tools/conv_filter_grad_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
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


def up(x, m):
    return -(-x // m) * m


def prep_bytes(mode, n, C, H, W, cout, Kc, P):
    """bytes the preparation of both operands needs to move at the least: grad_output read and its prepared copy written, the
    images read once and the tap rows written once (f16x3: two fp16 pieces and a word per row; tf32x3: two fp32 pieces;
    tf32x1 / exact: the values)"""
    cols = n * P
    per = {"f16x3": 4, "tf32x3": 8}.get(mode, 4)
    rows = {"f16x3": 2 * 2 * up(cols, 8), "tf32x3": 2 * 4 * up(cols, 4)}.get(mode, 4 * up(cols, 4))
    return 4 * n * cout * P + cout * cols * per + 4 * n * C * H * W + Kc * rows


def workload(ishape, kshape, padding, strides):
    n, C, H, W = ishape
    cout = kshape[0]
    _, _, oh, ow = L.conv2d_out_shape(ishape, kshape, padding, strides)
    P, Kc = oh * ow, C * kshape[2] * kshape[3]
    x, dy = fill(n * C * H * W, 1), fill(n * cout * P, 2, -0.1, 0.1)
    cols = torch.empty(n * Kc * P, device="cuda")
    dw_f, dw_i = torch.empty(cout * Kc, device="cuda"), torch.empty(cout * Kc, device="cuda")
    x4, dy4 = x.view(ishape), dy.view(n, cout, oh, ow)

    def fused():
        L.conv2d_filter_grad_fused(dw_f, x, ishape, dy, kshape, padding, strides)

    def im2col():
        L.im2col(cols, x, ishape, kshape, padding, strides, images=n)
        L.gemm_strided_batch_reduce_fused(n, cout, Kc, P, 1.0, dy, P, 1, cout * P, cols, 1, P, Kc * P, 0.0, dw_i, Kc, 1)

    def tch():
        return torch.nn.grad.conv2d_weight(x4, kshape, dy4, stride=strides, padding=padding)

    return dict(fused=fused, im2col=im2col, torch=tch, dw_f=dw_f, dw_i=dw_i, geom=(n, C, H, W, cout, Kc, P),
                flops=2.0 * cout * Kc * n * P, ws_bytes=4 * n * Kc * P)


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
    ap.add_argument("--out", default=".", help="directory for conv_filter_grad_probe.json / .txt")
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
    arms = ("fused", "im2col", "torch")
    for name, ishape, kshape, padding, strides in WORKLOADS:
        w = workload(ishape, kshape, padding, strides)
        for _ in range(a.warmup):
            for arm in arms:
                w[arm]()
        torch.cuda.synchronize()
        launches, path = {}, None
        for arm in ("fused", "im2col"):
            n0 = L.launch_count()
            w[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path = path or _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))   # the fused call's
        identical = bool(torch.equal(w["dw_f"].view(torch.int32), w["dw_i"].view(torch.int32)))
        want = w["torch"]().reshape(-1).double()
        rel = ((w["dw_f"].double() - want).norm() / want.norm()).item()
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
        tap_ms = sum(v for k, v in kt.items() if "im2col_tap_rows_kernel" in k)
        nb = prep_bytes(path, *w["geom"])
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, path=path, ms=med, ms_all=ms,
                    tflops={k: w["flops"] / v / 1e9 for k, v in med.items()}, launches=launches, profile=split,
                    kernel_ms=kt, tap_rows_ms=tap_ms, prep_bytes_needed=nb,
                    prep_gb_per_s=nb / (split["prep_ms"] * 1e6) if split["prep_ms"] > 0 else None,
                    im2col_workspace_bytes=w["ws_bytes"], fused_equals_im2col_bitwise=identical, normwise_vs_torch_fp32=rel)
        res["cases"].append(case)
        lines.append("%s [%s]\n  fused %8.3f ms  im2col+reduce %8.3f ms  torch %8.3f ms | fused: prep %.3f ms (%g launches; tap rows "
                     "%.3f ms) + GEMM %.3f ms (%g launches) | prep needs %.0f MB: %.0f GB/s | launches im2col arm %d | workspace "
                     "saved %.0f MB | fused == im2col bitwise %s | vs torch %.2e"
                     % (name, path, med["fused"], med["im2col"], med["torch"], split["prep_ms"], split["prep_launches"], tap_ms,
                        split["gemm_ms"], split["gemm_launches"], nb / 1e6, case["prep_gb_per_s"] or 0.0, launches["im2col"],
                        w["ws_bytes"] / 1e6, identical, rel))
        print(lines[-1], flush=True)
        del w
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, "conv_filter_grad_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_filter_grad_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
