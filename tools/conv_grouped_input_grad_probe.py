"""Grouped convolution input gradient (laser_b200_conv2d_grouped_input_grad_f32_fused_dev) on the depthwise and grouped layers of
MobileNet, ConvNeXt and ResNeXt (the nine workloads of tools/conv_grouped_probe.py), NCHW, 32 images, fp32, alpha = 1, beta = 0.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  auto      PATH_AUTO (the path it resolved to is recorded)
  simt      PATH_SIMT: the direct CUDA-core kernel over the transposed geometry
  f16x3     PATH_F16X3 and tf32x1 PATH_TF32X1: one filter copy and one batched tensor-core GEMM, the rotated filters repeating
            every G problems
  loop      G calls of laser_b200_conv2d_input_grad_f32_fused_dev (PATH_AUTO) over per-group copies made once before timing
  torch     torch.nn.grad.conv2d_input(groups=G), fp32, cuDNN TF32 off; torch_tf32 with cuDNN TF32 on
Also: launches per call of each library arm, and for the direct kernel the bytes it must move (dY read once, filters read
once, dX written once) and the FMAs it issues (every input pixel times K' = c_out / G * kH * kW taps of the zero-dilated
window, holes included; `useful_fmas` are the forward's count), as GB/s and TFLOP/s against the H100 SXM data-sheet bounds
(3.35 TB/s HBM3, 67 TFLOP/s FP32), with the bound that limits the workload; the card name, power limit and SM clock read in the
same run.

python tools/conv_grouped_input_grad_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
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

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12   # H100 SXM data sheet (700 W)
WORKLOADS = [   # name, ishape (n, c, h, w), kshape (c_out, c_in / G, kH, kW), padding, strides, groups
    ("depthwise 3x3 56^2 144 ch", (32, 144, 56, 56), (144, 1, 3, 3), (1, 1), (1, 1), 144),
    ("depthwise 3x3 s2 112^2->56^2 96 ch", (32, 96, 112, 112), (96, 1, 3, 3), (1, 1), (2, 2), 96),
    ("depthwise 7x7 56^2 96 ch (ConvNeXt)", (32, 96, 56, 56), (96, 1, 7, 7), (3, 3), (1, 1), 96),
    ("depthwise 3x3 14^2 576 ch", (32, 576, 14, 14), (576, 1, 3, 3), (1, 1), (1, 1), 576),
    ("depthwise x2 3x3 28^2 32->64", (32, 32, 28, 28), (64, 1, 3, 3), (1, 1), (1, 1), 32),
    ("ResNeXt 3x3 56^2 128->128 G=32", (32, 128, 56, 56), (128, 4, 3, 3), (1, 1), (1, 1), 32),
    ("ResNeXt 3x3 7^2 1024->1024 G=32", (32, 1024, 7, 7), (1024, 32, 3, 3), (1, 1), (1, 1), 32),
    ("3x3 28^2 512->512 G=4", (32, 512, 28, 28), (512, 128, 3, 3), (1, 1), (1, 1), 4),
    ("3x3 14^2 1024->1024 G=8", (32, 1024, 14, 14), (1024, 128, 3, 3), (1, 1), (1, 1), 8),
]


def fill(shape, seed, lo=-1.0, hi=1.0):
    n = 1
    for d in shape:
        n *= d
    t = torch.empty(n, device="cuda")
    L.fill_uniform_f32(t, n, seed, lo, hi)
    return t.view(shape)


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
    ap.add_argument("--out", default=".", help="directory for conv_grouped_input_grad_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi (name, power limit, SM clock, max SM clock)": smi[0] if smi else "unavailable",
           "reps": a.reps, "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "bounds": {"hbm_bytes_per_s": HBM_BPS, "fp32_flops": FP32_FLOPS},
           "cases": []}
    lines = ["card (name, power limit, SM clock, max SM clock): %s" % (smi[0] if smi else "unavailable"),
             "medians over %d alternating timed calls, CUDA events, ms; direct kernel (simt) against the data-sheet bounds "
             "3.35 TB/s, 67 TFLOP/s" % a.reps, ""]
    for name, ishape, kshape, padding, strides, groups in WORKLOADS:
        n, C, H, W = ishape
        co, cg, kH, kW = kshape
        mg = co // groups
        oshape = L.conv2d_out_shape((n, cg, H, W), (mg, cg, kH, kW), padding, strides)
        oshape = (n, co, oshape[2], oshape[3])
        dy = fill(oshape, 1)
        k = fill(kshape, 2, -0.1, 0.1)
        dx = torch.empty(ishape, device="cuda")
        dys = [dy[:, g * mg:(g + 1) * mg].contiguous() for g in range(groups)]
        ks = [k[g * mg:(g + 1) * mg].contiguous() for g in range(groups)]
        dxs = [torch.empty((n, cg, H, W), device="cuda") for _ in range(groups)]

        def lib(path):
            return lambda: L.conv2d_grouped_input_grad_fused(dx, ishape, dy, k, kshape, padding, strides, groups, path=path)

        def loop():
            for g in range(groups):
                L.conv2d_input_grad_fused(dxs[g], (n, cg, H, W), dys[g], ks[g], (mg, cg, kH, kW), padding, strides)

        def conv_torch(tf32):
            def fn():
                torch.backends.cudnn.allow_tf32 = tf32
                torch.nn.grad.conv2d_input(ishape, k, dy, stride=strides, padding=padding, groups=groups)
            return fn
        arms = dict(auto=lib(L.PATH_AUTO), simt=lib(L.PATH_SIMT), f16x3=lib(L.PATH_F16X3), tf32x1=lib(L.PATH_TF32X1), loop=loop,
                    torch=conv_torch(False), torch_tf32=conv_torch(True))
        for _ in range(a.warmup):
            for fn in arms.values():
                fn()
        torch.cuda.synchronize()
        launches, path = {}, {}
        for arm in ("auto", "simt", "f16x3", "tf32x1", "loop"):
            n0 = L.launch_count()
            arms[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path[arm] = _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm, fn in arms.items():
                ms[arm].append(timed(fn))
        torch.backends.cudnn.allow_tf32 = False
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        P = oshape[2] * oshape[3]
        fma = n * C * H * W * mg * kH * kW          # issued: every input pixel's zero-dilated window
        useful = n * co * P * cg * kH * kW
        bytes_ = 4 * (dy.numel() + k.numel() + dx.numel())
        t_mem, t_flop = bytes_ / HBM_BPS, 2.0 * fma / FP32_FLOPS
        s = med["simt"] * 1e-3
        direct = dict(bytes=bytes_, fmas=fma, useful_fmas=useful, gb_per_s=bytes_ / s / 1e9, tflops=2.0 * fma / s / 1e12,
                      bound="bandwidth" if t_mem >= t_flop else "fp32 compute", bound_ms=1e3 * max(t_mem, t_flop),
                      share_of_bound=max(t_mem, t_flop) / s)
        tc_best = min(med["f16x3"], med["tf32x1"]) if res["f32_mode"] == "tf32x1" else med["f16x3"]
        fastest_lib = "simt" if med["simt"] <= tc_best else res["f32_mode"]
        auto_took = "simt" if path["auto"] == "simt" else path["auto"]
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, groups=groups, path=path, ms=med,
                    ms_all=ms, launches=launches, direct=direct, auto_took_faster=(auto_took == fastest_lib),
                    auto_over_faster=med["auto"] / min(med["simt"], tc_best), auto_over_loop=med["auto"] / med["loop"],
                    auto_over_torch=med["auto"] / med["torch"])
        res["cases"].append(case)
        lines.append("%-36s auto(%s) %7.3f  simt %7.3f  f16x3 %7.3f  tf32x1 %7.3f  loop(%d calls) %8.3f  torch %7.3f  torch_tf32 %7.3f"
                     " | launches auto %d f16x3 %d loop %d | direct %.0f GB/s %.2f TFLOP/s, %s-bound (%.3f ms, %.0f %% of it) | auto "
                     "took the faster: %s" % (name, path["auto"], med["auto"], med["simt"], med["f16x3"], med["tf32x1"], groups,
                                         med["loop"], med["torch"], med["torch_tf32"], launches["auto"], launches["f16x3"],
                                         launches["loop"],
                                         direct["gb_per_s"], direct["tflops"], direct["bound"], direct["bound_ms"],
                                         100 * direct["share_of_bound"], case["auto_took_faster"]))
        print(lines[-1], flush=True)
        del dys, ks, dxs
    with open(os.path.join(a.out, "conv_grouped_input_grad_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_grouped_input_grad_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
