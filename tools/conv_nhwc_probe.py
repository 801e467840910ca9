"""Channels-last fused convolution against the NCHW fused entry, the unfused NHWC route and torch, on the tensor-core layers of
tools/conv_probe.py and the reference's conv bench.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  nhwc     laser_b200_conv2d_nhwc_f32_fused_dev (the windows prepared straight from the NHWC images, one GEMM)
  nchw     laser_b200_conv2d_f32_fused_dev on the same data in NCHW
  unfused  the NHWC im2col rows materialised by torch (unfold, then a copy into (kh, kw, c) order), then the fused GEMM
  torch    torch.nn.functional.conv2d on channels_last tensors in fp32, cuDNN TF32 off
The library arms run on PATH_AUTO (no epilogue; nhwc and nchw resolve to the same path).  Where PATH_AUTO takes the exact
kernel, the nhwc entry is also timed on f16x3 and tf32x1.  Also: launches per call, the nhwc call's preparation and GEMM
milliseconds (laser_b200_profile_begin / _end, a separate call) next to the nchw call's, the preparation kernels' bytes moved per
second (images read once, filters read once, prepared rows and scale words written once), whether the nhwc output equals the
fused GEMM over the materialised rows bit for bit, and the card name, power limit and SM clock read in the same run.

python tools/conv_nhwc_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
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

WORKLOADS = [   # name, ishape (n, c, h, w), kshape (c_out, c_in, kH, kW), padding, strides
    ("3x3 56^2 64->64, 32 images", (32, 64, 56, 56), (64, 64, 3, 3), (1, 1), (1, 1)),
    ("3x3 28^2 128->128, 32 images", (32, 128, 28, 28), (128, 128, 3, 3), (1, 1), (1, 1)),
    ("3x3 14^2 256->256, 32 images", (32, 256, 14, 14), (256, 256, 3, 3), (1, 1), (1, 1)),
    ("3x3 stride 2 56^2 64->128, 32 images", (32, 64, 56, 56), (128, 64, 3, 3), (1, 1), (2, 2)),
    ("1x1 56^2 256->64, 32 images", (32, 256, 56, 56), (64, 256, 1, 1), (0, 0), (1, 1)),
    ("reference bench 224^2 3->20 3x3, 16 images", (16, 3, 224, 224), (20, 3, 3, 3), (0, 0), (1, 1)),
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


def rows_of(x_nchw, kshape, padding, strides, rows):
    """the NHWC im2col rows [n * P][ld] in (kh, kw, c) order, zeros past K"""
    n, C = x_nchw.shape[:2]
    kH, kW = kshape[2:]
    cols = torch.nn.functional.unfold(x_nchw, (kH, kW), padding=padding, stride=strides)   # [n][(c, kh, kw)][P]
    P = cols.shape[2]
    rows.view(n, P, -1)[:, :, :C * kH * kW].view(n, P, kH * kW, C).copy_(cols.view(n, C, kH * kW, P).permute(0, 3, 2, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=".", help="directory for conv_nhwc_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi (name, power limit, SM clock, max SM clock)": smi[0] if smi else "unavailable",
           "reps": a.reps, "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "cases": []}
    lines = ["card (name, power limit, SM clock, max SM clock): %s" % (smi[0] if smi else "unavailable"),
             "medians over %d alternating timed calls, CUDA events; default fp32 mode %s; prep / GEMM: the call's preparation and "
             "GEMM kernels (profile_begin/end, separate calls)" % (a.reps, res["f32_mode"]), ""]
    for name, ishape, kshape, padding, strides in WORKLOADS:
        n, C, H, W = ishape
        co, _, kH, kW = kshape
        oshape = L.conv2d_out_shape(ishape, kshape, padding, strides)
        P, K = oshape[2] * oshape[3], C * kH * kW
        ld = -(-K // 4) * 4
        x = fill((n, H, W, C), 1)                                  # NHWC images
        wmat = fill((kH, kW, C, co), 2, -0.1, 0.1).view(K, co)     # kernel_to_hwcc's [kH][kW][C_in][C_out]
        x_nchw = x.permute(0, 3, 1, 2).contiguous()
        x_cl = x.permute(0, 3, 1, 2)                               # channels_last view of the same memory
        k_nchw = wmat.view(kH, kW, C, co).permute(3, 2, 0, 1).contiguous()
        k_cl = k_nchw.to(memory_format=torch.channels_last)
        out_h, out_c, out_u = torch.empty(n * P, co, device="cuda"), torch.empty(oshape, device="cuda"), torch.empty(n * P, co, device="cuda")
        rows = torch.zeros(n * P, ld, device="cuda")

        def unfused():
            rows_of(x_nchw, kshape, padding, strides, rows)
            L.gemm_strided_fused(n * P, co, K, 1.0, rows, ld, 1, wmat, co, 1, 0.0, out_u, co, 1)
        arms = dict(
            nhwc=lambda: L.conv2d_nhwc_fused(out_h, x, ishape, wmat, kshape, padding, strides),
            nchw=lambda: L.conv2d_fused(out_c, x_nchw, ishape, k_nchw, kshape, padding, strides),
            unfused=unfused,
            torch=lambda: torch.nn.functional.conv2d(x_cl, k_cl, padding=padding, stride=strides))
        for _ in range(a.warmup):
            for fn in arms.values():
                fn()
        torch.cuda.synchronize()
        launches, path = {}, {}
        for arm in ("nhwc", "nchw"):
            n0 = L.launch_count()
            arms[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path[arm] = _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))
        if path["nhwc"] == "simt":   # the exact path: the tensor-core modes of the same entry for comparison
            for mode, pid in (("f16x3", L.PATH_F16X3), ("tf32x1", L.PATH_TF32X1)):
                arms["nhwc_" + mode] = (lambda pid: lambda: L.conv2d_nhwc_fused(out_h, x, ishape, wmat, kshape, padding, strides,
                                                                                 path=pid))(pid)
                for _ in range(a.warmup):
                    arms["nhwc_" + mode]()
        # bit-identity: the nhwc output against the fused GEMM over the materialised rows on the path it resolved
        arms["nhwc"]()
        rows_of(x_nchw, kshape, padding, strides, rows)
        ref = torch.empty(n * P, co, device="cuda")
        resolved = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1}[path["nhwc"]]
        L.gemm_strided_fused(n * P, co, K, 1.0, rows, ld, 1, wmat, co, 1, 0.0, ref, co, 1, path=resolved)
        torch.cuda.synchronize()
        identical = bool(torch.equal(out_h.view(torch.int32), ref.view(torch.int32)))
        prof = {}
        for arm in ("nhwc", "nchw"):
            L.profile_begin()
            arms[arm]()
            prof[arm] = L.profile_end()
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm, fn in arms.items():
                ms[arm].append(timed(fn))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        # bytes the preparation kernels need: images (or the 1x1 A in place) read once, filters read once, the prepared pieces
        # and scale words of both operands written once
        piece = {"f16x3": 4, "tf32x3": 8, "tf32x1": 4}.get(path["nhwc"], 0)
        prep_bytes = 4 * (x.numel() + wmat.numel()) + piece * (n * P + co) * K + 4 * (n * P + co)
        gbps = {arm: prep_bytes / (prof[arm]["prep_ms"] * 1e6) if prof[arm]["prep_ms"] > 0 else 0.0 for arm in prof}
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, path=path, ms=med, ms_all=ms,
                    launches=launches, prep_ms={k: v["prep_ms"] for k, v in prof.items()},
                    gemm_ms={k: v["gemm_ms"] for k, v in prof.items()}, prep_launches={k: v["prep_launches"] for k, v in prof.items()},
                    prep_bytes=prep_bytes, prep_gb_per_s=gbps, nhwc_equals_materialised_bitwise=identical,
                    tflops={arm: 2.0 * n * P * co * K / v / 1e9 for arm, v in med.items()})
        res["cases"].append(case)
        extra = "".join("  %s %7.3f ms" % (arm, med[arm]) for arm in med if arm.startswith("nhwc_"))
        lines.append("%-44s nhwc %7.3f ms  nchw %7.3f ms  unfused %7.3f ms  torch(cl) %7.3f ms%s | path %s | launches %d | "
                     "prep nhwc %.3f ms (%.0f GB/s) nchw %.3f ms (%.0f GB/s) | gemm nhwc %.3f nchw %.3f ms | bit-identical %s"
                     % (name, med["nhwc"], med["nchw"], med["unfused"], med["torch"], extra, path["nhwc"], launches["nhwc"],
                        prof["nhwc"]["prep_ms"], gbps["nhwc"], prof["nchw"]["prep_ms"], gbps["nchw"], prof["nhwc"]["gemm_ms"],
                        prof["nchw"]["gemm_ms"], identical))
        print(lines[-1], flush=True)
        del rows, ref
    with open(os.path.join(a.out, "conv_nhwc_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_nhwc_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
