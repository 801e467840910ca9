"""Fused convolution against the im2col + GEMM entry and torch, on the convolution layers of a ResNet-style network and the
reference's conv bench.

Per workload, alternating after warm-up, medians over --reps timed calls (CUDA events around each call):
  fused   laser_b200_conv2d_f32_fused_dev (im2col folded into the preparation of B, one GEMM launch for the images)
  im2col  laser_b200_conv2d_im2col_f32_dev with a workspace for every image (im2col kernel, then the GEMM per image)
  torch   torch.nn.functional.conv2d in fp32, cuDNN TF32 off
Both library arms run on PATH_AUTO (no epilogue: they resolve to the same path).  Also: launches per call, the fused call's
preparation and GEMM milliseconds (laser_b200_profile_begin / _end, a separate call), the preparation kernels' bytes moved per
second (images read once, prepared rows written once, filters), whether the fused output equals the batched fused product over
the materialised im2col matrix bit for bit, and the card name, power limit and SM clock read in the same run.

python tools/conv_probe.py [--reps 20] [--warmup 3] [--out DIR]"""
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


def materialised(x, k, ishape, kshape, padding, strides, out):
    """the batched fused product over the im2col matrices, transposed into the rows the preparation kernel writes (for a
    1 x 1 kernel with unit strides and no padding: over the images as they are)"""
    n, C, H, W = ishape
    M, K = kshape[0], C * kshape[2] * kshape[3]
    N = out.numel() // (n * M)
    if kshape[2:] == (1, 1) and padding == (0, 0) and strides == (1, 1):
        B, rsB, csB, bsB = x, N, 1, C * H * W
    else:
        ld = -(-K // 4) * 4
        cols = torch.nn.functional.unfold(x.view(ishape), kshape[2:], padding=padding, stride=strides)   # [n][K][N], (c, kh, kw)
        rows = torch.zeros(n, N, ld, device="cuda")
        rows[:, :, :K] = cols.transpose(1, 2)
        B, rsB, csB, bsB = rows, 1, ld, N * ld
    L.gemm_strided_batched_fused(n, M, N, K, 1.0, k, K, 1, 0, B, rsB, csB, bsB, 0.0, out, N, 1, M * N)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=".", help="directory for conv_probe.json / .txt")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi (name, power limit, SM clock, max SM clock)": smi[0] if smi else "unavailable",
           "reps": a.reps, "f32_mode": _capi.PATH_NAMES[L.get_f32_mode()], "cases": []}
    lines = ["card (name, power limit, SM clock, max SM clock): %s" % (smi[0] if smi else "unavailable"),
             "medians over %d alternating timed calls, CUDA events; default fp32 mode %s; prep / GEMM: the fused call's "
             "preparation and GEMM kernels (profile_begin/end, separate calls)" % (a.reps, res["f32_mode"]), ""]
    for name, ishape, kshape, padding, strides in WORKLOADS:
        n = ishape[0]
        oshape = L.conv2d_out_shape(ishape, kshape, padding, strides)
        x, k = fill(n * ishape[1] * ishape[2] * ishape[3], 1), fill(kshape[0] * kshape[1] * kshape[2] * kshape[3], 2, -0.1, 0.1)
        out_f, out_i = torch.empty(oshape, device="cuda"), torch.empty(oshape, device="cuda")
        ws = torch.empty(n * max(1, L.im2col_workspace_size(ishape, kshape, padding, strides)), device="cuda")
        xt, kt = x.view(ishape), k.view(kshape)
        arms = dict(
            fused=lambda: L.conv2d_fused(out_f, x, ishape, k, kshape, padding, strides),
            im2col=lambda: L.conv2d_im2col(out_i, x, ishape, k, kshape, padding, strides, workspace=ws, workspace_images=n),
            torch=lambda: torch.nn.functional.conv2d(xt, kt, padding=padding, stride=strides))
        for _ in range(a.warmup):
            for fn in arms.values():
                fn()
        torch.cuda.synchronize()
        launches, path = {}, {}
        for arm in ("fused", "im2col"):
            n0 = L.launch_count()
            arms[arm]()
            torch.cuda.synchronize()
            launches[arm] = L.launch_count() - n0
            path[arm] = _capi.PATH_NAMES.get(L.last_path(), str(L.last_path()))
        ref = torch.empty(oshape, device="cuda")
        materialised(x, k, ishape, kshape, padding, strides, ref)
        torch.cuda.synchronize()
        identical = bool(torch.equal(out_f.view(torch.int32), ref.view(torch.int32)))
        L.profile_begin()
        arms["fused"]()
        prof = L.profile_end()
        ms = {arm: [] for arm in arms}
        for _ in range(a.reps):
            for arm, fn in arms.items():
                ms[arm].append(timed(fn))
        med = {arm: statistics.median(v) for arm, v in ms.items()}
        M, K, N = kshape[0], ishape[1] * kshape[2] * kshape[3], oshape[2] * oshape[3]
        # bytes the preparation kernels need: images (or the 1x1 B in place) read once, filters read once, the prepared pieces
        # and scale words of both operands written once
        piece = {"f16x3": 4, "tf32x3": 8, "tf32x1": 4}.get(path["fused"], 0)
        prep_bytes = 4 * (x.numel() + k.numel()) + piece * (n * N + M) * K + 4 * (n * N + M)
        gbps = prep_bytes / (prof["prep_ms"] * 1e6) if prof["prep_ms"] > 0 else 0.0
        case = dict(name=name, ishape=ishape, kshape=kshape, padding=padding, strides=strides, path=path, ms=med, ms_all=ms,
                    launches=launches, prep_ms=prof["prep_ms"], gemm_ms=prof["gemm_ms"], prep_launches=prof["prep_launches"],
                    gemm_launches=prof["gemm_launches"], prep_bytes=prep_bytes, prep_gb_per_s=gbps,
                    fused_equals_materialised_bitwise=identical, tflops={arm: 2.0 * n * M * N * K / v / 1e9 for arm, v in med.items()})
        res["cases"].append(case)
        lines.append("%-44s fused %7.3f ms  im2col %7.3f ms  torch %7.3f ms | path %s | launches fused %d im2col %d | "
                     "prep %.3f ms (%d launches, %.0f GB/s) gemm %.3f ms | bit-identical %s"
                     % (name, med["fused"], med["im2col"], med["torch"], path["fused"], launches["fused"], launches["im2col"],
                        prof["prep_ms"], prof["prep_launches"], gbps, prof["gemm_ms"], identical))
        print(lines[-1], flush=True)
        del ws
    with open(os.path.join(a.out, "conv_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(a.out, "conv_probe.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
