"""Timing of the steps either side of the GEMM on one H100 (HBM roofline), at the reference's own
bench shapes: transpose 4000x2000 f32 (benchmarks/transpose/transpose_bench.nim:54-55; the
reference's best CPU variant: 9.2 ms = 0.78 GMEMOP/s), NCHW<->NHWC, im2col and conv2d_im2col on
16x3x224x224 with 20 3x3 filters (benchmarks/convolution/conv2d_bench.nim:52-62).
Usage: python tools/layers_bench.py  (prints one JSON line per kernel)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import laser_b200 as L  # noqa: E402

PEAK = 6573.2
try:
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
        PEAK = json.load(f)["hbm_gbs"]
except Exception:
    pass


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def report(name, ms, nbytes, **extra):
    gbs = nbytes / ms / 1e6
    print(json.dumps(dict(kernel=name, ms=round(ms, 4), algorithmic_bytes=nbytes, gbs=round(gbs, 1),
                          frac_of_hbm_peak=round(gbs / PEAK, 3), **extra)), flush=True)


def main():
    L.init()
    for NR, NC in ((4000, 2000), (8192, 8192), (16384, 16384)):
        src = torch.rand(NR * NC, device="cuda"); dst = torch.empty_like(src)
        ms = timeit(lambda: L.transpose2D_copy(dst, src, NR, NC))
        assert torch.equal(dst.view(NC, NR), src.view(NR, NC).t())
        report("transpose2D_copy f32 %dx%d" % (NR, NC), ms, 2 * 4 * NR * NC)
    N, C, H, W = 64, 64, 112, 112
    x = torch.rand(N * C * H * W, device="cuda"); y = torch.empty_like(x)
    ms = timeit(lambda: L.nchw2nhwc(y, x, N, C, H, W))
    assert torch.equal(y.view(N, H, W, C), x.view(N, C, H, W).permute(0, 2, 3, 1))
    report("nchw2nhwc f32 %dx%dx%dx%d" % (N, C, H, W), ms, 2 * 4 * x.numel())
    ms = timeit(lambda: L.nhwc2nchw(x, y, N, C, H, W))
    report("nhwc2nchw f32 %dx%dx%dx%d" % (N, C, H, W), ms, 2 * 4 * x.numel())

    ish, ksh, pad, st = (16, 3, 224, 224), (20, 3, 3, 3), (0, 0), (1, 1)
    osh = L.conv2d_out_shape(ish, ksh, pad, st)
    per = L.im2col_workspace_size(ish, ksh, pad, st)
    inp = torch.rand(ish, device="cuda"); ker = torch.rand(ksh, device="cuda")
    ws = torch.empty(ish[0] * per, device="cuda"); out = torch.empty(osh, device="cuda")
    ms = timeit(lambda: L.im2col(ws, inp, ish, ksh, pad, st, images=ish[0]))
    report("im2col 16x3x224x224 k3", ms, 4 * (ish[0] * per + inp.numel()))
    flops = 2 * ish[0] * ksh[0] * ksh[1] * 9 * osh[2] * osh[3]      # conv2d_common.nim:47-78
    # AUTO sends each image's 20 x 49284 x 27 product to the tensor cores (one launch sequence per image);
    # PATH_SIMT runs all images of a workspace chunk as ONE launch of the exact kernel -- for so small an M
    # and K the latter may well win: measure both before choosing a dispatch rule for convolutions
    for path, pname in ((L.PATH_AUTO, "auto"), (L.PATH_SIMT, "exact")):
        for wi in (1, 16):
            ms = timeit(lambda: L.conv2d_im2col(out, inp, ish, ker, ksh, pad, st, workspace=ws, workspace_images=wi, path=path))
            report("conv2d_im2col 16x3x224x224 -> 20 k3, path=%s, workspace_images=%d" % (pname, wi), ms,
                   4 * (inp.numel() + ker.numel() + out.numel()), gflops=round(flops / ms / 1e6, 1),
                   reference_cpu_note="reference bench prints GFLOP/s for the same shape (conv2d_bench.nim)")
    cout = out.clone()
    # forEach o in output, x in a, y in b, z in c: o = x + y - sin z   (iter_bench_prod.nim:86-107, float64)
    for name, shape, transposed in (("contiguous", (1000, 1000), False), ("transposed inputs", (100, 10000), True),
                                    ("contiguous 8192^2", (8192, 8192), False)):
        hx = np.random.rand(*shape)
        x = L.toTensor(hx, "f64"); out = L.newTensor(list(shape), "f64")
        if transposed:
            y = L.toTensor(np.random.rand(shape[1], shape[0]), "f64").transpose(); z = L.toTensor(np.random.rand(shape[1], shape[0]), "f64").transpose()
        else:
            y = L.toTensor(np.random.rand(*shape), "f64"); z = L.toTensor(np.random.rand(*shape), "f64")
        ms = timeit(lambda: L.forEach("bench", out, x, y, z))
        report("forEach o = x + y - sin z, f64 %s %s" % (shape, name), ms, 4 * 8 * shape[0] * shape[1])
    ref = torch.nn.functional.conv2d(inp, ker)
    print(json.dumps(dict(check="conv2d vs torch", max_rel=float(((cout - ref).abs().max() / ref.abs().max()).item()))))


if __name__ == "__main__":
    main()
