"""Sanity at the edges of the shape space: very large / very skewed problems, sampled rows vs oracle."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import laser_b200 as L, oracle as O
torch.cuda.set_device(0); L.init()
def check(M, N, K, path=L.PATH_AUTO, nrows=12):
    A = torch.empty(M * K, device="cuda"); B = torch.empty(K * N, device="cuda"); L.fill_uniform_f32(A, M * K, 1, 0, 1); L.fill_uniform_f32(B, K * N, 2, 0, 1)
    C = torch.full((M, N), float("nan"), device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    L.gemm_strided(M, N, K, 1.0, A, K, 1, B, N, 1, 0.0, C, N, 1, path=path); torch.cuda.synchronize()
    e0.record(); L.gemm_strided(M, N, K, 1.0, A, K, 1, B, N, 1, 0.0, C, N, 1, path=path); e1.record(); torch.cuda.synchronize()
    rows = np.unique(np.random.default_rng(0).integers(0, M, nrows))
    a = A.view(M, K)[rows].cpu().numpy(); b = B.view(K, N).cpu().numpy()
    want = np.zeros((len(rows), N), np.float32); O.gemm_strided(len(rows), N, K, 1.0, a, K, 1, b, N, 1, 0.0, want, N, 1)
    err = O.max_relative_error(C[rows].cpu().numpy(), want); ms = e0.elapsed_time(e1)
    print("%8d x %6d x %6d path=%s  %.3f ms  %.1f TFLOP/s  max_rel_err %.2e  nan=%s" % (M, N, K, L.PATH_NAMES[L.last_path()], ms, 2.0 * M * N * K / ms / 1e9, err, bool(torch.isnan(C).any())), flush=True)
    assert err < 1e-4
check(16384, 16384, 16384)
check(262144, 256, 512)
check(256, 262144, 512)
check(128, 128, 1048576)
check(100000, 3, 4096)
check(8200, 8200, 8200)
check(65536, 8192, 64)
check(4096, 4096, 4096)          # split-K of the last partial wave
check(2560, 2304, 8192)          # 360 tiles on 132 SMs: the last wave (96) is more than half full, nothing is split
check(20, 788544, 27)            # the im2col convolution's product as one call (AUTO: tensor cores; exact: few-rows kernel)
check(20, 788544, 27, path=L.PATH_SIMT)
print("ok")
