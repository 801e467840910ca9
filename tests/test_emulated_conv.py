"""CPU-only: the fused convolution's preparation kernel (laser_b200/csrc/split.cuh: im2col_rows_kernel) on host threads in its
three modes, against the materialised, transposed im2col matrix of the oracle run through the row kernels it stands in for
(plain values exactly; f16x2 words and pieces as f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel); and the GPU
test file of the fused convolution against the host-emulated library."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
F32, TF32, F16X2 = 0, 1, 2


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_im2col_rows.argtypes = [ci, ci, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_f16x2_rows.argtypes = [ci, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_tf32_rows.argtypes = [vp, i64, i64, i64, vp, vp, i64, ci]
    for n in ("emu_im2col_rows", "emu_f16x2_rows", "emu_tf32_rows"):
        getattr(L, n).restype = None
    return L


def p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def up(x, m):
    return -(-x // m) * m


# (images, C, H, W, kH, kW, pH, pW, sH, sW)
CASES = {
    "padding_K27": (2, 3, 7, 7, 3, 3, 1, 1, 1, 1),
    "stride2_K36": (3, 4, 9, 8, 3, 3, 1, 1, 2, 2),
    "non_square_K20": (2, 2, 6, 9, 2, 5, 1, 2, 1, 2),
    "non_square_K21_no_padding": (1, 7, 5, 6, 1, 3, 0, 0, 1, 1),
    "one_by_one_stride2_K5": (2, 5, 7, 7, 1, 1, 0, 0, 2, 2),
    "one_by_one_padded_K6": (1, 6, 4, 5, 1, 1, 1, 1, 1, 1),
    "long_rows_K1053": (1, 117, 5, 5, 3, 3, 1, 1, 1, 1),
}


def setup(case, seed):
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    ishape, kshape = (n, C, H, W), (1, C, kH, kW)
    x = np.random.default_rng(seed).uniform(-3, 3, (n, C, H, W)).astype(np.float32)
    x[:, :, 0, 0] = 0.0
    _, _, oh, ow = O.conv2d_out_shape(ishape, kshape, (pH, pW), (sH, sW))
    K, N = C * kH * kW, oh * ow
    # the im2col matrix [K][N] of each image, transposed and stacked: rows [n * N][K], 16-byte aligned (ld multiple of 4)
    ref = np.zeros((n * N, up(K, 4)), np.float32)
    for b in range(n):
        ref[b * N:(b + 1) * N, :K] = O.im2col(np.ascontiguousarray(x[b]), ishape, kshape, (pH, pW), (sH, sW)).T
    geom = np.array([C, H, W, kH, kW, pH, pW, sH, sW], np.int64)
    return x, geom, n, n * N, K, ref


def group_of(K):
    return 32 if up(K, 8) <= 1024 else 256


@pytest.mark.parametrize("case", list(CASES))
def test_plain_rows_equal_the_im2col_matrix(emu, case):
    x, geom, n, R, K, ref = setup(case, 1)
    ld = up(K, 4)
    dst = np.full((R, ld), 7.0, np.float32)
    emu.emu_im2col_rows(F32, group_of(K), p(x), p(geom), n, p(dst), None, None, None, ld, None, 3)
    assert np.array_equal(dst[:, :K], ref[:, :K])
    assert np.all(dst[:, K:] == 0)


@pytest.mark.parametrize("case", list(CASES))
def test_tf32_pieces_equal_split_rows_tf32(emu, case):
    x, geom, n, R, K, ref = setup(case, 2)
    ld = up(K, 4)
    hi = np.full((R, ld), 7.0, np.float32); lo = np.full((R, ld), 7.0, np.float32)
    emu.emu_im2col_rows(TF32, group_of(K), p(x), p(geom), n, p(hi), p(lo), None, None, ld, None, 2)
    hr = np.full((R, ld), 9.0, np.float32); lr = np.full((R, ld), 9.0, np.float32)
    emu.emu_tf32_rows(p(ref), R, K, ld, p(hr), p(lr), ld, 3)
    assert np.array_equal(hi.view(np.uint32), hr.view(np.uint32)) and np.array_equal(lo.view(np.uint32), lr.view(np.uint32))
    assert np.all(hi[:, K:] == 0) and np.all(lo[:, K:] == 0)


@pytest.mark.parametrize("case", list(CASES))
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, case):
    x, geom, n, R, K, ref = setup(case, 3)
    ldb, group = up(K, 8), group_of(K)
    w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    emu.emu_im2col_rows(F16X2, group, p(x), p(geom), n, None, None, p(hb), p(lb), ldb, p(w), 3)
    wr = np.full(R, 55, np.uint32); hr = np.full((R, ldb), 5, np.uint16); lr = np.full((R, ldb), 5, np.uint16)
    emu.emu_f16x2_rows(group, p(ref), R, K, up(K, 4), p(hr), p(lr), ldb, p(wr), 2)
    c4 = up(K, 4)   # the row kernel writes the columns of whole float4 groups; the rest of ld is ours to zero
    assert np.array_equal(w, wr)
    assert np.array_equal(hb[:, :c4], hr[:, :c4]) and np.array_equal(lb[:, :c4], lr[:, :c4])
    assert np.all(hb[:, K:] == 0) and np.all(lb[:, K:] == 0)


def test_fused_conv_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_fused.py (backend-neutral) on the CPU build of the whole library, minus the sizes skipped there"""
    assert _run_gpu_files(["test_gpu_conv_fused.py"], [], 2400) >= 40
