"""CPU-only: the filter gradient's preparation kernel (laser_b200/csrc/split.cuh: im2col_tap_rows_kernel) on host threads in its
three modes, against the oracle's im2col matrix of each image, concatenated along the pixels (the tap rows of every image end
to end, as the batch-reduced product prepares the matrices read transposed) and run through the row kernels it stands in for:
plain values exactly; f16x2 words and pieces as f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel.  Words,
pieces and padding are compared bit for bit.  Also the GPU test file of the entry against the host-emulated library."""
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
    L = ctypes.CDLL(build_emu("conv_grad_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_tap_rows.argtypes = [ci, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_tap_rows.restype = None
    return L


@pytest.fixture(scope="module")
def rows():
    """the row kernels the tap rows replace (tests/emu/conv_emu.cpp)"""
    L = ctypes.CDLL(build_emu("conv_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_f16x2_rows.argtypes = [ci, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_tf32_rows.argtypes = [vp, i64, i64, i64, vp, vp, i64, ci]
    for n in ("emu_f16x2_rows", "emu_tf32_rows"):
        getattr(L, n).restype = None
    return L


def p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def up(x, m):
    return -(-x // m) * m


# (images, C, H, W, kH, kW, pH, pW, sH, sW); n * P: 98, 60, 108, 48, 245, 36 and 4800 columns -- none but 48 a multiple of 8,
# and 4800 spans two tiles of 4096 with an image boundary inside the first
CASES = {
    "padding": (2, 3, 7, 7, 3, 3, 1, 1, 1, 1),
    "stride2": (3, 4, 9, 8, 3, 3, 1, 1, 2, 2),
    "non_square_3x5": (2, 2, 6, 9, 3, 5, 1, 2, 1, 1),
    "one_by_one_stride2": (3, 5, 7, 7, 1, 1, 0, 0, 2, 2),
    "odd_batch_7x7_outputs": (5, 2, 9, 9, 3, 3, 0, 0, 1, 1),
    "single_image": (1, 4, 6, 6, 3, 3, 1, 1, 1, 1),
    "two_tiles": (3, 2, 40, 40, 3, 3, 1, 1, 1, 1),
}


def setup(case, seed, inf=0.0):
    """images whose channels are scaled by their own powers of two (so the tap rows get different scale words), optionally one
    +-inf pixel -> (images, geometry, images, tap rows K, columns n * P, the concatenated im2col matrix [K][up(n * P, 4)])"""
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    ishape, kshape = (n, C, H, W), (1, C, kH, kW)
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, C, H, W)).astype(np.float32)
    x *= (2.0 ** rng.integers(-12, 13, C)).astype(np.float32)[None, :, None, None]
    x[:, :, 0, 0] = 0.0
    if inf:
        x[n - 1, C - 1, H // 2, W // 2] = inf
    _, _, oh, ow = O.conv2d_out_shape(ishape, kshape, (pH, pW), (sH, sW))
    K, cols = C * kH * kW, n * oh * ow
    ref = np.zeros((K, up(cols, 4)), np.float32)
    ref[:, :cols] = np.concatenate([O.im2col(np.ascontiguousarray(x[b]), ishape, kshape, (pH, pW), (sH, sW)) for b in range(n)],
                                   axis=1)
    geom = np.array([C, H, W, kH, kW, pH, pW, sH, sW], np.int64)
    return x, geom, n, K, cols, ref


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


INF = {"finite": 0.0, "plus_inf": np.inf, "minus_inf": -np.inf}


@pytest.mark.parametrize("inf", list(INF))
@pytest.mark.parametrize("case", list(CASES))
def test_plain_rows_equal_the_concatenated_im2col_matrix(emu, case, inf):
    x, geom, n, K, cols, ref = setup(case, 1, INF[inf])
    ld = up(cols, 4)
    dst = np.full((K, ld), 7.0, np.float32)
    emu.emu_tap_rows(F32, p(x), p(geom), n, p(dst), None, None, None, ld, None, 3)
    same_bits(dst, ref)


@pytest.mark.parametrize("inf", list(INF))
@pytest.mark.parametrize("case", list(CASES))
def test_tf32_pieces_equal_split_rows_tf32(emu, rows, case, inf):
    x, geom, n, K, cols, ref = setup(case, 2, INF[inf])
    ld = up(cols, 4)
    hi = np.full((K, ld), 7.0, np.float32); lo = np.full((K, ld), 7.0, np.float32)
    emu.emu_tap_rows(TF32, p(x), p(geom), n, p(hi), p(lo), None, None, ld, None, 2)
    hr = np.full((K, ld), 9.0, np.float32); lr = np.full((K, ld), 9.0, np.float32)
    rows.emu_tf32_rows(p(ref), K, cols, ld, p(hr), p(lr), ld, 3)
    same_bits(hi, hr); same_bits(lo, lr)


@pytest.mark.parametrize("inf", list(INF))
@pytest.mark.parametrize("case", list(CASES))
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, rows, case, inf):
    x, geom, n, K, cols, ref = setup(case, 3, INF[inf])
    ldb = up(cols, 8)
    w = np.zeros(K, np.uint32); hb = np.full((K, ldb), 9, np.uint16); lb = np.full((K, ldb), 9, np.uint16)
    emu.emu_tap_rows(F16X2, p(x), p(geom), n, None, None, p(hb), p(lb), ldb, p(w), 3)
    wr = np.full(K, 55, np.uint32); hr = np.zeros((K, ldb), np.uint16); lr = np.zeros((K, ldb), np.uint16)
    rows.emu_f16x2_rows(32 if cols <= 1024 else 256, p(ref), K, cols, ref.shape[1], p(hr), p(lr), ldb, p(wr), 2)
    # the row kernel writes whole float4 groups; the columns up to round_up(n * P, 8) are zero in both
    same_bits(w, wr); same_bits(hb, hr); same_bits(lb, lr)
    assert len(set(w.tolist())) > 1, "the channels' scales must give the tap rows different words"


def test_filter_grad_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_filter_grad.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_conv_filter_grad.py"], [], 2400) >= 60
