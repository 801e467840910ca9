"""CPU-only: the channels-last filter gradient's preparation kernel (laser_b200/csrc/split.cuh: im2col_nhwc_tap_rows_kernel) on
host threads in its three modes and in its ABSMAX pass, against the tap rows built in numpy -- the NHWC forward's window rows
transposed, [kH * kW * c][n * outH * outW], 0 outside the image -- run through the row kernels it stands in for: plain values
exactly; f16x2 words and pieces as f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel.  Words, pieces and padding
columns are compared bit for bit, on the vector path (c % 4 == 0, aligned input) and the scalar one (c = 3, 5, or a misaligned
input).  Also the GPU test file of the entry against the host-emulated library."""
import ctypes

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
F32, TF32, F16X2 = 0, 1, 2


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_nhwc_grad_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_nhwc_tap_rows.argtypes = [ci, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_nhwc_tap_rows.restype = ci
    L.emu_nhwc_tap_absmax.argtypes = [vp, vp, i64, i64, vp, ci]
    L.emu_nhwc_tap_absmax.restype = None
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


# (images, C, H, W, kH, kW, pH, pW, sH, sW).  K = kH * kW * C and the columns n * P:
#   c8_padding 72 x 98, stride2 36 x 60, non_square_1x2 60 x 60 (3 x 5 kernel, strides (1, 2)), rgb_c3 27 x 200 (K below one
#   tile of 32 taps), c5 30 x 60, c12_odd 108 x 125, c64 576 x 243 (18 tap tiles), c4_blocks 36 x 1152 (four and a half pixel
#   blocks, an image boundary inside the third), one_by_one_stride2 8 x 48.  Of the column counts 98, 60, 125 and 243 are not
#   multiples of 8, 98, 125 and 243 not of 4, and none is a multiple of the 256-column pixel block.
CASES = {
    "c8_padding": (2, 8, 7, 7, 3, 3, 1, 1, 1, 1),
    "stride2": (3, 4, 9, 8, 3, 3, 1, 1, 2, 2),
    "non_square_1x2": (2, 4, 6, 9, 3, 5, 1, 2, 1, 2),
    "rgb_c3": (2, 3, 10, 10, 3, 3, 1, 1, 1, 1),
    "c5": (3, 5, 7, 6, 3, 2, 1, 0, 2, 1),
    "c12_odd": (5, 12, 7, 7, 3, 3, 0, 0, 1, 1),
    "c64": (3, 64, 9, 9, 3, 3, 1, 1, 1, 1),
    "c4_blocks": (2, 4, 24, 24, 3, 3, 1, 1, 1, 1),
    "one_by_one_stride2": (3, 8, 7, 7, 1, 1, 0, 0, 2, 2),
}


def out_hw(case):
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    return 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW


def tap_rows(x, case):
    """[kH * kW * C][n * outH * outW]: the NHWC forward's window rows of the images x, transposed"""
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    oh, ow = out_hw(case)
    xp = np.zeros((n, H + 2 * pH, W + 2 * pW, C), np.float32)
    xp[:, pH:pH + H, pW:pW + W] = x
    hi = (np.arange(oh) * sH)[:, None] + np.arange(kH)[None, :]
    wi = (np.arange(ow) * sW)[:, None] + np.arange(kW)[None, :]
    g = xp[:, hi[:, None, :, None], wi[None, :, None, :], :]       # [n][oh][ow][kH][kW][C]
    return np.ascontiguousarray(g.reshape(n * oh * ow, kH * kW * C).T)


def setup(case, seed):
    """-> (x [n][H][W][C], K, columns n * P, the reference rows [K][up(n * P, 4)]): signed data with images, pixels and channels
    at their own powers of two, so that the tap rows' scale words differ; one +inf and one -inf pixel value"""
    n, C, H, W = CASES[case][:4]
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, H, W, C))
    x *= 2.0 ** rng.integers(-8, 9, n)[:, None, None, None] * 2.0 ** rng.integers(-8, 9, (1, H, W, 1)) * \
        2.0 ** rng.integers(-8, 9, C)[None, None, None, :]
    x = x.astype(np.float32)
    x[0, 0, 0, :] = 0.0
    x[n - 1, H // 2, W // 2, C - 1] = np.inf
    x[0, H - 1, W // 3, 0] = -np.inf
    oh, ow = out_hw(case)
    K, cols = C * CASES[case][4] * CASES[case][5], n * oh * ow
    ref = np.zeros((K, up(cols, 4)), np.float32)
    ref[:, :cols] = tap_rows(x, case)
    return x, K, cols, ref


def geom_of(case):
    return np.array(CASES[case][1:], np.int64)


def misaligned(x):
    """a copy of x one float past a 16-byte boundary"""
    buf = np.zeros(x.size + 4, np.float32)
    assert buf.ctypes.data % 16 == 0
    v = buf[1:1 + x.size]
    v[:] = x.ravel()
    return v


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def run(emu, mode, x, case, dst, lo, hb, lb, ld, w):
    return emu.emu_nhwc_tap_rows(mode, p(x), p(geom_of(case)), CASES[case][0], p(dst), p(lo), p(hb), p(lb), ld, p(w), 3)


def expected_vec(case, x):
    return CASES[case][1] % 4 == 0 and x.ctypes.data % 16 == 0


SHIFTS = {"aligned": False, "misaligned": True}


@pytest.mark.parametrize("shift", list(SHIFTS))
@pytest.mark.parametrize("case", list(CASES))
def test_plain_rows_equal_the_transposed_windows(emu, case, shift):
    x, K, cols, ref = setup(case, 1)
    xs = misaligned(x) if SHIFTS[shift] else x
    ld = up(cols, 4)
    dst = np.full((K, ld), 7.0, np.float32)
    assert run(emu, F32, xs, case, dst, None, None, None, ld, None) == expected_vec(case, xs)
    same_bits(dst, ref)


@pytest.mark.parametrize("shift", list(SHIFTS))
@pytest.mark.parametrize("case", list(CASES))
def test_tf32_pieces_equal_split_rows_tf32(emu, rows, case, shift):
    x, K, cols, ref = setup(case, 2)
    xs = misaligned(x) if SHIFTS[shift] else x
    ld = up(cols, 4)
    hi = np.full((K, ld), 7.0, np.float32); lo = np.full((K, ld), 7.0, np.float32)
    assert run(emu, TF32, xs, case, hi, lo, None, None, ld, None) == expected_vec(case, xs)
    hr = np.full((K, ld), 9.0, np.float32); lr = np.full((K, ld), 9.0, np.float32)
    rows.emu_tf32_rows(p(ref), K, cols, ld, p(hr), p(lr), ld, 3)
    same_bits(hi, hr); same_bits(lo, lr)


@pytest.mark.parametrize("shift", list(SHIFTS))
@pytest.mark.parametrize("case", list(CASES))
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, rows, case, shift):
    x, K, cols, ref = setup(case, 3)
    xs = misaligned(x) if SHIFTS[shift] else x
    ldb = up(cols, 8)
    w = np.zeros(K, np.uint32); hb = np.full((K, ldb), 9, np.uint16); lb = np.full((K, ldb), 9, np.uint16)
    assert run(emu, F16X2, xs, case, None, None, hb, lb, ldb, w) == expected_vec(case, xs)
    wr = np.full(K, 55, np.uint32); hr = np.zeros((K, ldb), np.uint16); lr = np.zeros((K, ldb), np.uint16)
    rows.emu_f16x2_rows(32 if cols <= 1024 else 256, p(ref), K, cols, ref.shape[1], p(hr), p(lr), ldb, p(wr), 2)
    # the row kernel writes whole float4 groups; the columns up to round_up(n * P, 8) are zero in both
    same_bits(w, wr); same_bits(hb, hr); same_bits(lb, lr)
    assert len(set(w.tolist())) > 3, "the scales must give the tap rows different words"


@pytest.mark.parametrize("case", ["rgb_c3", "c64", "c12_odd"])
def test_absmax_pass_alone_gives_the_row_maxima(emu, case):
    """the ABSMAX launch writes nothing but the words: the largest finite |value| of each tap row (infinities set no scale)"""
    x, K, cols, ref = setup(case, 4)
    w = np.zeros(K, np.uint32)
    emu.emu_nhwc_tap_absmax(p(x), p(geom_of(case)), CASES[case][0], up(cols, 8), p(w), 2)
    a = np.abs(ref)
    want = np.where(np.isfinite(a), a, 0).max(axis=1).astype(np.float32)
    same_bits(w, want.view(np.uint32))


def test_padding_taps_are_zero(emu):
    """the taps of the first output pixel that fall in the padding are 0 (the image has no zero there)"""
    case = "c8_padding"
    x, K, cols, ref = setup(case, 5)
    x = np.abs(np.where(np.isfinite(x), x, 1.0)).astype(np.float32) + 1.0
    dst = np.full((K, up(cols, 4)), 7.0, np.float32)
    run(emu, F32, x, case, dst, None, None, None, dst.shape[1], None)
    C, kH, kW = CASES[case][1], CASES[case][4], CASES[case][5]
    taps = dst[:, 0].reshape(kH, kW, C)
    assert np.all(taps[0] == 0) and np.all(taps[:, 0] == 0) and np.all(taps[1:, 1:] != 0)
    assert np.all(dst[:, cols:] == 0)


def test_nhwc_filter_grad_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_nhwc_filter_grad.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_conv_nhwc_filter_grad.py"], [], 2400) >= 60
