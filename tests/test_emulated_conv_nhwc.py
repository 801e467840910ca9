"""CPU-only: the channels-last preparation kernel (laser_b200/csrc/split.cuh: im2col_rows_kernel over an Im2colNhwcSrc, the NHWC
instantiations) on host threads in its three modes and both groups, against the NHWC im2col rows built in numpy -- one row per
output pixel, the window in (kh, kw, c) order, 0 outside the image -- run through the row kernels it stands in for: plain
values exactly; f16x2 words and pieces as f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel.  Words, pieces and
padding columns are compared bit for bit, on the vector path (c % 4 == 0, aligned input) and the scalar one (c = 3, 5, or a
misaligned input).  Also the GPU test file of the entry against the host-emulated library."""
import ctypes

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
F32, TF32, F16X2 = 0, 1, 2


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_nhwc_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_nhwc_rows.argtypes = [ci, ci, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_nhwc_rows.restype = ci
    return L


@pytest.fixture(scope="module")
def rows():
    """the row kernels the channels-last windows replace (tests/emu/conv_emu.cpp)"""
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


# (images, C, H, W, kH, kW, pH, pW, sH, sW)
CASES = {
    "padding": (2, 8, 7, 7, 3, 3, 1, 1, 1, 1),
    "stride2": (2, 4, 9, 9, 3, 3, 0, 0, 2, 2),
    "non_square": (2, 4, 6, 9, 3, 5, 1, 2, 1, 2),        # 3 x 5 kernel, strides (1, 2)
    "one_by_one_stride2": (2, 8, 7, 7, 1, 1, 0, 0, 2, 2),
    "c3": (2, 3, 8, 8, 3, 3, 1, 1, 1, 1),                # the first layer of an RGB network: the scalar path
    "c5": (2, 5, 7, 6, 3, 2, 1, 0, 2, 1),
    "long_rows": (1, 128, 5, 5, 3, 3, 1, 1, 1, 1),       # K = 1152: the CTA per row
    "long_rows_c117": (1, 117, 4, 4, 3, 3, 1, 1, 1, 1),  # K = 1053, scalar
}


def out_hw(case):
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    return 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW


def nhwc_rows(x, case):
    """[n * outH * outW][kH * kW * C] rows of the NHWC images x: output pixel (oh, ow)'s window in (kh, kw, c) order"""
    n, C, H, W, kH, kW, pH, pW, sH, sW = CASES[case]
    oh, ow = out_hw(case)
    xp = np.zeros((n, H + 2 * pH, W + 2 * pW, C), np.float32)
    xp[:, pH:pH + H, pW:pW + W] = x
    hi = (np.arange(oh) * sH)[:, None] + np.arange(kH)[None, :]
    wi = (np.arange(ow) * sW)[:, None] + np.arange(kW)[None, :]
    g = xp[:, hi[:, None, :, None], wi[None, :, None, :], :]       # [n][oh][ow][kH][kW][C]
    return np.ascontiguousarray(g.reshape(n * oh * ow, kH * kW * C))


def setup(case, seed):
    """-> (x [n][H][W][C], rows R, K, the reference rows [R][up(K, 4)]): signed data with images, pixels and channels at their
    own powers of two, so that the rows' scale words differ; one infinity"""
    n, C, H, W = CASES[case][:4]
    rng = np.random.default_rng(seed)
    x = rng.uniform(-3, 3, (n, H, W, C))
    x *= 2.0 ** rng.integers(-8, 9, n)[:, None, None, None] * 2.0 ** rng.integers(-8, 9, (1, H, W, 1)) * \
        2.0 ** rng.integers(-8, 9, C)[None, None, None, :]
    x = x.astype(np.float32)
    x[0, 0, 0, :] = 0.0
    x[n - 1, H // 2, W // 2, C - 1] = np.inf
    oh, ow = out_hw(case)
    K = C * CASES[case][4] * CASES[case][5]
    ref = np.zeros((n * oh * ow, up(K, 4)), np.float32)
    ref[:, :K] = nhwc_rows(x, case)
    return x, n * oh * ow, K, ref


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


def run(emu, mode, group, x, case, dst, lo, hb, lb, ld, w):
    return emu.emu_nhwc_rows(mode, group, p(x), p(geom_of(case)), CASES[case][0], p(dst), p(lo), p(hb), p(lb), ld, p(w), 3)


def expected_vec(case, x):
    return CASES[case][1] % 4 == 0 and x.ctypes.data % 16 == 0


@pytest.mark.parametrize("shift", [False, True], ids=["aligned", "misaligned"])
@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case", list(CASES))
def test_plain_rows_equal_the_windows(emu, case, group, shift):
    x, R, K, ref = setup(case, 1)
    xs = misaligned(x) if shift else x
    ld = up(K, 4)
    dst = np.full((R, ld), 7.0, np.float32)
    assert run(emu, F32, group, xs, case, dst, None, None, None, ld, None) == expected_vec(case, xs)
    same_bits(dst, ref)


@pytest.mark.parametrize("shift", [False, True], ids=["aligned", "misaligned"])
@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case", list(CASES))
def test_tf32_pieces_equal_split_rows_tf32(emu, rows, case, group, shift):
    x, R, K, ref = setup(case, 2)
    xs = misaligned(x) if shift else x
    ld = up(K, 4)
    hi = np.full((R, ld), 7.0, np.float32); lo = np.full((R, ld), 7.0, np.float32)
    assert run(emu, TF32, group, xs, case, hi, lo, None, None, ld, None) == expected_vec(case, xs)
    hr = np.full((R, ld), 9.0, np.float32); lr = np.full((R, ld), 9.0, np.float32)
    rows.emu_tf32_rows(p(ref), R, K, ld, p(hr), p(lr), ld, 3)
    same_bits(hi, hr); same_bits(lo, lr)


@pytest.mark.parametrize("shift", [False, True], ids=["aligned", "misaligned"])
@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case", list(CASES))
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, rows, case, group, shift):
    x, R, K, ref = setup(case, 3)
    xs = misaligned(x) if shift else x
    ldb = up(K, 8)
    w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    assert run(emu, F16X2, group, xs, case, None, None, hb, lb, ldb, w) == expected_vec(case, xs)
    wr = np.full(R, 55, np.uint32); hr = np.full((R, ldb), 5, np.uint16); lr = np.full((R, ldb), 5, np.uint16)
    rows.emu_f16x2_rows(group, p(ref), R, K, ref.shape[1], p(hr), p(lr), ldb, p(wr), 2)
    c4 = up(K, 4)   # the row kernel writes the columns of whole float4 groups; the rest of ld is ours to zero
    same_bits(w, wr)
    same_bits(hb[:, :c4], hr[:, :c4]); same_bits(lb[:, :c4], lr[:, :c4])
    assert np.all(hb[:, K:] == 0) and np.all(lb[:, K:] == 0)
    assert len(np.unique(w)) > 3   # the rows' words differ: a wrong word would show


def test_padding_taps_are_zero(emu):
    """the taps of the first output pixel that fall in the padding are 0 (the image has no zero there)"""
    case = "padding"
    x, R, K, ref = setup(case, 4)
    x = np.abs(x) + 1.0
    dst = np.full((R, up(K, 4)), 7.0, np.float32)
    run(emu, F32, 32, x, case, dst, None, None, None, dst.shape[1], None)
    C, kW = CASES[case][1], CASES[case][5]
    taps = dst[0, :K].reshape(CASES[case][4], kW, C)
    assert np.all(taps[0] == 0) and np.all(taps[:, 0] == 0) and np.all(taps[1:, 1:] != 0)


def test_nhwc_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_nhwc.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_conv_nhwc.py"], [], 2400) >= 60
