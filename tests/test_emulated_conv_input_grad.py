"""CPU-only: the input gradient's preparation kernel (laser_b200/csrc/split.cuh: im2col_rows_kernel over an Im2colGradSrc, the
DIL and HAS_OP instantiations) on host threads in its three modes and both groups, against the transposed windows built in
numpy -- grad_output zero-dilated by the strides, padded by kH - 1 - pH, holes 0 after the op -- run through the row kernels it
stands in for: plain values exactly; f16x2 words and pieces as f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel.
Words, pieces and padding are compared bit for bit.  Also the GPU test file of the entry against the host-emulated library."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
F32, TF32, F16X2 = 0, 1, 2
OPS = {"none": 0, "relu": 1, "sigmoid": 3, "relu_grad": 4, "tanh_grad": 5, "sigmoid_grad": 6}


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_input_grad_emu", ["split.cuh", "f16_scale.cuh", "layers.cuh"]))
    L.emu_tconv_rows.argtypes = [ci, ci, ci, ci, vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_operand_op.argtypes = [ci, vp, vp, i64, vp]
    for n in ("emu_tconv_rows", "emu_operand_op"):
        getattr(L, n).restype = None
    return L


@pytest.fixture(scope="module")
def rows():
    """the row kernels the transposed windows replace (tests/emu/conv_emu.cpp)"""
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


# forward geometries (images, C, H, W, c_out, kH, kW, pH, pW, sH, sW)
CASES = {
    "padding": (2, 3, 7, 7, 4, 3, 3, 1, 1, 1, 1),
    "stride2_tail_rows": (2, 3, 8, 8, 4, 3, 3, 0, 0, 2, 2),        # (8 - 3) mod 2: row and column 7 get no window
    "stride3_negative_h": (2, 2, 11, 10, 3, 5, 5, 0, 1, 3, 3),     # h = ih - 4 + kh' down to -4: -3 is a "multiple" of 3
    "non_square_3x5": (2, 2, 6, 9, 3, 3, 5, 1, 2, 1, 1),
    "one_by_one_stride2": (2, 5, 7, 7, 3, 1, 1, 0, 0, 2, 2),
    "one_by_one_padded": (1, 3, 4, 5, 6, 1, 1, 1, 1, 1, 1),        # p' = -1
    "pad_past_kernel": (1, 2, 6, 6, 3, 2, 2, 2, 3, 1, 2),          # pH >= kH: p' < 0 on both axes
    "long_rows": (1, 4, 5, 5, 117, 3, 3, 1, 1, 1, 1),              # K' = 1053: the CTA per row
}


def transposed_rows(z, case):
    """[n * H * W][K'] rows: input pixel (ih, iw)'s window over z (dY, op applied) dilated by the strides, padded by kH - 1 - pH"""
    n, C, H, W, co, kH, kW, pH, pW, sH, sW = CASES[case]
    oh, ow = z.shape[2:]

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, pH, sH, oh)
    wq, vw = axis(W, kW, pW, sW, ow)
    g = z[:, :, hq[:, :, None, None], wq[None, None, :, :]]                          # [n][co][H][kH][W][kW]
    g = np.where((vh[:, :, None, None] & vw[None, None, :, :])[None, None], g, np.float32(0))
    return np.ascontiguousarray(g.transpose(0, 2, 4, 1, 3, 5).reshape(n * H * W, co * kH * kW)).astype(np.float32)


def setup(emu, case, seed, op, inf=0.0):
    """-> (dY, aux, geometry, images, rows R, K', the reference rows [R][up(K', 4)] with the op applied and holes 0)"""
    n, C, H, W, co, kH, kW, pH, pW, sH, sW = CASES[case]
    oshape = tuple(O.conv2d_out_shape((n, C, H, W), (co, C, kH, kW), (pH, pW), (sH, sW)))
    rng = np.random.default_rng(seed)
    dy = rng.uniform(-3, 3, oshape).astype(np.float32)
    dy *= (2.0 ** rng.integers(-12, 13, co)).astype(np.float32)[None, :, None, None]   # channels at their own scales
    dy[:, :, 0, 0] = 0.0
    if inf:
        dy[n - 1, co - 1, oshape[2] // 2, oshape[3] // 2] = inf
    aux = rng.uniform(-1, 1, oshape).astype(np.float32) if OPS[op] >= 4 else None
    z = np.empty_like(dy)
    emu.emu_operand_op(OPS[op], p(dy), p(aux), dy.size, p(z))
    K = co * kH * kW
    ref = np.zeros((n * H * W, up(K, 4)), np.float32)
    ref[:, :K] = transposed_rows(z, case)
    geom = np.array([C, H, W, kH, kW, pH, pW, sH, sW, co], np.int64)
    return dy, aux, geom, n, n * H * W, K, ref


def group_of(K):
    return 32 if up(K, 8) <= 1024 else 256


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def run(emu, mode, case, op, dy, aux, geom, n, dst, lo, hb, lb, ld, w, K):
    sH, sW = CASES[case][9:11]
    emu.emu_tconv_rows(mode, group_of(K), 1 if (sH, sW) != (1, 1) or op == "none" else 0, OPS[op], p(dy), p(aux), p(geom), n,
                       p(dst), p(lo), p(hb), p(lb), ld, p(w), 3)


VARIANTS = [("none", 0.0), ("relu_grad", 0.0), ("sigmoid", 0.0), ("tanh_grad", np.inf), ("none", -np.inf), ("relu", 0.0),
            ("sigmoid_grad", 0.0)]


@pytest.mark.parametrize("op,inf", VARIANTS)
@pytest.mark.parametrize("case", list(CASES))
def test_plain_rows_equal_the_transposed_windows(emu, case, op, inf):
    dy, aux, geom, n, R, K, ref = setup(emu, case, 1, op, inf)
    ld = up(K, 4)
    dst = np.full((R, ld), 7.0, np.float32)
    run(emu, F32, case, op, dy, aux, geom, n, dst, None, None, None, ld, None, K)
    same_bits(dst, ref)


@pytest.mark.parametrize("op,inf", VARIANTS)
@pytest.mark.parametrize("case", list(CASES))
def test_tf32_pieces_equal_split_rows_tf32(emu, rows, case, op, inf):
    dy, aux, geom, n, R, K, ref = setup(emu, case, 2, op, inf)
    ld = up(K, 4)
    hi = np.full((R, ld), 7.0, np.float32); lo = np.full((R, ld), 7.0, np.float32)
    run(emu, TF32, case, op, dy, aux, geom, n, hi, lo, None, None, ld, None, K)
    hr = np.full((R, ld), 9.0, np.float32); lr = np.full((R, ld), 9.0, np.float32)
    rows.emu_tf32_rows(p(ref), R, K, ld, p(hr), p(lr), ld, 3)
    same_bits(hi, hr); same_bits(lo, lr)


@pytest.mark.parametrize("op,inf", VARIANTS)
@pytest.mark.parametrize("case", list(CASES))
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, rows, case, op, inf):
    dy, aux, geom, n, R, K, ref = setup(emu, case, 3, op, inf)
    ldb, group = up(K, 8), group_of(K)
    w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    run(emu, F16X2, case, op, dy, aux, geom, n, None, None, hb, lb, ldb, w, K)
    wr = np.full(R, 55, np.uint32); hr = np.full((R, ldb), 5, np.uint16); lr = np.full((R, ldb), 5, np.uint16)
    rows.emu_f16x2_rows(group, p(ref), R, K, ref.shape[1], p(hr), p(lr), ldb, p(wr), 2)
    c4 = up(K, 4)   # the row kernel writes the columns of whole float4 groups; the rest of ld is ours to zero
    same_bits(w, wr)
    same_bits(hb[:, :c4], hr[:, :c4]); same_bits(lb[:, :c4], lr[:, :c4])
    assert np.all(hb[:, K:] == 0) and np.all(lb[:, K:] == 0)


def test_sigmoid_holes_stay_zero(emu):
    """sigmoid(0) = 0.5: a hole that took the op would show as 0.5 in the rows; holes are 0 after the op"""
    dy, aux, geom, n, R, K, ref = setup(emu, "stride2_tail_rows", 4, "sigmoid")
    dst = np.full((R, up(K, 4)), 7.0, np.float32)
    run(emu, F32, "stride2_tail_rows", "sigmoid", dy, aux, geom, n, dst, None, None, None, dst.shape[1], None, K)
    taps = transposed_rows(np.ones_like(dy), "stride2_tail_rows") != 0
    assert taps.mean() < 0.3                       # about three quarters of the taps are holes at stride 2
    assert np.all(dst[:, :K][~taps] == 0) and np.any(dst[:, :K][taps] != 0)
    same_bits(dst, ref)


def test_tail_rows_have_no_window(emu):
    """(H + 2pH - kH) mod sH input rows and columns lie past every window: their rows are all zero"""
    dy, aux, geom, n, R, K, ref = setup(emu, "stride2_tail_rows", 5, "none")
    dst = np.full((R, up(K, 4)), 7.0, np.float32)
    run(emu, F32, "stride2_tail_rows", "none", dy, aux, geom, n, dst, None, None, None, dst.shape[1], None, K)
    H, W = CASES["stride2_tail_rows"][2:4]
    pix = dst.reshape(n, H, W, -1)
    assert np.all(pix[:, H - 1] == 0) and np.all(pix[:, :, W - 1] == 0)
    assert np.any(pix[:, H - 2] != 0)


def test_input_grad_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_input_grad.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_conv_input_grad.py"], [], 2400) >= 60
