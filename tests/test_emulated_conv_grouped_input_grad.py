"""CPU-only: the direct grouped-convolution kernel in its input-gradient instantiation (laser_b200/csrc/gemm_simt.cuh:
conv_grouped_direct_kernel<MC, true>, the exact path of laser_b200_conv2d_grouped_input_grad_f32_fused_dev) on host threads, with
the tile the library plans over the transposed geometry, against the oracle per image and group, bit for bit:
gemm_strided(W'_g, rows_{n,g}, alpha, beta) with W'_g the group's filters rotated by 180 degrees with the channel axes swapped
and rows_{n,g} the input pixels' windows over op(dY) of the group's channels, zero-dilated by the strides and padded by
kH - 1 - pH, built in numpy (holes 0 after the op).  Cases: depthwise, channel multiplier 2, stride 2, sH != sW with a
non-square kernel, 7 x 7 with padding 3, Cg = 4, K' = 576 (the chain restarts at 512), grouped 1 x 1, 1 x 1 at stride 2, input
rows no window covers, an odd input width, two column tiles and fewer CTAs than tiles; every case with alpha = 1, beta = 0
over a NaN-filled dX, relu_grad with alpha = -0.5, beta = 1.25, tanh_grad and sigmoid_grad with alpha = 2, and sigmoid (an op
that is not 0 at 0) with beta = 1.  Also the GPU test file of the entry against the host-emulated library, which runs the
periodic A of the tensor-core paths on the wgmma kernel's functional model."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci, f32 = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_float
OPS = {"none": 0, "sigmoid": 3, "relu_grad": 4, "tanh_grad": 5, "sigmoid_grad": 6}

# forward geometries (n, C, H, W, Cout, kH, kW, pH, pW, sH, sW, groups)
CASES = {
    "depthwise": (2, 8, 9, 9, 8, 3, 3, 1, 1, 1, 1, 8),
    "multiplier2": (2, 4, 7, 7, 8, 3, 3, 1, 1, 1, 1, 4),
    "depthwise_stride2": (2, 6, 12, 10, 6, 3, 3, 1, 1, 2, 2, 6),
    "stride21_non_square": (2, 6, 12, 9, 6, 3, 2, 1, 0, 2, 1, 6),
    "depthwise_7x7_pad3": (1, 3, 11, 10, 3, 7, 7, 3, 3, 1, 1, 3),
    "cg4": (2, 16, 8, 8, 16, 3, 3, 1, 1, 1, 1, 4),
    "mg64_kc_flush": (1, 8, 5, 5, 128, 3, 3, 1, 1, 1, 1, 2),      # K' = 64 * 9 = 576 > 512
    "grouped_1x1": (2, 8, 6, 6, 12, 1, 1, 0, 0, 1, 1, 4),
    "grouped_1x1_stride2": (2, 8, 7, 7, 8, 1, 1, 0, 0, 2, 2, 4),
    "tail_rows": (2, 4, 8, 8, 4, 3, 3, 0, 0, 2, 2, 4),              # (8 - 3) mod 2: row and column 7 get no window
    "odd_in_w": (2, 6, 6, 13, 6, 3, 3, 1, 1, 1, 2, 3),              # dX 13 wide, Cg = 2
    "two_column_tiles": (1, 2, 4, 150, 2, 3, 3, 1, 1, 1, 1, 2),
    "multiplier3_rows": (3, 2, 40, 5, 6, 3, 3, 1, 1, 1, 1, 2),      # Mg = 3, several row tiles
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dX (never read), beta != 0 over a seeded one
VARIANTS = {"plain": ("none", 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 2.0, 0.0), "sigmoid": ("sigmoid", 0.75, 1.0)}


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_grouped_input_grad_emu", ["gemm_simt.cuh", "gemm_simt_kernel.inc", "layers.cuh", "ptx.cuh",
                                                               "split.cuh", "f16_scale.cuh", "tc_params.h"]))
    L.emu_conv_grouped_input_grad.argtypes = [vp, vp, vp, vp, i64, f32, f32, ci, vp, ci]
    L.emu_conv_grouped_input_grad.restype = ci
    L.emu_operand_op.argtypes = [ci, vp, vp, i64, vp]
    L.emu_operand_op.restype = None
    return L


def p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def out_hw(case):
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    return 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW


def data(case, seed, op):
    """-> (dY, filters, aux or None, dX0)"""
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    oh, ow = out_hw(case)
    rng = np.random.default_rng(seed)
    dy = rng.uniform(-2, 2, (n, Co, oh, ow)).astype(np.float32)
    k = rng.uniform(-1, 1, (Co, C // G, kH, kW)).astype(np.float32)
    aux = rng.uniform(-1, 1, dy.shape).astype(np.float32) if OPS[op] >= 4 else None
    x0 = rng.uniform(-1, 1, (n, C, H, W)).astype(np.float32)
    return dy, k, aux, x0


def windows(z, case):
    """[n][H * W][K'] rows of z [n][c][outH][outW]: input pixel (ih, iw)'s window zero-dilated by the strides and padded by
    kH - 1 - pH, in the order (c, kh', kw'); 0 wherever a tap falls between, before or past z's rows and columns"""
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    oh, ow = z.shape[2:]

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, pH, sH, oh)
    wq, vw = axis(W, kW, pW, sW, ow)
    g = z[:, :, hq[:, :, None, None], wq[None, None, :, :]]
    g = np.where((vh[:, :, None, None] & vw[None, None, :, :])[None, None], g, np.float32(0))
    return np.ascontiguousarray(g.transpose(0, 2, 4, 1, 3, 5).reshape(n, H * W, z.shape[1] * kH * kW)).astype(np.float32)


def oracle(emu, case, dy, k, aux, x0, op, alpha, beta):
    """gemm_strided(W'_g, rows_{n,g}, alpha, beta) per image and group, into dX0 (NaN-filled when beta = 0)"""
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    Cg, Mg, HW = C // G, Co // G, H * W
    z = np.empty_like(dy)
    emu.emu_operand_op(OPS[op], p(dy), p(aux), dy.size, p(z))
    K = Mg * kH * kW
    out = (x0 if beta != 0 else np.full_like(x0, np.nan)).reshape(n, C, HW).copy()
    for g in range(G):
        a = np.ascontiguousarray(k[g * Mg:(g + 1) * Mg, :, ::-1, ::-1].transpose(1, 0, 2, 3).reshape(Cg, K))
        rows = windows(np.ascontiguousarray(z[:, g * Mg:(g + 1) * Mg]), case)
        for i in range(n):
            c = np.ascontiguousarray(out[i, g * Cg:(g + 1) * Cg])
            O.gemm_strided(Cg, HW, K, alpha, a, K, 1, np.ascontiguousarray(rows[i]), 1, K, beta, c, HW, 1)
            out[i, g * Cg:(g + 1) * Cg] = c
    return out.reshape(x0.shape)


def run(emu, case, dy, k, aux, x0, op, alpha, beta, grid=0):
    dx = x0.copy() if beta != 0 else np.full_like(x0, np.nan)
    geom = np.array(CASES[case][:11], np.int64)
    mc = emu.emu_conv_grouped_input_grad(p(dx), p(dy), p(k), p(geom), CASES[case][11], alpha, beta, OPS[op], p(aux), grid)
    assert mc in (1, 2, 4)
    return dx, mc


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.nanmax(np.abs(a - b))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", list(CASES))
def test_direct_kernel_equals_the_oracle_per_image_and_group(emu, case, variant):
    op, alpha, beta = VARIANTS[variant]
    dy, k, aux, x0 = data(case, 1, op)
    got, mc = run(emu, case, dy, k, aux, x0, op, alpha, beta)
    same_bits(got, oracle(emu, case, dy, k, aux, x0, op, alpha, beta))
    if beta == 0:
        assert not np.isnan(got).any()
    Cg = CASES[case][1] // CASES[case][11]
    assert mc == (4 if Cg % 4 == 0 else 2 if Cg % 2 == 0 else 1)


def test_grid_stride_pass_covers_every_tile(emu):
    """fewer CTAs than tiles: each CTA walks several tiles, restaging the dilated patch and dX's beta term each time"""
    dy, k, aux, x0 = data("cg4", 2, "relu_grad")
    got, _ = run(emu, "cg4", dy, k, aux, x0, "relu_grad", -0.5, 1.25, grid=3)
    same_bits(got, oracle(emu, "cg4", dy, k, aux, x0, "relu_grad", -0.5, 1.25))


def test_rows_no_window_covers_get_beta_dx_only(emu):
    """(H + 2pH - kH) mod sH = 1: the last input row and column lie in no window, so they are beta * dX0 (every tap a hole)"""
    dy, k, aux, x0 = data("tail_rows", 3, "relu_grad")
    got, _ = run(emu, "tail_rows", dy, k, aux, x0, "relu_grad", -0.5, 1.25)
    np.testing.assert_array_equal(got[:, :, -1, :], np.float32(1.25) * x0[:, :, -1, :])
    np.testing.assert_array_equal(got[:, :, :, -1], np.float32(1.25) * x0[:, :, :, -1])
    assert np.any(got[:, :, -2, :-1] != np.float32(1.25) * x0[:, :, -2, :-1])


@pytest.mark.parametrize("case", ["depthwise", "depthwise_stride2"])
def test_inf_filter_tap_on_holes_and_padding_gives_nan_where_the_oracle_does(emu, case):
    """a filter tap of Inf is multiplied by the zeros of the padding (stride 1) or of the holes (stride 2) for some input
    pixels: NaN exactly there, as in the GEMM over the windows; the other pixels keep the oracle's bits"""
    dy, k, aux, x0 = data(case, 4, "none")
    k[2, 0, 0, 0] = np.inf    # channel 2's top-left tap: W'_2's last tap, past the bottom and right edges for some pixels
    got, _ = run(emu, case, dy, k, aux, x0, "none", 1.0, 0.0)
    want = oracle(emu, case, dy, k, aux, x0, "none", 1.0, 0.0)
    nan = np.isnan(want)
    assert nan[:, 2].any() and not nan[:, 2].all() and not np.delete(nan, 2, axis=1).any()
    assert np.array_equal(np.isnan(got), nan)
    same_bits(got[~nan], want[~nan])


def test_grouped_input_grad_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_grouped_input_grad.py (backend-neutral) on the CPU build of the whole library, minus the H100-only
    cases"""
    assert _run_gpu_files(["test_gpu_conv_grouped_input_grad.py"], [], 2400) >= 80
