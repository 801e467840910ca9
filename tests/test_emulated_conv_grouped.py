"""CPU-only: the direct grouped-convolution kernel (laser_b200/csrc/gemm_simt.cuh: conv_grouped_direct_kernel, the exact path of
laser_b200_conv2d_grouped_f32_fused_dev) on host threads, with the tile the library plans, against the oracle's
conv2d_im2col of each group's slice -- bit for bit, bias and every activation included (tanh and sigmoid through the exact
kernel's simt_bias_act).  Cases: depthwise, channel multiplier 2, stride 2 with a non-square kernel, 7 x 7 with padding 3,
Cg = 4, Cg = 64 (Kg = 576: the chain restarts at 512 like the exact GEMM's), grouped 1 x 1, an odd output width, two column
tiles, and more images than a grid-stride pass.  Also the GPU test file of the entry against the host-emulated library, which
runs the wgmma kernel's periodic A on the functional model."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int

# (n, C, H, W, Cout, kH, kW, pH, pW, sH, sW, groups)
CASES = {
    "depthwise": (2, 8, 9, 9, 8, 3, 3, 1, 1, 1, 1, 8),
    "multiplier2": (2, 4, 7, 7, 8, 3, 3, 1, 1, 1, 1, 4),
    "stride2_non_square": (2, 6, 12, 9, 6, 3, 2, 1, 0, 2, 1, 6),
    "depthwise_7x7_pad3": (1, 3, 11, 10, 3, 7, 7, 3, 3, 1, 1, 3),
    "cg4": (2, 16, 8, 8, 16, 3, 3, 1, 1, 1, 1, 4),
    "cg64_kc_flush": (1, 128, 5, 5, 8, 3, 3, 1, 1, 1, 1, 2),
    "grouped_1x1": (2, 8, 6, 6, 12, 1, 1, 0, 0, 1, 1, 4),
    "odd_out_w": (2, 6, 6, 13, 6, 3, 3, 1, 1, 1, 2, 3),
    "two_column_tiles": (1, 2, 4, 150, 2, 3, 3, 1, 1, 1, 1, 2),
    "multiplier3_rows": (3, 2, 40, 5, 6, 3, 3, 1, 1, 1, 1, 2),   # Mg = 3: one channel per thread, several row tiles
}
ACTS = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_grouped_emu", ["gemm_simt.cuh", "gemm_simt_kernel.inc", "layers.cuh",
                                                   "ptx.cuh"]))
    L.emu_conv_grouped.argtypes = [vp, vp, vp, vp, i64, vp, ci, ci]
    L.emu_conv_grouped.restype = ci
    L.emu_bias_act.argtypes = [vp, i64, i64, vp, ci]
    L.emu_bias_act.restype = None
    return L


def p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def data(case, seed):
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    rng = np.random.default_rng(seed)
    x = rng.uniform(-2, 2, (n, C, H, W)).astype(np.float32)
    k = rng.uniform(-1, 1, (Co, C // G, kH, kW)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, Co).astype(np.float32)
    return x, k, b


def oracle(case, x, k):
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    Cg, Mg = C // G, Co // G
    parts = [O.conv2d_im2col(np.ascontiguousarray(x[:, g * Cg:(g + 1) * Cg]), (n, Cg, H, W),
                             np.ascontiguousarray(k[g * Mg:(g + 1) * Mg]), (Mg, Cg, kH, kW), (pH, pW), (sH, sW)) for g in range(G)]
    return np.ascontiguousarray(np.concatenate(parts, axis=1))


def run(emu, case, x, k, bias, act, grid=0):
    n, C, H, W, Co, kH, kW, pH, pW, sH, sW, G = CASES[case]
    oh, ow = 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW
    out = np.full((n, Co, oh, ow), np.nan, np.float32)
    geom = np.array(CASES[case][:11], np.int64)
    mc = emu.emu_conv_grouped(p(out), p(x), p(k), p(geom), G, p(bias), ACTS[act], grid)
    assert mc in (1, 2, 4)
    return out, mc


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.nanmax(np.abs(a - b))


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("case", list(CASES))
def test_direct_kernel_equals_the_oracle_per_group(emu, case, act):
    x, k, b = data(case, 1)
    got, mc = run(emu, case, x, k, b if act != "none" else None, act)
    want = oracle(case, x, k)
    if act != "none":
        n, co = want.shape[:2]
        flat = np.ascontiguousarray(want.transpose(1, 0, 2, 3).reshape(co, -1))
        emu.emu_bias_act(p(flat), co, flat.shape[1], p(b), ACTS[act])
        want = np.ascontiguousarray(flat.reshape((co, n) + want.shape[2:]).transpose(1, 0, 2, 3))
    same_bits(got, want)
    Mg = CASES[case][4] // CASES[case][11]
    assert mc == (4 if Mg % 4 == 0 else 2 if Mg % 2 == 0 else 1)


def test_grid_stride_pass_covers_every_tile(emu):
    """fewer CTAs than tiles: each CTA walks several tiles, restaging the patch each time"""
    x, k, b = data("cg4", 2)
    got, _ = run(emu, "cg4", x, k, None, "none", grid=3)
    same_bits(got, oracle("cg4", x, k))


def test_padding_taps_multiply_zero(emu):
    """an Inf filter tap that only ever meets the padding for the first output row gives NaN there, as the GEMM over the
    im2col matrix does (0 * Inf), and finite values elsewhere"""
    x, k, b = data("depthwise", 3)
    k[2, 0, 0, :] = np.inf    # top row of taps of channel 2: in the padding for output row 0
    got, _ = run(emu, "depthwise", x, k, None, "none")
    want = oracle("depthwise", x, k)
    assert np.isnan(want[:, 2, 0]).all()
    same_bits(got, want)


def test_grouped_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_grouped.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_conv_grouped.py"], [], 2400) >= 80
