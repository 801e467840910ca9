"""CPU-only: the channels-last transposed preparation (laser_b200/csrc/split.cuh: im2col_rows_kernel over an Im2colNhwcGradSrc,
the NHWC DIL / HAS_OP instantiations) on host threads in its three modes and both groups, with and without op, against the
transposed NHWC windows built in numpy -- one row per input pixel, the window over op(dY) zero-dilated by the strides in (kh',
kw', co) order, holes 0 -- run through the row kernels it stands in for: plain values exactly; f16x2 words and pieces as
f16x2_rows_fused_kernel; tf32 hi / lo as split_rows_tf32_kernel.  Words, pieces and padding columns are compared bit for bit, on
the vector path (c_out % 4 == 0, aligned dY and aux) and the scalar one (c_out = 3, 5, 117, or a misaligned dY or aux).  Also
the GPU test file of the entry against the host-emulated library."""
import ctypes

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
F32, TF32, F16X2 = 0, 1, 2
OPS = {None: 0, "relu": 1, "tanh": 2, "sigmoid": 3, "relu_grad": 4, "tanh_grad": 5, "sigmoid_grad": 6}
HEADERS = ["split.cuh", "f16_scale.cuh", "layers.cuh"]


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("conv_nhwc_input_grad_emu", HEADERS))
    L.emu_nhwc_tconv_rows.argtypes = [ci, ci, ci, ci, vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, ci]
    L.emu_nhwc_tconv_rows.restype = ci
    return L


@pytest.fixture(scope="module")
def rows():
    """the row kernels the windows replace (tests/emu/conv_emu.cpp) and the library's operand op (conv_input_grad_emu.cpp)"""
    L = ctypes.CDLL(build_emu("conv_emu", HEADERS))
    L.emu_f16x2_rows.argtypes = [ci, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_tf32_rows.argtypes = [vp, i64, i64, i64, vp, vp, i64, ci]
    for n in ("emu_f16x2_rows", "emu_tf32_rows"):
        getattr(L, n).restype = None
    O = ctypes.CDLL(build_emu("conv_input_grad_emu", HEADERS))
    O.emu_operand_op.argtypes = [ci, vp, vp, i64, vp]
    O.emu_operand_op.restype = None
    return L, O


def p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def up(x, m):
    return -(-x // m) * m


# the FORWARD geometry: (images, c_in, H, W, kH, kW, pH, pW, sH, sW, c_out)
CASES = {
    # (8 - 3) mod 2 = 1: the last input row and column lie in no window
    "stride2_tail": (2, 3, 8, 8, 3, 3, 0, 0, 2, 2, 8),
    # pH >= kH: p' = kH - 1 - pH = -1
    "pad_ge_k": (2, 2, 5, 5, 3, 3, 3, 3, 1, 1, 4),
    "pad_ge_k_stride2": (2, 2, 6, 5, 2, 2, 2, 3, 2, 2, 8),
    "non_square": (2, 3, 8, 9, 3, 5, 1, 2, 1, 2, 8),          # 3 x 5 kernel, strides (1, 2)
    "cout3": (2, 4, 7, 7, 3, 3, 1, 1, 2, 2, 3),
    "cout5": (2, 4, 7, 6, 3, 2, 1, 0, 2, 1, 5),
    "one_by_one_stride2": (2, 4, 7, 7, 1, 1, 0, 0, 2, 2, 8),
    "long_rows": (1, 2, 5, 5, 3, 3, 1, 1, 2, 2, 128),         # K' = 1152: the CTA per row, vector path
    "long_rows_cout117": (1, 2, 4, 4, 3, 3, 1, 1, 1, 1, 117),  # K' = 1053, scalar
}
# op, and which of dY / the aux sits one float past a 16-byte boundary
VARIANTS = {"plain": (None, ""), "relu_grad": ("relu_grad", ""), "sigmoid": ("sigmoid", ""),
            "tanh_grad_misaligned_dy": ("tanh_grad", "dy"), "sigmoid_grad_misaligned_aux": ("sigmoid_grad", "aux")}


def out_hw(case):
    n, C, H, W, kH, kW, pH, pW, sH, sW, co = CASES[case]
    return 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW


def tconv_rows(z, case):
    """[n * H * W][kH * kW * c_out] rows over z [n][outH][outW][c_out]: input pixel (ih, iw)'s window zero-dilated by the strides
    and padded by kH - 1 - pH, in (kh', kw', co) order; 0 wherever a tap falls between, before or past z's rows and columns"""
    n, C, H, W, kH, kW, pH, pW, sH, sW, co = CASES[case]
    oh, ow = out_hw(case)

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, pH, sH, oh)
    wq, vw = axis(W, kW, pW, sW, ow)
    g = z[:, hq[:, None, :, None], wq[None, :, None, :], :]                  # [n][H][W][kH][kW][co]
    ok = (vh[:, None, :, None] & vw[None, :, None, :])[None, :, :, :, :, None]
    g = np.where(ok, g, np.zeros((), z.dtype))
    return np.ascontiguousarray(g.reshape(n * H * W, kH * kW * co))


def setup(case, seed):
    """-> (dy [n][outH][outW][c_out], aux (the forward output's sigmoid, in (0, 1)), rows R, K'): signed data with images,
    pixels and channels at their own powers of two, so that the rows' scale words differ; +inf and -inf"""
    n, co = CASES[case][0], CASES[case][10]
    oh, ow = out_hw(case)
    rng = np.random.default_rng(seed)
    dy = rng.uniform(-3, 3, (n, oh, ow, co))
    dy *= 2.0 ** rng.integers(-8, 9, n)[:, None, None, None] * 2.0 ** rng.integers(-8, 9, (1, oh, ow, 1)) * \
        2.0 ** rng.integers(-8, 9, co)[None, None, None, :]
    dy = dy.astype(np.float32)
    dy[0, 0, 0, :] = 0.0
    dy[n - 1, oh // 2, ow // 2, co - 1] = np.inf
    dy[0, oh - 1, ow - 1, 0] = -np.inf
    aux = (1 / (1 + np.exp(-rng.uniform(-4, 4, dy.shape)))).astype(np.float32)
    K = co * CASES[case][4] * CASES[case][5]
    return dy, aux, n * CASES[case][2] * CASES[case][3], K


def lib_op(rows, name, x, y):
    out = np.empty_like(x)
    rows[1].emu_operand_op(OPS[name], p(np.ascontiguousarray(x)), p(np.ascontiguousarray(y)) if y is not None else None, x.size,
                           p(out))
    return out


def reference(rows, case, dy, aux, op):
    """the rows as the library must write them: op(dY) with the library's own op at the source positions, holes 0"""
    z = dy if op is None else lib_op(rows, op, dy, aux if op.endswith("_grad") else None)
    R, K = CASES[case][0] * CASES[case][2] * CASES[case][3], dy.shape[-1] * CASES[case][4] * CASES[case][5]
    ref = np.zeros((R, up(K, 4)), np.float32)
    ref[:, :K] = tconv_rows(z, case)
    return ref


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


def run(emu, mode, group, case, variant, dy, aux, dst, lo, hb, lb, ld, w):
    """-> the vec flag the kernel ran with; asserts it is the one the alignment rule gives"""
    op, shifted = VARIANTS[variant]
    ds = misaligned(dy) if shifted == "dy" else dy
    ys = (misaligned(aux) if shifted == "aux" else aux) if op and op.endswith("_grad") else None
    sH, sW = CASES[case][8:10]
    vec = emu.emu_nhwc_tconv_rows(mode, group, int((sH, sW) != (1, 1)), OPS[op], p(ds), p(ys), p(geom_of(case)), CASES[case][0],
                                  p(dst), p(lo), p(hb), p(lb), ld, p(w), 3)
    want = CASES[case][10] % 4 == 0 and ds.ctypes.data % 16 == 0 and (ys is None or ys.ctypes.data % 16 == 0)
    assert vec == want
    return vec


GRID = [(c, v) for c in CASES for v in VARIANTS]


@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case,variant", GRID)
def test_plain_rows_equal_the_windows(emu, rows, case, variant, group):
    dy, aux, R, K = setup(case, 1)
    ld = up(K, 4)
    dst = np.full((R, ld), 7.0, np.float32)
    run(emu, F32, group, case, variant, dy, aux, dst, None, None, None, ld, None)
    same_bits(dst, reference(rows, case, dy, aux, VARIANTS[variant][0]))


@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case,variant", GRID)
def test_tf32_pieces_equal_split_rows_tf32(emu, rows, case, variant, group):
    dy, aux, R, K = setup(case, 2)
    ld = up(K, 4)
    hi = np.full((R, ld), 7.0, np.float32); lo = np.full((R, ld), 7.0, np.float32)
    run(emu, TF32, group, case, variant, dy, aux, hi, lo, None, None, ld, None)
    ref = reference(rows, case, dy, aux, VARIANTS[variant][0])
    hr = np.full((R, ld), 9.0, np.float32); lr = np.full((R, ld), 9.0, np.float32)
    rows[0].emu_tf32_rows(p(ref), R, K, ld, p(hr), p(lr), ld, 3)
    same_bits(hi, hr); same_bits(lo, lr)


@pytest.mark.parametrize("group", [32, 256])
@pytest.mark.parametrize("case,variant", GRID)
def test_f16x2_words_and_pieces_equal_the_fused_row_kernel(emu, rows, case, variant, group):
    dy, aux, R, K = setup(case, 3)
    ldb = up(K, 8)
    w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    run(emu, F16X2, group, case, variant, dy, aux, None, None, hb, lb, ldb, w)
    ref = reference(rows, case, dy, aux, VARIANTS[variant][0])
    wr = np.full(R, 55, np.uint32); hr = np.full((R, ldb), 5, np.uint16); lr = np.full((R, ldb), 5, np.uint16)
    rows[0].emu_f16x2_rows(group, p(ref), R, K, ref.shape[1], p(hr), p(lr), ldb, p(wr), 2)
    c4 = up(K, 4)   # the row kernel writes the columns of whole float4 groups; the rest of ld is ours to zero
    same_bits(w, wr)
    same_bits(hb[:, :c4], hr[:, :c4]); same_bits(lb[:, :c4], lr[:, :c4])
    assert np.all(hb[:, K:] == 0) and np.all(lb[:, K:] == 0)


@pytest.mark.parametrize("case", ["stride2_tail", "cout3"])
def test_holes_under_sigmoid_are_zero(emu, rows, case):
    """sigmoid(0) = 0.5, but a hole is a structural zero: exactly where numpy's window has no source value the row is 0, and
    every source position holds a sigmoid value in (0, 1]; the uncovered tail row at stride 2 is all 0"""
    dy, aux, R, K = setup(case, 4)
    dy = np.clip(np.where(np.isfinite(dy), dy, 0.0), -10, 10).astype(np.float32)   # sigmoid > 0 at every source value
    ld = up(K, 4)
    dst = np.full((R, ld), 7.0, np.float32)
    run(emu, F32, 32, case, "sigmoid", dy, aux, dst, None, None, None, ld, None)
    # the source positions: numpy's rows over a tensor of ones
    mask = tconv_rows(np.ones_like(dy), case) != 0
    assert mask.any() and (~mask).any()
    assert np.all(dst[:, :K][~mask] == 0) and np.all(dst[:, :K][mask] > 0)
    assert np.all(dst[:, K:] == 0)
    if case == "stride2_tail":
        n, C, H, W = CASES[case][:4]
        assert np.all(dst.reshape(n, H, W, ld)[:, H - 1] == 0)


def test_infinities_pass_through(emu, rows):
    """+inf and -inf in dY reach the rows unchanged (no op), and the f16x2 word ignores them"""
    case = "stride2_tail"
    dy, aux, R, K = setup(case, 5)
    dst = np.full((R, up(K, 4)), 7.0, np.float32)
    run(emu, F32, 32, case, "plain", dy, aux, dst, None, None, None, dst.shape[1], None)
    assert np.isposinf(dst).any() and np.isneginf(dst).any()


def test_nhwc_input_grad_file_against_the_host_emulated_library():
    """tests/test_gpu_conv_nhwc_input_grad.py (backend-neutral) on the CPU build of the whole library, minus the H100-only
    cases"""
    assert _run_gpu_files(["test_gpu_conv_nhwc_input_grad.py"], [], 2400) >= 60
