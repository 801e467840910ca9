"""CPU-only: prologue fusion -- an elementwise op (relu / tanh / sigmoid or a derivative with its aux tensor) applied to an
operand by the preparation kernels of laser_b200/csrc/split.cuh (HAS_OP instantiations), executed on host threads against
numpy restatements; and the GPU test file of the fused entry against the host-emulated library.

Exact ops (none, relu and the three derivatives, every operation rounded on its own) must match bit for bit, pieces and
scale words alike; tanh and sigmoid (libm on the host, numpy here) within a few ulp."""
import ctypes

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
EXACT_OPS = (0, 1, 4, 5, 6)
ALL_OPS = (0, 1, 2, 3, 4, 5, 6)


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("prologue_emu", ["split.cuh", "f16_scale.cuh"]))
    L.emu_op_split_rows_tf32.argtypes = [ci, vp, i64, vp, i64, i64, i64, vp, vp, i64, ci]
    L.emu_op_f16x2_rows_fused.argtypes = [ci, ci, vp, i64, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_op_absmax_cols.argtypes = [ci, vp, i64, vp, i64, i64, i64, vp, ci]
    L.emu_op_split_cols_f16x2.argtypes = [ci, vp, i64, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_op_pack_general_f32.argtypes = [ci, ci, vp, i64, i64, vp, i64, i64, i64, i64, vp, vp, i64, ci, ci]
    for n in ("emu_op_split_rows_tf32", "emu_op_f16x2_rows_fused", "emu_op_absmax_cols", "emu_op_split_cols_f16x2",
              "emu_op_pack_general_f32"):
        getattr(L, n).restype = None
    return L


def p(a, off=0):
    return ctypes.c_void_p(a.ctypes.data + off * a.itemsize) if a is not None else None


def op_ref(op, x, y):
    """the header's formulas, float32 step by step (numpy rounds every float32 operation on its own)"""
    x = np.asarray(x, np.float32); y = np.asarray(y, np.float32)
    one = np.float32(1)
    with np.errstate(all="ignore"):
        if op == 0:
            return x
        if op == 1:
            return np.fmax(x, np.float32(0))
        if op == 2:
            return np.tanh(x)
        if op == 3:
            return one / (one + np.exp(-x))
        if op == 4:
            return np.where(y > 0, x, np.float32(0)).astype(np.float32)
        if op == 5:
            return x * (one - y * y)
        return x * (y * (one - y))


def data(shape, op, seed):
    """operand and aux: aux in the range each derivative is used with (tanh / sigmoid outputs, signed pre-activations)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape).astype(np.float32)
    if op == 5:
        y = rng.uniform(-1, 1, shape).astype(np.float32)
    elif op == 6:
        y = rng.uniform(0, 1, shape).astype(np.float32)
    else:
        y = rng.standard_normal(shape).astype(np.float32)
    return x, y


def assert_close_ulp(got, want, ulps):
    g = got.astype(np.float32).view(np.int32).astype(np.int64)
    w = want.astype(np.float32).view(np.int32).astype(np.int64)
    assert np.abs(g - w).max() <= ulps, np.abs(g - w).max()


def f16_restate(xo, words, per_col):
    """the two fp16 pieces of xo scaled by the power of two of its word (test_emulated_split.py restates the same)"""
    e = (words >> 23).astype(np.int64)
    scale = (2.0 ** np.where(e == 0, 0, np.clip(14 - (e - 127), -126, 126))).astype(np.float32)
    with np.errstate(all="ignore"):
        xs = xo * (scale[None, :] if per_col else scale[:, None])
        h = xs.astype(np.float16)
        l = (xs - h.astype(np.float32)).astype(np.float16)
    return h.view(np.uint16), l.view(np.uint16), xs


def check_f16(op, xo, words, hb, lb, Cc, per_col):
    ld = -(-Cc // 4) * 4
    want_w = np.abs(xo).max(axis=0 if per_col else 1).astype(np.float32).view(np.uint32)
    h, l, xs = f16_restate(xo, words, per_col)
    if op in EXACT_OPS:
        assert np.array_equal(words, want_w)
        assert np.array_equal(hb[:, :Cc], h) and np.array_equal(lb[:, :Cc], l)
    else:
        assert np.abs(words.astype(np.int64) - want_w.astype(np.int64)).max() <= 4
        sc = xs / np.where(xo == 0, 1, xo)                     # the per-row / per-column scale
        rec = (hb[:, :Cc].view(np.float16).astype(np.float64) + lb[:, :Cc].view(np.float16)) / sc
        assert np.abs(rec - xo).max() <= 4 * 2.0 ** -23 * np.abs(xo).max() + 1e-30
    assert np.all(hb[:, Cc:ld] == 0) and np.all(lb[:, Cc:ld] == 0)   # padding stays zero (it feeds the MMA)


@pytest.mark.parametrize("op", ALL_OPS)
@pytest.mark.parametrize("R,Cc,src_ld", [(33, 30, 32), (9, 300, 300), (20, 1500, 1504)])
def test_k_major_fused_rows(emu, op, R, Cc, src_ld):
    """f16x2_rows_fused_kernel<32 / 256, true>: the abs-max word, the scale and the pieces are those of op(x).  1500 floats
    per row is a length the ring kernel would take without an op (16-byte aligned rows, 1024 < Cc <= 8192)."""
    x, y = data((R, src_ld), op, 10 + op)
    xo = op_ref(op, x[:, :Cc], y[:, :Cc])
    ldb = -(-Cc // 8) * 8
    for group, grid in ((32, 2), (256, 3)):
        w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
        emu.emu_op_f16x2_rows_fused(group, op, p(y) if op >= 4 else None, src_ld, p(x), R, Cc, src_ld, p(hb), p(lb), ldb, p(w),
                                    grid)
        check_f16(op, xo, w, hb, lb, Cc, per_col=False)


@pytest.mark.parametrize("op", ALL_OPS)
@pytest.mark.parametrize("R,Cc,src_ld", [(40, 30, 32), (130, 257, 260)])
def test_mn_major_absmax_and_split(emu, op, R, Cc, src_ld):
    """absmax_mn_kernel<true, true> + split_rows_f16x2_kernel<true, true>: one word per column, over op(x)"""
    x, y = data((R, src_ld), op, 20 + op)
    xo = op_ref(op, x[:, :Cc], y[:, :Cc])
    ldb = -(-Cc // 8) * 8
    w = np.zeros(Cc, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    aux = p(y) if op >= 4 else None
    emu.emu_op_absmax_cols(op, aux, src_ld, p(x), R, Cc, src_ld, p(w), 3)
    emu.emu_op_split_cols_f16x2(op, aux, src_ld, p(x), R, Cc, src_ld, p(hb), p(lb), ldb, p(w), 2)
    check_f16(op, xo, w, hb, lb, Cc, per_col=True)


def tf32_rna(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.mark.parametrize("op", ALL_OPS)
def test_tf32_split_rows(emu, op):
    R, Cc, src_ld = 33, 30, 32
    x, y = data((R, src_ld), op, 30 + op)
    xo = op_ref(op, x[:, :Cc], y[:, :Cc])
    ld = 32
    hi = np.full((R, ld), 9, np.float32); lo = np.full((R, ld), 9, np.float32)
    emu.emu_op_split_rows_tf32(op, p(y) if op >= 4 else None, src_ld, p(x), R, Cc, src_ld, p(hi), p(lo), ld, 3)
    if op in EXACT_OPS:
        h = tf32_rna(xo)
        assert np.array_equal(hi[:, :Cc], h) and np.array_equal(lo[:, :Cc], tf32_rna(xo - h))
    else:
        assert np.abs((hi[:, :Cc].astype(np.float64) + lo[:, :Cc]) - xo).max() <= 8 * 2.0 ** -24
    assert np.all(hi[:, Cc:] == 0) and np.all(lo[:, Cc:] == 0)


def strided(R, Cc, sr, sc, base, seed, op=0):
    """a buffer holding an R x Cc view with element strides (sr, sc) starting `base` elements in; -> buffer, offset, view"""
    lo_off = min(0, (R - 1) * sr) + min(0, (Cc - 1) * sc)
    hi_off = max(0, (R - 1) * sr) + max(0, (Cc - 1) * sc)
    buf, _ = data(base + hi_off - lo_off + 1, 0, seed)
    if op == 5:
        buf = np.tanh(buf)
    elif op == 6:
        buf = (1 / (1 + np.exp(-buf))).astype(np.float32)
    off = base - lo_off
    return buf, off, buf[off + np.arange(R)[:, None] * sr + np.arange(Cc)[None, :] * sc]


@pytest.mark.parametrize("op", ALL_OPS)
@pytest.mark.parametrize("aux_layout", ["same", "transposed", "negative", "misaligned"])
@pytest.mark.parametrize("mode", [0, 1])
def test_general_gather(emu, op, aux_layout, mode):
    """pack_general_kernel<float, MODE, true>: operand every other column, aux with its own strides"""
    R, Cc, sr, sc = 37, 45, 100, 2
    buf, off, x = strided(R, Cc, sr, sc, 0, 40 + op)
    ar, ac, base = {"same": (sr, sc, 0), "transposed": (1, R, 0), "negative": (-Cc, -1, 0), "misaligned": (Cc, 1, 1)}[aux_layout]
    abuf, aoff, y = strided(R, Cc, ar, ac, base, 50 + op, op)
    xo = op_ref(op, x, y)
    ld = 48
    dst = np.full((R, ld), 7, np.float32); dlo = np.full((R, ld), 7, np.float32)
    emu.emu_op_pack_general_f32(mode, op, p(abuf, aoff) if op >= 4 else None, ar, ac, p(buf, off), R, Cc, sr, sc, p(dst), p(dlo),
                                ld, 0, 4)
    got = dst[:, :Cc] if mode == 0 else dst[:, :Cc].astype(np.float64) + dlo[:, :Cc]
    if op in EXACT_OPS:
        if mode == 0:
            assert np.array_equal(got, xo)
        else:
            h = tf32_rna(xo)
            assert np.array_equal(dst[:, :Cc], h) and np.array_equal(dlo[:, :Cc], tf32_rna(xo - h))
    elif mode == 0:
        assert_close_ulp(got, xo, 4)
    else:
        assert np.abs(got - xo).max() <= 8 * 2.0 ** -24
    assert np.all(dst[:, Cc:] == 7)


def test_scale_is_taken_after_the_op(emu):
    """raw rows below 1e-20 under SIGMOID (outputs ~0.5) and TANH_GRAD with |aux| up to 300 (factors near -9e4): a scale
    word taken over the raw values would overflow / waste the fp16 range; these must equal the words of the op's output"""
    R, Cc = 8, 64
    rng = np.random.default_rng(7)
    x = (rng.uniform(-1, 1, (R, Cc)) * 1e-21).astype(np.float32)
    w = np.zeros(R, np.uint32); hb = np.zeros((R, Cc), np.uint16); lb = np.zeros((R, Cc), np.uint16)
    emu.emu_op_f16x2_rows_fused(32, 3, None, Cc, p(x), R, Cc, Cc, p(hb), p(lb), Cc, p(w), 2)
    assert np.all(w.view(np.float32) == np.float32(0.5))
    y = rng.uniform(-300, 300, (R, Cc)).astype(np.float32)
    x = rng.uniform(-1, 1, (R, Cc)).astype(np.float32)
    xo = op_ref(5, x, y)
    emu.emu_op_f16x2_rows_fused(32, 5, p(y), Cc, p(x), R, Cc, Cc, p(hb), p(lb), Cc, p(w), 2)
    check_f16(5, xo, w, hb, lb, Cc, per_col=False)
    wc = np.zeros(Cc, np.uint32)
    emu.emu_op_absmax_cols(5, p(y), Cc, p(x), R, Cc, Cc, p(wc), 2)
    emu.emu_op_split_cols_f16x2(5, p(y), Cc, p(x), R, Cc, Cc, p(hb), p(lb), Cc, p(wc), 2)
    check_f16(5, xo, wc, hb, lb, Cc, per_col=True)


def test_relu_grad_is_a_select(emu):
    """z <= 0 or NaN gives 0 even for x = inf; z > 0 passes x, NaN included"""
    x = np.array([[np.inf, np.inf, np.nan, 3.0, -np.inf]], np.float32)
    z = np.array([[0.0, np.nan, 1.0, -1.0, 2.0]], np.float32)
    dst = np.full((1, 8), 7, np.float32)
    emu.emu_op_pack_general_f32(0, 4, p(z), 5, 1, p(x), 1, 5, 5, 1, p(dst), None, 8, 0, 1)
    got = dst[0]
    assert got[0] == 0 and got[1] == 0 and np.isnan(got[2]) and got[3] == 0 and got[4] == -np.inf
    assert np.array_equal(op_ref(4, x, z)[0], got[:5], equal_nan=True)


def test_fused_prologue_file_against_the_host_emulated_library():
    """tests/test_gpu_fused_prologue.py (backend-neutral) on the CPU build of the whole library, minus the sizes skipped there"""
    assert _run_gpu_files(["test_gpu_fused_prologue.py"], [], 2400) >= 60
