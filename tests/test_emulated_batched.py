"""CPU-only: the batched fused product.  The BATCHED instantiations of the preparation kernels (laser_b200/csrc/split.cuh) on
host threads against numpy restatements, problem by problem (exact ops bit for bit); the GPU test file of the batched entry
against the host-emulated library, which runs the BATCHED tensor-core kernel on host threads; and the shipped library's
batched GEMM kernels issue 3-D TMA loads."""
import collections
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_prologue import EXACT_OPS, assert_close_ulp, check_f16, data, op_ref, p, tf32_rna
from test_emulated_python_mirror import _run_gpu_files
from test_sass_evidence import L as _L

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
OPS = (0, 1, 2, 4, 5, 6)


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("batched_emu", ["split.cuh", "f16_scale.cuh"]))
    L.emu_b_split_rows_tf32.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, ci]
    L.emu_b_f16x2_rows_fused.argtypes = [ci, ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_b_absmax_cols.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, ci]
    L.emu_b_split_cols_f16x2.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_b_pack_general_f32.argtypes = [ci, ci, vp, i64, i64, i64, vp, i64, i64, i64, i64, i64, i64, vp, vp, i64, ci]
    for n in ("emu_b_split_rows_tf32", "emu_b_f16x2_rows_fused", "emu_b_absmax_cols", "emu_b_split_cols_f16x2",
              "emu_b_pack_general_f32"):
        getattr(L, n).restype = None
    return L


def problems(n, R, src_ld, bs, op, seed):
    """n problems of R x src_ld floats, bs apart (bs < 0: the last one first in memory, 0: one shared matrix); -> buffer,
    offset of problem 0, operand and aux views per problem, aux buffer and its offset (aux laid out like the operand)"""
    m = 1 if bs == 0 else n
    per = abs(bs) if bs else R * src_ld
    x, y = data((m * per,), op, seed)
    base = (m - 1) * per if bs < 0 else 0
    view = lambda buf, b: buf[base + b * bs:base + b * bs + R * src_ld].reshape(R, src_ld)
    return x, base, [view(x, b) for b in range(n)], y, [view(y, b) for b in range(n)]


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("bs_kind", ["stacked", "padded", "negative", "shared"])
def test_k_major_rows(emu, op, bs_kind):
    """f16x2_rows_fused_kernel<32 / 256, true, true>: stacked words and pieces of op(x) per problem"""
    n, R, Cc, src_ld = 3, 9, 300, 304
    bs = {"stacked": R * src_ld, "padded": R * src_ld + 8, "negative": -(R * src_ld + 4), "shared": 0}[bs_kind]
    x, base, xs, y, ys = problems(n, R, src_ld, bs, op, 10 + op)
    ldb = -(-Cc // 8) * 8
    for group, grid in ((32, 2), (256, 3)):
        w = np.full(n * R, 77, np.uint32); hb = np.full((n * R, ldb), 9, np.uint16); lb = np.full((n * R, ldb), 9, np.uint16)
        emu.emu_b_f16x2_rows_fused(group, op, p(y, base) if op >= 4 else None, src_ld, bs, p(x, base), R, Cc, src_ld, bs, n,
                                   p(hb), p(lb), ldb, p(w), grid)
        for b in range(n):
            check_f16(op, op_ref(op, xs[b][:, :Cc], ys[b][:, :Cc]), w[b * R:(b + 1) * R], hb[b * R:(b + 1) * R],
                      lb[b * R:(b + 1) * R], Cc, per_col=False)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("bs_kind", ["stacked", "negative"])
def test_mn_major_scales_and_split(emu, op, bs_kind):
    """absmax_mn_kernel<true, true, true> + split_rows_f16x2_kernel<true, true, true>: one word per (problem, column); the
    row blocks (64 rows) end at each problem's last row"""
    n, R, Cc, src_ld = 3, 130, 257, 260
    bs = R * src_ld if bs_kind == "stacked" else -(R * src_ld + 4)
    x, base, xs, y, ys = problems(n, R, src_ld, bs, op, 20 + op)
    ldb = -(-Cc // 8) * 8
    w = np.zeros(n * Cc, np.uint32); hb = np.full((n * R, ldb), 9, np.uint16); lb = np.full((n * R, ldb), 9, np.uint16)
    aux = p(y, base) if op >= 4 else None
    emu.emu_b_absmax_cols(op, aux, src_ld, bs, p(x, base), R, Cc, src_ld, bs, n, p(w), 3)
    emu.emu_b_split_cols_f16x2(op, aux, src_ld, bs, p(x, base), R, Cc, src_ld, bs, n, p(hb), p(lb), ldb, p(w), 2)
    for b in range(n):
        check_f16(op, op_ref(op, xs[b][:, :Cc], ys[b][:, :Cc]), w[b * Cc:(b + 1) * Cc], hb[b * R:(b + 1) * R], lb[b * R:(b + 1) * R],
                  Cc, per_col=True)


@pytest.mark.parametrize("op", OPS)
def test_tf32_split_rows(emu, op):
    n, R, Cc, src_ld = 3, 33, 30, 32
    bs = -(R * src_ld + 12)
    x, base, xs, y, ys = problems(n, R, src_ld, bs, op, 30 + op)
    hi = np.full((n * R, 32), 9, np.float32); lo = np.full((n * R, 32), 9, np.float32)
    emu.emu_b_split_rows_tf32(op, p(y, base) if op >= 4 else None, src_ld, bs, p(x, base), R, Cc, src_ld, bs, n, p(hi), p(lo), 32, 3)
    for b in range(n):
        xo = op_ref(op, xs[b][:, :Cc], ys[b][:, :Cc])
        h, l = hi[b * R:(b + 1) * R, :Cc], lo[b * R:(b + 1) * R, :Cc]
        if op in EXACT_OPS:
            assert np.array_equal(h, tf32_rna(xo)) and np.array_equal(l, tf32_rna(xo - tf32_rna(xo)))
        else:
            assert np.abs((h.astype(np.float64) + l) - xo).max() <= 8 * 2.0 ** -24
    assert np.all(hi[:, Cc:] == 0) and np.all(lo[:, Cc:] == 0)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("mode", [0, 1])
def test_general_gather(emu, op, mode):
    """pack_general_kernel<float, MODE, true, true>: every other column, problems with a negative stride, aux transposed with
    its own batch stride"""
    n, R, Cc = 3, 37, 45
    sr, sc = 2 * Cc, 2
    per = R * 2 * Cc + 3
    x, _ = data((n * per,), 0, 40 + op)
    base = (n - 1) * per
    y, _ = data((n * R * Cc + 5 * n,), op, 50 + op)
    if op == 5:
        y = np.tanh(y)
    elif op == 6:
        y = (1 / (1 + np.exp(-y))).astype(np.float32)
    aux_bs = R * Cc + 5
    ld = 48
    dst = np.full((n * R, ld), 7, np.float32); dlo = np.full((n * R, ld), 7, np.float32)
    emu.emu_b_pack_general_f32(mode, op, p(y) if op >= 4 else None, 1, R, aux_bs, p(x, base), R, Cc, sr, sc, -per, n, p(dst), p(dlo),
                               ld, 4)
    i, j = np.arange(R)[:, None], np.arange(Cc)[None, :]
    for b in range(n):
        xo = op_ref(op, x[base - b * per + i * sr + j * sc], y[b * aux_bs + i + j * R])
        got = dst[b * R:(b + 1) * R, :Cc]
        if mode == 1:
            if op in EXACT_OPS:
                assert np.array_equal(got, tf32_rna(xo)) and np.array_equal(dlo[b * R:(b + 1) * R, :Cc], tf32_rna(xo - tf32_rna(xo)))
        elif op in EXACT_OPS:
            assert np.array_equal(got, xo)
        else:
            assert_close_ulp(got, xo, 4)
    assert np.all(dst[:, Cc:] == 7)


def test_batched_gemm_kernels_issue_3d_tma_loads():
    """every batched instantiation of the tensor-core kernel (template argument BATCHED = true) loads through 3-D tensor
    maps only, every one-problem instantiation through 2-D maps only"""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    if not os.path.exists(exe) or not os.path.exists(filt):
        pytest.skip("cuobjdump / cu++filt not installed")
    out = subprocess.run([exe, "-sass", _L.lib_path()], capture_output=True, text=True, check=True).stdout
    loads, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            loads[cur] = collections.Counter()
        elif cur:
            for d in re.findall(r"UTMALDG\.(\dD)", line):
                loads[cur][d] += 1
    syms = [s for s in loads if "gemm_tc_kernel" in s]
    names = subprocess.run([filt], input="\n".join(syms), capture_output=True, text=True, check=True).stdout.splitlines()
    batched = plain = 0
    for sym, name in zip(syms, names):
        # gemm_tc_kernel<ESZ, FMT16, NPASS, A_MN, B_MN, OutT, SCALED, BATCHED>(...)
        m = re.match(r"void lb200::gemm_tc_kernel<.*, \(bool\)([01])>\(", name)
        assert m, name
        if m.group(1) == "1":
            batched += 1
            assert set(loads[sym]) == {"3D"}, (name, loads[sym])
        else:
            plain += 1
            assert set(loads[sym]) == {"2D"}, (name, loads[sym])
    assert batched == 6 and plain == 10, (batched, plain)   # batched: f16x3 x 4 majors, tf32x3, tf32x1


def test_batched_file_against_the_host_emulated_library():
    """tests/test_gpu_batched_fused.py (backend-neutral) on the CPU build of the whole library, minus the H100-only case"""
    assert _run_gpu_files(["test_gpu_batched_fused.py"], [], 2400) >= 75
