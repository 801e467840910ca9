"""CPU-only: the batch-reduced fused product.  The CONCAT instantiations of the preparation kernels (laser_b200/csrc/split.cuh)
on host threads must write, bit for bit, what the plain kernels write for the materialised concatenation of the problems along
k -- scale words, fp16 pieces, tf32 pieces and gathered values alike; and the GPU test file of the entry against the
host-emulated library."""
import ctypes

import numpy as np
import pytest

from emu_build import build_emu
from test_emulated_batched import problems
from test_emulated_prologue import data, p
from test_emulated_python_mirror import _run_gpu_files

i64, vp, ci = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int
OPS = (0, 1, 2, 4, 5, 6)
BS_KINDS = ("stacked", "padded", "negative", "shared")
N_PROB = 3


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("batch_reduce_emu", ["split.cuh", "f16_scale.cuh"]))
    L.emu_c_split_rows_tf32.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, ci]
    L.emu_c_f16x2_rows_fused.argtypes = [ci, ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_c_absmax_cols.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, ci]
    L.emu_c_split_cols_f16x2.argtypes = [ci, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_c_pack_general_f32.argtypes = [ci, ci, vp, i64, i64, i64, vp, i64, i64, i64, i64, i64, i64, vp, vp, i64, ci]
    for n in ("emu_c_split_rows_tf32", "emu_c_f16x2_rows_fused", "emu_c_absmax_cols", "emu_c_split_cols_f16x2",
              "emu_c_pack_general_f32"):
        getattr(L, n).restype = None
    return L


@pytest.fixture(scope="module")
def plain():
    """the one-problem HAS_OP kernels (tests/emu/prologue_emu.cpp): the reference over the materialised concatenation"""
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


def padded(a):
    """a copy of a 2-D array with rows of a multiple of 4 floats (16-byte aligned, as the row kernels read them)"""
    out = np.zeros((a.shape[0], -(-a.shape[1] // 4) * 4), a.dtype)
    out[:, :a.shape[1]] = a
    return out


def batch_of(R, Cc, bs_kind, op, seed):
    """N_PROB problems of R x Cc floats in rows of src_ld (a multiple of 4 floats, as the host passes them) -> (buffer and
    offset of problem 0, aux buffer, batch stride, src_ld, the materialised concatenations -- rows end to end [R][n*Cc] and
    rows stacked [n*R][Cc] -- of operand and aux, in 16-byte aligned rows)"""
    src_ld = -(-Cc // 4) * 4 + 4
    bs = {"stacked": R * src_ld, "padded": R * src_ld + 8, "negative": -(R * src_ld + 4), "shared": 0}[bs_kind]
    x, base, xs, y, ys = problems(N_PROB, R, src_ld, bs, op, seed)
    cat = lambda vs, axis: padded(np.concatenate([v[:, :Cc] for v in vs], axis=axis))
    return x, base, y, bs, src_ld, cat(xs, 1), cat(ys, 1), cat(xs, 0), cat(ys, 0)


def same_bits(a, b):
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# K = 3: segments shorter than a float4; 301: boundaries off the 16-byte grid; 300 / 402: rows of 900 and 1206 floats, on
# either side of the warp-per-row limit (1024)
@pytest.mark.parametrize("K", [3, 300, 301, 402])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("bs_kind", BS_KINDS)
def test_k_major_rows_f16x2(emu, plain, K, op, bs_kind):
    """f16x2_rows_fused_kernel<GROUP, true, true, true>: one word per row over every problem, pieces [R][round_up(nK, 8)]"""
    R = 9
    x, base, y, bs, src_ld, xc, yc, _, _ = batch_of(R, K, bs_kind, op, 100 + op + K)
    nK = N_PROB * K
    ldb = -(-nK // 8) * 8
    aux = p(y, base) if op >= 4 else None
    for group, grid in ((32, 2), (256, 3)):
        w = np.full(R, 77, np.uint32); hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
        emu.emu_c_f16x2_rows_fused(group, op, aux, src_ld, bs, p(x, base), R, K, src_ld, bs, N_PROB, p(hb), p(lb), ldb, p(w), grid)
        rw = np.full(R, 77, np.uint32); rh = np.full((R, ldb), 9, np.uint16); rl = np.full((R, ldb), 9, np.uint16)
        plain.emu_op_f16x2_rows_fused(group, op, p(yc) if op >= 4 else None, xc.shape[1], p(xc), R, nK, xc.shape[1], p(rh), p(rl),
                                      ldb, p(rw), grid)
        same_bits(w, rw); same_bits(hb, rh); same_bits(lb, rl)


@pytest.mark.parametrize("K", [3, 301, 402])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("bs_kind", BS_KINDS)
def test_k_major_rows_tf32(emu, plain, K, op, bs_kind):
    R = 7
    x, base, y, bs, src_ld, xc, yc, _, _ = batch_of(R, K, bs_kind, op, 200 + op + K)
    nK = N_PROB * K
    ld = -(-nK // 4) * 4
    hi = np.full((R, ld), 9, np.float32); lo = np.full((R, ld), 9, np.float32)
    emu.emu_c_split_rows_tf32(op, p(y, base) if op >= 4 else None, src_ld, bs, p(x, base), R, K, src_ld, bs, N_PROB, p(hi), p(lo),
                              ld, 3)
    rhi = np.full((R, ld), 9, np.float32); rlo = np.full((R, ld), 9, np.float32)
    plain.emu_op_split_rows_tf32(op, p(yc) if op >= 4 else None, xc.shape[1], p(xc), R, nK, xc.shape[1], p(rhi), p(rlo), ld, 3)
    same_bits(hi, rhi); same_bits(lo, rlo)


@pytest.mark.parametrize("R", [3, 130])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("bs_kind", BS_KINDS)
def test_mn_major_scales_and_split(emu, plain, R, op, bs_kind):
    """absmax_mn_kernel / split_rows_f16x2_kernel<true, true, true, true>: the problems' k-rows stacked, ONE word per column
    over all of them (n * Cc words would be the batched layout); row blocks of 64 end at each problem's last row"""
    Cc = 257
    x, base, y, bs, src_ld, _, _, xc, yc = batch_of(R, Cc, bs_kind, op, 300 + op + R)
    ldb = -(-Cc // 8) * 8
    aux = p(y, base) if op >= 4 else None
    w = np.zeros(Cc + 5, np.uint32); hb = np.full((N_PROB * R, ldb), 9, np.uint16); lb = np.full((N_PROB * R, ldb), 9, np.uint16)
    emu.emu_c_absmax_cols(op, aux, src_ld, bs, p(x, base), R, Cc, src_ld, bs, N_PROB, p(w), 3)
    emu.emu_c_split_cols_f16x2(op, aux, src_ld, bs, p(x, base), R, Cc, src_ld, bs, N_PROB, p(hb), p(lb), ldb, p(w), 2)
    rw = np.zeros(Cc + 5, np.uint32); rh = np.full((N_PROB * R, ldb), 9, np.uint16); rl = np.full((N_PROB * R, ldb), 9, np.uint16)
    raux = p(yc) if op >= 4 else None
    pitch = xc.shape[1]
    plain.emu_op_absmax_cols(op, raux, pitch, p(xc), N_PROB * R, Cc, pitch, p(rw), 3)
    plain.emu_op_split_cols_f16x2(op, raux, pitch, p(xc), N_PROB * R, Cc, pitch, p(rh), p(rl), ldb, p(rw), 2)
    same_bits(w, rw); same_bits(hb, rh); same_bits(lb, rl)
    assert np.all(w[Cc:] == 0)


@pytest.mark.parametrize("K", [3, 45])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("bs_kind", BS_KINDS)
def test_general_gather(emu, plain, K, op, mode, bs_kind):
    """pack_general_kernel<float, MODE, true, true, true>: every other column of each problem, aux transposed with its own batch
    stride, problem b written to columns b * K ..; the padding columns stay unwritten"""
    R = 37
    sr, sc = 2 * K, 2
    per = R * 2 * K + 3
    bs = {"stacked": per, "padded": per + 5, "negative": -per, "shared": 0}[bs_kind]
    m = 1 if bs == 0 else N_PROB
    x, _ = data((m * (abs(bs) or per),), 0, 400 + op)
    base = (m - 1) * abs(bs) if bs < 0 else 0
    aux_bs = R * K + 5
    y, _ = data((N_PROB * aux_bs,), op, 500 + op)
    if op == 5:
        y = np.tanh(y)
    elif op == 6:
        y = (1 / (1 + np.exp(-y))).astype(np.float32)
    nK = N_PROB * K
    ld = -(-nK // 4) * 4 + 4
    dst = np.full((R, ld), 7, np.float32); dlo = np.full((R, ld), 7, np.float32)
    emu.emu_c_pack_general_f32(mode, op, p(y) if op >= 4 else None, 1, R, aux_bs, p(x, base), R, K, sr, sc, bs, N_PROB, p(dst),
                               p(dlo), ld, 4)
    i, j = np.arange(R)[:, None], np.arange(K)[None, :]
    xc = np.ascontiguousarray(np.concatenate([x[base + b * bs + i * sr + j * sc] for b in range(N_PROB)], axis=1))
    yc = np.ascontiguousarray(np.concatenate([y[b * aux_bs + i + j * R] for b in range(N_PROB)], axis=1))
    rdst = np.full((R, ld), 7, np.float32); rlo = np.full((R, ld), 7, np.float32)
    plain.emu_op_pack_general_f32(mode, op, p(yc) if op >= 4 else None, nK, 1, p(xc), R, nK, nK, 1, p(rdst), p(rlo), ld, 0, 4)
    same_bits(dst, rdst)
    if mode == 1:
        same_bits(dlo, rlo)
    assert np.all(dst[:, nK:] == 7)


def test_batch_reduce_file_against_the_host_emulated_library():
    """tests/test_gpu_batch_reduce_fused.py (backend-neutral) on the CPU build of the whole library, minus the H100-only cases"""
    assert _run_gpu_files(["test_gpu_batch_reduce_fused.py"], [], 2400) >= 105
