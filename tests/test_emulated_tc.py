"""CPU-only: the wgmma GEMM kernel (laser_b200/csrc/gemm_tc.cuh) executed on host threads on top of a
functional model of the PTX it uses (tests/emu/ptx_emu.h: mbarrier, TMA boxes with zero fill, wgmma
through the shared-memory descriptors and its accumulator fragments), launched with the
library's own planning (tc_plan).  Covered: the producer / consumer / epilogue protocol of all modes (a protocol error is a
deadlock -> timeout, or a wrong sum), tile scheduler + raster, kc-blocked accumulation, split-K, ragged
M / N / K, K-major and MN-major operands, every epilogue path.  Not covered
(silicon properties, see ptx_emu.h): swizzle patterns, encodings, the accumulator's rounding."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from util import bf16_bits_to_f32, f32_to_bf16_bits

i64, vp, ci, f32 = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_float
pytestmark = pytest.mark.timeout(300)


KIND = {"tf32x1": 0, "tf32x3": 1, "bf16": 2, "f16x3": 3}


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("tc_emu", ["gemm_tc.cuh", "tc_params.h", "f16_scale.cuh", "ptx.cuh", "split.cuh"]))
    L.emu_gemm_tc.restype = ci
    L.emu_gemm_tc.argtypes = [ci, ci, ci, i64, i64, i64, f32, f32, vp, vp, i64, vp, vp, i64, vp, i64, i64, ci, ci, ci, ci,
                              vp, ci, ci, vp, i64, ctypes.POINTER(ci), ctypes.POINTER(ci), vp, vp, ci, ci]
    return L


def tf32_rna(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_trunc(x):
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def lay(x, mn_major, pad):
    """logical [mn][k] -> the stored array: K-major [mn][ld] or MN-major [k][ld]; ld a multiple of `pad`."""
    src = x.T if mn_major else x
    ld = -(-src.shape[1] // pad) * pad
    out = np.full((src.shape[0], ld), 3 if src.dtype == np.uint16 else 777.0, src.dtype)   # junk in the padding
    out[:, :src.shape[1]] = src
    return out, ld


def ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def run_tc(emu, mode, a, b, c, rsC, csC, alpha=1.0, beta=0.0, a_mn=False, b_mn=False, kc=128, raster=0,
           splitk=1, sms=4, epi=None, c_base=None, dyn=1, tail_min_k=0):
    """a: logical (M, K) fp32; b: logical (K, N) fp32; c: flat output buffer (float32, or uint16 for bf16).
    Returns (expected sum A*B in float64 under the mode's operand model, k_splits, grid); run_tc.n_direct holds the number
    of tiles the last launch computed without splitting (tc_params.h)."""
    M, K = a.shape
    N = b.shape[1]
    bt = np.ascontiguousarray(b.T)              # B seen as [n][k]
    arrs = {"A": [None] * 2, "B": [None] * 2}
    ld = {"A": 0, "B": 0}
    amax = {"A": None, "B": None}
    f = np.float64
    if mode == "f16x3":
        # two fp16 pieces of the scaled operand (split.cuh: f16x2_rows_fused_kernel / absmax_mn_kernel + split_rows_f16x2_kernel)
        def pieces(x):          # one power-of-two scale per mn index (row of x), from its abs-max word (f16_scale.cuh)
            words = np.abs(x).max(axis=1).astype(np.float32).view(np.uint32)
            e = (words >> 23).astype(np.int64)
            s_exp = np.where(e == 0, 0, np.clip(14 - (e - 127), -126, 126))
            xs = x * (2.0 ** s_exp).astype(np.float32)[:, None]
            h16 = xs.astype(np.float16); l16 = (xs - h16.astype(np.float32)).astype(np.float16)
            return h16.view(np.uint16), l16.view(np.uint16), h16.astype(f), l16.astype(f), 2.0 ** (-s_exp.astype(f)), words
        ha, la, haf, laf, ua, amax["A"] = pieces(a)
        hb, lb_, hbf, lbf, ub, amax["B"] = pieces(bt)
        arrs["A"][0], ld["A"] = lay(ha, a_mn, 8); arrs["A"][1], _ = lay(la, a_mn, 8)
        arrs["B"][0], ld["B"] = lay(hb, b_mn, 8); arrs["B"][1], _ = lay(lb_, b_mn, 8)
        exact = (haf @ lbf.T + laf @ hbf.T + haf @ hbf.T) * ua[:, None] * ub[None, :]
    elif mode == "bf16":
        ab, bb = f32_to_bf16_bits(a).reshape(M, K), f32_to_bf16_bits(bt).reshape(N, K)
        arrs["A"][0], ld["A"] = lay(ab, a_mn, 8); arrs["B"][0], ld["B"] = lay(bb, b_mn, 8)
        exact = bf16_bits_to_f32(ab).astype(np.float64) @ bf16_bits_to_f32(bb).astype(np.float64).T
    elif mode == "tf32x1":
        arrs["A"][0], ld["A"] = lay(a, a_mn, 4); arrs["B"][0], ld["B"] = lay(bt, b_mn, 4)
        exact = tf32_trunc(a).astype(np.float64) @ tf32_trunc(bt).astype(np.float64).T
    else:
        assert mode == "tf32x3"
        ha, hb = tf32_rna(a), tf32_rna(bt)
        la, lb_ = tf32_rna(a - ha), tf32_rna(bt - hb)
        arrs["A"][0], ld["A"] = lay(ha, a_mn, 4); arrs["B"][0], ld["B"] = lay(hb, b_mn, 4)
        arrs["A"][1], _ = lay(la, a_mn, 4); arrs["B"][1], _ = lay(lb_, b_mn, 4)
        exact = ha.astype(f) @ lb_.astype(f).T + la.astype(f) @ hb.astype(f).T + ha.astype(f) @ hb.astype(f).T
    bias, per_row, act = epi if epi else (None, 0, 0)
    ws = np.full(16 * (-(-M // 256) * 256) * (-(-N // 256) * 256), np.nan, np.float32)   # every tile split 16 ways fits
    ks, grid = (ci * 2)(0, 0), ci(0)
    rc = emu.emu_gemm_tc(KIND[mode], int(a_mn), int(b_mn), M, N, K, alpha, beta,
                         ptr(arrs["A"][0]), ptr(arrs["A"][1]), ld["A"], ptr(arrs["B"][0]), ptr(arrs["B"][1]), ld["B"],
                         ctypes.c_void_p(c.ctypes.data + (c_base or 0) * c.itemsize), rsC, csC, kc, raster, splitk, sms,
                         ptr(bias), per_row, act, ptr(ws), ws.size, ks, ctypes.byref(grid), ptr(amax["A"]), ptr(amax["B"]), dyn, tail_min_k)
    assert rc == 0          # (the harness runs the reduce kernel of a split launch itself, like capi.cu: tc_run)
    run_tc.n_direct = ks[1]
    return exact, ks[0], grid.value


def rnd(shape, seed, lo=-1.0, hi=1.0):
    return O.fill_uniform_f32(int(np.prod(shape)), seed, lo, hi).reshape(shape)


@pytest.mark.parametrize("mode", ["tf32x1", "tf32x3", "f16x3"])
@pytest.mark.parametrize("dyn", [0, 1])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_modes_and_majorness(emu, mode, dyn, a_mn, b_mn):
    M, N, K = 200, 300, 150                      # ragged in all three dimensions
    a, b = rnd((M, K), 1), rnd((K, N), 2)
    c = np.full(M * N + 64, -9.0, np.float32)
    exact, ks, grid = run_tc(emu, mode, a, b, c, N, 1, a_mn=a_mn, b_mn=b_mn, sms=2, dyn=dyn)
    assert ks == 1 and grid == 2                 # 6 tiles on 2 CTAs: the persistent loop iterates
    got = c[:M * N].reshape(M, N)
    assert np.abs(got - exact).max() <= 2e-6 * np.abs(exact).max()
    assert np.all(c[M * N:] == -9.0)
    if mode != "tf32x1":                         # the split operands reproduce the fp32 product
        ref = np.zeros((M, N), np.float32)
        O.gemm_strided(M, N, K, 1.0, a, K, 1, b, N, 1, 0.0, ref, N, 1)
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("layout", ["row_vec", "row_odd", "col", "strided"])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (0.5, -1.25)])
def test_epilogue_paths(emu, layout, alpha, beta):
    M, N, K = 150, 270, 70
    a, b = rnd((M, K), 3), rnd((K, N), 4)
    c0 = rnd((M, N), 5)
    if layout == "row_vec":
        rs, cs, size = N + 2, 1, M * (N + 2)     # 16-byte aligned rows: vector stores, scalar on the ragged edge
    elif layout == "row_odd":
        rs, cs, size = N + 1, 1, M * (N + 1)     # odd pitch: scalar path
    elif layout == "col":
        rs, cs, size = 1, M, M * N               # transposed C
    else:
        rs, cs, size = 2 * N, 2, 2 * M * N
    buf = np.full(size, np.nan if beta == 0.0 else -7.0, np.float32)
    idx = np.arange(M)[:, None] * rs + np.arange(N)[None, :] * cs
    if beta != 0.0:
        buf[idx] = c0
    before = buf.copy()
    exact, _, _ = run_tc(emu, "f16x3", a, b, buf, rs, cs, alpha=alpha, beta=beta, sms=4)
    want = alpha * exact + (beta * c0 if beta != 0.0 else 0.0)
    assert np.abs(buf[idx] - want).max() <= 3e-6 * max(1.0, np.abs(want).max())
    mask = np.ones(size, bool); mask[idx.reshape(-1)] = False
    assert np.array_equal(buf[mask], before[mask], equal_nan=True)   # nothing outside the view is written


@pytest.mark.parametrize("per_row,act", [(0, 1), (1, 2), (0, 3)])
def test_fused_epilogue(emu, per_row, act):
    M, N, K = 130, 260, 64
    a, b = rnd((M, K), 6), rnd((K, N), 7)
    bias = rnd((M if per_row else N,), 8)
    c = np.zeros(M * N, np.float32)
    exact, _, _ = run_tc(emu, "f16x3", a, b, c, N, 1, epi=(bias, per_row, act))
    v = exact + (bias[:, None] if per_row else bias[None, :])
    want = {1: np.maximum(v, 0), 2: np.tanh(v), 3: 1 / (1 + np.exp(-v))}[act]
    assert np.abs(c.reshape(M, N) - want).max() <= 3e-6 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("mode,kc", [("f16x3", 64), ("f16x3", 128), ("f16x3", 256), ("tf32x3", 64), ("tf32x1", 128)])
def test_accumulation_blocks_and_ragged_k(emu, mode, kc):
    M, N, K = 140, 100, 333                      # several kc blocks, the last one partial, K % 32 != 0
    a, b = rnd((M, K), 9, 0, 1), rnd((K, N), 10, 0, 1)
    c = np.zeros(M * N, np.float32)
    exact, ks, _ = run_tc(emu, mode, a, b, c, N, 1, kc=kc, sms=2)
    assert ks == 1
    assert np.abs(c.reshape(M, N) - exact).max() <= 2e-6 * np.abs(exact).max()


@pytest.mark.parametrize("M", [100, 250])
@pytest.mark.parametrize("mode", ["tf32x3", "f16x3"])
def test_split_k(emu, M, mode):
    N, K = 120, 1400                             # one or two output tiles, long K: the planner splits K over idle SMs
    a, b = rnd((M, K), 11), rnd((K, N), 12)
    c0 = rnd((M, N), 13)
    c = c0.reshape(-1).copy()
    exact, ks, grid = run_tc(emu, mode, a, b, c, N, 1, alpha=0.5, beta=2.0, kc=64, sms=8)
    assert ks >= 2 and grid == -(-M // 128) * ks
    want = 0.5 * exact + 2.0 * c0
    assert np.abs(c.reshape(M, N) - want).max() <= 3e-6 * np.abs(want).max()


@pytest.mark.parametrize("mode,dyn", [("tf32x3", 1), ("f16x3", 1), ("tf32x3", 0)])
@pytest.mark.parametrize("ccol", [False, True])
def test_split_k_of_the_last_partial_wave(emu, mode, dyn, ccol):
    """more tiles than persistent CTAs, the remainder at most half a wave: the full waves are computed directly, the
    tiles of the remainder as K-ranges through the workspace + reduce kernel (tc_params.h), alpha / beta / bias on both"""
    M, N, K = 128 + 40, 3 * 128 - 10, 1040            # 2 x 3 = 6 tiles on 4 CTAs: 4 direct, 2 split in two halves of K (>= 512 each)
    sms = 4
    a, b = rnd((M, K), 21), rnd((K, N), 22)
    c0 = rnd((M, N), 23)
    bias = rnd((N,), 24)
    buf = np.ascontiguousarray(c0.T if ccol else c0).reshape(-1).copy()
    rs, cs = (1, M) if ccol else (N, 1)
    exact, ks, grid = run_tc(emu, mode, a, b, buf, rs, cs, alpha=0.5, beta=2.0, kc=64, sms=sms, dyn=dyn,
                             epi=(bias, 0, 1), tail_min_k=256)
    assert ks == 2 and run_tc.n_direct == 4 and grid == sms
    want = np.maximum(0.5 * exact + 2.0 * c0 + bias[None, :], 0.0)
    got = buf.reshape(N, M).T if ccol else buf.reshape(M, N)
    tol = 2e-3 if mode == "tf32x1" else 3e-6
    assert np.abs(got - want).max() <= tol * np.abs(want).max()
    # without the threshold override the same problem runs unsplit (K is short)
    buf2 = np.ascontiguousarray(c0.T if ccol else c0).reshape(-1).copy()
    _, ks2, _ = run_tc(emu, mode, a, b, buf2, rs, cs, alpha=0.5, beta=2.0, kc=64, sms=sms, dyn=dyn, epi=(bias, 0, 1))
    assert ks2 == 1 and run_tc.n_direct == 6
    got2 = buf2.reshape(N, M).T if ccol else buf2.reshape(M, N)
    assert np.abs(got2 - want).max() <= tol * np.abs(want).max()


@pytest.mark.parametrize("mode", ["f16x3", "tf32x1"])
def test_padded_c_equals_compact_c(emu, mode):
    """fp32 C with a row pitch ldc > N (vector stores of column pairs, ragged rows and a ragged last column block): every
    element bit-identical to the same product into a compact C (ldc = N), the padding of C untouched, beta / bias /
    activation included"""
    M, N, K = 300, 520, 96                       # ragged rows; the last column block (8 of 128 columns) is ragged
    a, b = rnd((M, K), 31), rnd((K, N), 32)
    ldc = N + 8
    c0 = rnd((M, ldc), 33)
    bias = rnd((N,), 34)
    outs = []
    for pitch in (ldc, N):
        buf = np.ascontiguousarray(c0[:, :pitch]).reshape(-1).copy()
        exact, _, _ = run_tc(emu, mode, a, b, buf, pitch, 1, alpha=0.5, beta=2.0, sms=4, epi=(bias, 0, 1))
        outs.append(buf.reshape(M, pitch))
    assert np.array_equal(outs[0][:, :N], outs[1])
    assert np.array_equal(outs[0][:, N:], c0[:, N:])                 # the padding of C is not written
    want = np.maximum(0.5 * exact + 2.0 * c0[:, :N] + bias[None, :], 0.0)
    assert np.abs(outs[0][:, :N] - want).max() <= (2e-3 if mode == "tf32x1" else 3e-6) * np.abs(want).max()


@pytest.mark.parametrize("raster", [1, 2, 16])
def test_raster_groups_cover_every_tile_once(emu, raster):
    M, N, K = 600, 520, 32                       # 5 x 5 tiles of 128 x 128 on 4 persistent CTAs
    a, b = rnd((M, K), 14), rnd((K, N), 15)
    c = np.full(M * N, np.nan, np.float32)
    exact, _, grid = run_tc(emu, "tf32x1", a, b, c, N, 1, raster=raster, sms=4)
    assert grid == 4
    assert np.abs(c.reshape(M, N) - exact).max() <= 2e-6 * np.abs(exact).max()


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_bf16(emu, a_mn, b_mn):
    M, N, K = 200, 264, 100
    a, b = rnd((M, K), 16), rnd((K, N), 17)
    c0 = f32_to_bf16_bits(rnd((M, N), 18)).reshape(M, N)
    c = c0.reshape(-1).copy()
    exact, _, _ = run_tc(emu, "bf16", a, b, c, N, 1, alpha=1.0, beta=0.5, a_mn=a_mn, b_mn=b_mn)
    want = exact + 0.5 * bf16_bits_to_f32(c0)
    got = bf16_bits_to_f32(c.reshape(M, N))
    assert np.abs(got - want).max() <= 2.0 ** -8 * max(1.0, np.abs(want).max())


# ---- property-based: random problems / configurations against the mode's operand model -------------
from hypothesis import HealthCheck, given, settings, strategies as st  # noqa: E402


@settings(max_examples=40, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture, HealthCheck.too_slow])
@given(mode=st.sampled_from(["tf32x1", "tf32x3", "bf16", "f16x3"]), dyn=st.sampled_from([0, 1]), M=st.integers(1, 300), N=st.integers(1, 300),
       K=st.integers(1, 400), a_mn=st.booleans(), b_mn=st.booleans(),
       kc=st.sampled_from([32, 64, 128, 512]), raster=st.sampled_from([0, 1, 3]), sms=st.sampled_from([2, 4, 10]),
       splitk=st.booleans(), ccol=st.booleans(), beta=st.sampled_from([0.0, 1.0, -0.75]), seed=st.integers(0, 2**30))
def test_property_random_configurations(emu, mode, dyn, M, N, K, a_mn, b_mn, kc, raster, sms, splitk, ccol, beta, seed):
    a, b = rnd((M, K), seed), rnd((K, N), seed + 1)
    c0 = rnd((M, N), seed + 2)
    rs, cs = (1, M) if ccol else (N, 1)
    idx = np.arange(M)[:, None] * rs + np.arange(N)[None, :] * cs
    if mode == "bf16":
        c0b = f32_to_bf16_bits(c0).reshape(M, N)
        buf = np.zeros(M * N, np.uint16); buf[idx] = c0b
        exact, _, _ = run_tc(emu, mode, a, b, buf, rs, cs, beta=beta, a_mn=a_mn, b_mn=b_mn, kc=kc, raster=raster,
                             splitk=int(splitk), sms=sms, dyn=dyn)
        want = exact + beta * bf16_bits_to_f32(c0b)
        assert np.abs(bf16_bits_to_f32(buf[idx]) - want).max() <= 2.0 ** -8 * max(1.0, np.abs(want).max())
        return
    buf = np.full(M * N, np.nan, np.float32)
    if beta != 0.0:
        buf[idx] = c0
    exact, ks, _ = run_tc(emu, mode, a, b, buf, rs, cs, beta=beta, a_mn=a_mn, b_mn=b_mn, kc=kc, raster=raster,
                          splitk=int(splitk), sms=sms, dyn=dyn)
    want = exact + (beta * c0 if beta != 0.0 else 0.0)
    assert np.abs(buf[idx] - want).max() <= 4e-6 * max(1.0, np.abs(want).max()), (ks,)
