"""CPU-only: the operand-preparation kernels of laser_b200/csrc/split.cuh (hi/lo split of
TMA-addressable operands, gather of general-stride operands -- the descendant of the reference's
pack_A_mc_kc / pack_B_kc_nc, gemm_packing.nim:24-94 --, the deterministic split-K reduction and the
synthetic-input generator) executed on host threads (tests/emu/) against numpy restatements."""
import ctypes

import numpy as np
import pytest

import oracle as O
from emu_build import build_emu
from util import bf16_bits_to_f32, f32_to_bf16_bits

i64, vp, ci, f32 = ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_float


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(build_emu("split_emu", ["split.cuh", "f16_scale.cuh"]))
    L.emu_split_rows_tf32.argtypes = [vp, i64, i64, i64, vp, vp, i64, ci]
    L.emu_f16x2_rows_fused.argtypes = [ci, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_f16x2_rows_ring.argtypes = [vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_f16x2_rows_ring.restype = ci
    L.emu_absmax_mn.argtypes = [ci, vp, i64, i64, i64, vp, ci]
    L.emu_split_rows_f16x2.argtypes = [ci, vp, i64, i64, i64, vp, vp, i64, vp, ci]
    L.emu_pack_general_f32.argtypes = [ci, vp, i64, i64, i64, i64, vp, vp, i64, ci, ci]
    L.emu_pack_general_u16.argtypes = [vp, i64, i64, i64, i64, vp, i64, ci, ci]
    L.emu_splitk_tail_reduce.argtypes = [vp, ci, ci, ci, ci, ci, ci, ci, i64, i64, f32, f32, vp, i64, i64, vp, ci, ci, ci]
    L.emu_fill_uniform_f32.argtypes = [vp, i64, ctypes.c_uint64, f32, f32, ci]
    for n in ("emu_split_rows_tf32", "emu_f16x2_rows_fused", "emu_absmax_mn", "emu_split_rows_f16x2", "emu_pack_general_f32", "emu_pack_general_u16",
              "emu_splitk_tail_reduce", "emu_fill_uniform_f32"):
        getattr(L, n).restype = None
    return L


def p(a, off=0):
    return ctypes.c_void_p(a.ctypes.data + off * a.itemsize)


def tf32_rna(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def test_fill_uniform_matches_the_oracle_generator(emu):
    n = 10007
    out = np.zeros(n, np.float32)
    emu.emu_fill_uniform_f32(p(out), n, 42, -0.1, 0.1, 5)
    assert np.array_equal(out, O.fill_uniform_f32(n, 42, -0.1, 0.1))


@pytest.mark.parametrize("R,Cc,src_ld", [(5, 16, 16), (33, 30, 32), (7, 1, 4), (130, 257, 260)])
def test_split_rows(emu, R, Cc, src_ld):
    rng = np.random.default_rng(0)
    src = (rng.standard_normal((R, src_ld)) * 3).astype(np.float32)
    ld = -(-Cc // 4) * 4; ldb = -(-Cc // 8) * 8
    x = src[:, :Cc]
    h = tf32_rna(x)
    hi = np.full((R, ld), 9, np.float32); lo = np.full((R, ld), 9, np.float32)
    emu.emu_split_rows_tf32(p(src), R, Cc, src_ld, p(hi), p(lo), ld, 3)
    assert np.array_equal(hi[:, :Cc], h) and np.array_equal(lo[:, :Cc], tf32_rna(x - h))
    assert np.all(hi[:, Cc:] == 0) and np.all(lo[:, Cc:] == 0)        # k padding is zero (it feeds the MMA)
    assert np.abs((hi[:, :Cc].astype(np.float64) + lo[:, :Cc]) - x).max() <= 2.0 ** -21 * np.abs(x).max()


@pytest.mark.parametrize("R,Cc,src_ld", [(5, 16, 16), (33, 30, 32), (130, 257, 260), (70, 2100, 2100), (11, 8192, 8196), (300, 2300, 2304)])
@pytest.mark.parametrize("per_col", [0, 1])
def test_f16x2_scale_and_split(emu, R, Cc, src_ld, per_col):
    """LASER_B200_PATH_F16X3: one abs-max word per row (K-major operand) or per column (MN-major operand), a power-of-two
    scale per word putting that maximum into [2^14, 2^15), two fp16 pieces (numpy's float16 is IEEE binary16 with
    round-to-nearest-even, the conversion the kernel's software twin restates).  The rows / columns differ by up to
    2^+-60 in magnitude; one of them is all zero."""
    rng = np.random.default_rng(3)
    src = rng.standard_normal((R, src_ld)).astype(np.float32)
    n_mn = Cc if per_col else R
    mags = (2.0 ** rng.integers(-60, 60, n_mn)).astype(np.float32)
    mags[n_mn // 2] = 0.0
    src[:, :Cc] *= mags[None, :] if per_col else mags[:, None]
    src[0, 0] = np.inf; src[R - 1, Cc - 1] = np.nan          # non-finite entries must not set a scale
    src[:, Cc:] = 1e30                                        # nor may anything outside the view
    x = src[:, :Cc]
    words = np.zeros(n_mn, np.uint32)
    emu.emu_absmax_mn(per_col, p(src), R, Cc, src_ld, p(words), 3)
    want = np.where(np.isfinite(x), np.abs(x), 0).max(axis=0 if per_col else 1).astype(np.float32)
    assert np.array_equal(words, want.view(np.uint32))
    e = (words >> 23).astype(np.int64)
    s_exp = np.where(e == 0, 0, np.clip(14 - (e - 127), -126, 126))
    scale = (2.0 ** s_exp).astype(np.float32)
    ldb = -(-Cc // 8) * 8; ld = -(-Cc // 4) * 4
    hb = np.full((R, ldb), 9, np.uint16); lb = np.full((R, ldb), 9, np.uint16)
    emu.emu_split_rows_f16x2(per_col, p(src), R, Cc, src_ld, p(hb), p(lb), ldb, p(words), 2)
    with np.errstate(invalid="ignore", over="ignore"):
        xs = x * (scale[None, :] if per_col else scale[:, None])
        h = xs.astype(np.float16); l = (xs - h.astype(np.float32)).astype(np.float16)
    ok = np.isfinite(x)
    assert np.array_equal(hb[:, :Cc][ok], h.view(np.uint16)[ok]) and np.array_equal(lb[:, :Cc][ok], l.view(np.uint16)[ok])
    assert np.all(hb[:, Cc:ld] == 0) and np.all(lb[:, Cc:ld] == 0)
    assert np.all(lb[:, :Cc][~ok] == 0)            # non-finite entries: the low piece is 0 (x - h would be NaN)
    if not per_col:                                 # the fused single-pass kernel (the path K-major operands take)
        for group, grid in ((32, 2), (256, 3)):
            w2 = np.full(n_mn, 77, np.uint32); hb2 = np.full((R, ldb), 9, np.uint16); lb2 = np.full((R, ldb), 9, np.uint16)
            emu.emu_f16x2_rows_fused(group, p(src), R, Cc, src_ld, p(hb2), p(lb2), ldb, p(w2), grid)
            assert np.array_equal(w2, words)
            assert np.array_equal(hb2[:, :ld], hb[:, :ld]) and np.array_equal(lb2[:, :ld], lb[:, :ld])
        # ... and its variant with the rows prefetched into a shared-memory ring by bulk copies (long, 16-byte aligned rows)
        w3 = np.full(n_mn, 77, np.uint32); hb3 = np.full((R, ldb), 9, np.uint16); lb3 = np.full((R, ldb), 9, np.uint16)
        ran = emu.emu_f16x2_rows_ring(p(src), R, Cc, src_ld, p(hb3), p(lb3), ldb, p(w3), 2)
        assert ran == int(Cc % 4 == 0 and src_ld % 4 == 0 and 1024 < Cc <= 8192)
        if ran:
            assert np.array_equal(w3, words)
            assert np.array_equal(hb3[:, :ld], hb[:, :ld]) and np.array_equal(lb3[:, :ld], lb[:, :ld])
    mx = np.where(ok, np.abs(xs), 0).max(axis=0 if per_col else 1)
    assert np.all((mx == 0) | ((mx >= 2.0 ** 14) & (mx < 2.0 ** 15)))
    big = ok & (np.abs(xs) >= 2.0 ** -3)           # l = xs - h (<= 2^-11 |xs|) is then rounded at or above fp16's subnormal spacing 2^-24: 22 bits
    rec = h.astype(np.float64) + l.astype(np.float64)
    assert (np.abs(rec - xs)[big] <= 2.0 ** -22 * np.abs(xs)[big]).all()
    assert (np.abs(rec - xs)[ok & ~big] <= 2.0 ** -25).all()      # everything else: absolute precision of the fp16 subnormals


@pytest.mark.parametrize("R,Cc,sr,sc,along_r", [
    (40, 50, 50, 1, 0),       # plain row-major (copy)
    (40, 50, 1, 40, 1),       # column-major source: transposing gather
    (33, 65, 130, 2, 0),      # every other column
    (20, 31, -31, 1, 0),      # rows bottom-up
    (20, 31, 31, -1, 0),      # columns right-to-left
    (70, 3, 2, 140, 1),
])
@pytest.mark.parametrize("mode", [0, 1])
def test_pack_general(emu, R, Cc, sr, sc, along_r, mode):
    lo_off = min(0, (R - 1) * sr) + min(0, (Cc - 1) * sc)
    hi_off = max(0, (R - 1) * sr) + max(0, (Cc - 1) * sc)
    rng = np.random.default_rng(1)
    buf = (rng.standard_normal(hi_off - lo_off + 1) * 2).astype(np.float32)
    idx = -lo_off + np.arange(R)[:, None] * sr + np.arange(Cc)[None, :] * sc
    x = buf[idx]
    ld = -(-Cc // 4) * 4; ldb = -(-Cc // 8) * 8
    dst = np.full((R, ld), 7, np.float32); dlo = np.full((R, ld), 7, np.float32)
    xb = np.full((R, ldb), 7, np.uint16); lb = np.full((R, ldb), 7, np.uint16)
    emu.emu_pack_general_f32(mode, p(buf, -lo_off), R, Cc, sr, sc, p(dst), p(dlo), ld, along_r, 4)
    h = tf32_rna(x)
    if mode == 0:
        assert np.array_equal(dst[:, :Cc], x)
    else:
        assert np.array_equal(dst[:, :Cc], h) and np.array_equal(dlo[:, :Cc], tf32_rna(x - h))
    assert np.all(dst[:, Cc:] == 7)      # the gather never writes the padding (the host zeroes it once)


def test_pack_general_bf16(emu):
    R, Cc, sr, sc = 37, 29, 1, 37
    buf = np.arange(R * Cc, dtype=np.uint16)
    dst = np.zeros((R, 32), np.uint16)
    emu.emu_pack_general_u16(p(buf), R, Cc, sr, sc, p(dst), 32, 1, 2)
    assert np.array_equal(dst[:, :Cc], buf.reshape(Cc, R).T)


@pytest.mark.parametrize("S,alpha,beta,per_row,act", [(1, 1.0, 0.0, 0, 0), (4, 0.5, -1.25, 0, 0), (3, 1.0, 0.0, 1, 1),
                                                      (5, 2.0, 1.0, 0, 2)])
@pytest.mark.parametrize("n_direct,tile_m", [(0, 128), (3, 256)])
def test_splitk_tail_reduce_is_a_fixed_order_sum(emu, S, alpha, beta, per_row, act, n_direct, tile_m):
    """tile-local planes [S][n_tail][tile_m][BN] (BN = TC_BLOCK_N) of the tiles n_direct.. (raster order, tc_params.h: tile_coords) -> C;
    the direct tiles of C are not touched"""
    BN = 128                                             # tc_params.h: TC_BLOCK_N
    M, N, G = 2 * tile_m + 23, BN + 37, 2               # 3 x 2 tiles, ragged in both directions
    num_m, num_n = -(-M // tile_m), -(-N // BN)
    n_tail = num_m * num_n - n_direct
    rng = np.random.default_rng(2)
    ws = rng.standard_normal((S, n_tail, tile_m, BN)).astype(np.float32)
    C = rng.standard_normal((N, M)).astype(np.float32)            # column-major C: rsC = 1, csC = M
    bias = rng.standard_normal(M if per_row else N).astype(np.float32) if act else None
    c0 = C.copy()
    emu.emu_splitk_tail_reduce(p(ws), S, n_tail, n_direct, num_m, num_n, G, tile_m, M, N, alpha, beta, p(C), 1, M,
                               p(bias) if bias is not None else None, per_row, act, 3)
    want = c0.T.copy()

    def coords(t):                                                   # tc_params.h: tile_coords
        per_group = G * num_n
        g = t // per_group
        first = g * G
        gsz = min(G, num_m - first)
        r = t - g * per_group
        return first + r % gsz, r // gsz
    seen = set()
    for ti in range(n_tail):
        mb, nb = coords(n_direct + ti)
        seen.add((mb, nb))
        r0, c0_ = mb * tile_m, nb * BN
        rows, cols = min(tile_m, M - r0), min(BN, N - c0_)
        s = ws[0, ti, :rows, :cols].copy()
        for k in range(1, S):
            s = s + ws[k, ti, :rows, :cols]                          # planes in order 0..S-1, fp32
        v = np.float32(alpha) * s
        if beta != 0.0:
            old = c0.T[r0:r0 + rows, c0_:c0_ + cols]
            v = (np.float64(beta) * old.astype(np.float64) + v.astype(np.float64)).astype(np.float32)   # fmaf
        if act:
            v = v + (bias[r0:r0 + rows, None] if per_row else bias[None, c0_:c0_ + cols])
            v = np.maximum(v, 0) if act == 1 else np.tanh(v)
        want[r0:r0 + rows, c0_:c0_ + cols] = v
    assert len(seen) == n_tail
    assert np.allclose(C.T, want, rtol=1e-6, atol=1e-6)
    if S > 1 and beta == 0.0 and not act:
        assert np.array_equal(C.T, want)
