"""GPU: every fp32 entry in every operand class, on data where reading another row's, column's or problem's scale word, aux or
operand moves an element by orders of magnitude (the same file runs against the host-emulated library in the CPU suite,
tests/test_emulated_operand_classes.py, which also pins the case table).

Operand classes are the preparation routes of capi.cu: classify() -> K-major ("K"), MN-major ("MN") or general ("G") for a
single product; a batch adds own, shared (stride 0), negative and misaligned-gap batch strides; a convolution reads its images
or gradients in place (1 x 1) or through window gathers; a pre-pack gathers first.

Data.  Signed U(-1, 1), every row of A, column of B, problem of a batch and image, channel and spatial row of a convolution at
its own power of two, drawn from 2^[-12, 12] so that neighbours always differ (a few f16x3 cases: 2^[-40, 40], outside fp16's
range).

Cases.  A covering design per entry: for each mode every (class of A, class of B) pair occurs; the other factors (op and aux
layout, batch stride kinds, alpha / beta with beta = 0 over a NaN C, C layout, shape at a tile edge) are cycled over the
position of a case within its mode, so that each level meets each mode.

Reference.  Tensor-core paths: the per-element bound of tests/test_gpu_error_bounds.py against float64 over the operands as
multiplied after the op (tanh / sigmoid ops add their ulps per product).  The exact path: bit-exact against the CPU oracle over
the op'd operands materialised on the host, each operation rounded on its own as split.cuh: operand_op does; with a tanh /
sigmoid op (the device's tanhf / expf) within (4 * 2^-23 + 2K * 2^-24) * sum |a||b|.  PATH_AUTO: the rule of the path
last_path() reports.  Every case also checks that nothing outside the C view changed and that a repeated call gives the same
bits.  The largest err / bound per (mode, entry, class pair) is printed at the end of the file."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, emu_budget, sync
from test_gpu_error_bounds import (C_LAYOUTS, RATIOS, at, bound_and_check, c_view, conv_ref, launches, plan, sm_count,
                                   view_index)
from test_gpu_conv_input_grad import transposed_windows
from util import embed, f32_to_bf16_bits, bf16_bits_to_f32

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200._capi import lib  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHILD = os.environ.get("LASER_B200_OPCLS_CHILD", "0") == "1"
# the CPU build runs every fourth case of each table (LASER_B200_EMU_FULL=1: all of them)
FULL = not EMU or os.environ.get("LASER_B200_EMU_FULL", "0") == "1"
PATHS = {"f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "bf16": L.PATH_BF16, "simt": L.PATH_SIMT,
         "auto": L.PATH_AUTO}
NAMES = {v: k for k, v in PATHS.items() if k != "auto"}
TC = ("f16x3", "tf32x3", "tf32x1")
K_MAJOR, MN_MAJOR, GENERAL = 0, 1, 2
CLS = ("K", "MN", "G")
f64, f32 = np.float64, np.float32
INEXACT = {"tanh": 4 * 2.0 ** -23, "sigmoid": 8 * 2.0 ** -23}   # the device's tanhf (2 ulp); expf, add, divide
AUX_OPS = ("relu_grad", "tanh_grad", "sigmoid_grad")
OPS = ("relu", "tanh", "sigmoid", "relu_grad", "tanh_grad", "sigmoid_grad")
AB = [(1.0, 0.0), (-0.5, 1.25), (2.0, -1.0), (0.75, 0.0)]
EPIS = [(r, a) for a in ("none", "relu", "tanh", "sigmoid") for r in (True, False)]


def up(x, m):
    return -(-x // m) * m


# ------------------------------------------------------------------------------------------------ data
def exps(rng, n, lo=-12, hi=12):
    """n exponents in [lo, hi], each different from the one before"""
    span = hi - lo + 1
    e0 = int(rng.integers(lo, hi + 1))
    return lo + (e0 - lo + np.concatenate([[0], np.cumsum(rng.integers(1, span, n - 1))])) % span


def signed(rng, shape, rows=False, cols=False, wide=False):
    """U(-1, 1) of `shape` (..., R, C), every row / column (of every leading index) at its own power of two (float64)"""
    lim = 40 if wide else 12
    x = rng.uniform(-1.0, 1.0, shape)
    lead = int(np.prod(shape[:-2]))
    if rows:
        x = x * (2.0 ** exps(rng, lead * shape[-2], -lim, lim)).reshape(shape[:-2] + (shape[-2], 1))
    if cols:
        x = x * (2.0 ** exps(rng, lead * shape[-1], -lim, lim)).reshape(shape[:-2] + (1, shape[-1]))
    return x


def per_problem(rng, x):
    """each problem of a (batch, R, C) array at its own power of two"""
    return x * (2.0 ** exps(rng, x.shape[0]))[:, None, None]


def aux_values(rng, op, shape):
    """an op's aux: the forward output its derivative takes (relu: any sign; tanh: (-1, 1); sigmoid: (0, 1))"""
    return rng.uniform(0.0 if op == "sigmoid_grad" else -1.0, 1.0, shape).astype(f32)


def apply_op(op, x, y=None):
    """op(x) as the library multiplies it: float32 with every operation rounded on its own, float64 for tanh / sigmoid"""
    one = f32(1)
    if op is None:
        return x
    if op == "relu":
        return np.maximum(x, f32(0))
    if op == "tanh":
        return np.tanh(x.astype(f64))
    if op == "sigmoid":
        with np.errstate(over="ignore"):
            return 1.0 / (1.0 + np.exp(-x.astype(f64)))
    if op == "relu_grad":
        return np.where(y > 0, x, f32(0))
    if op == "tanh_grad":
        return x * (one - y * y)
    assert op == "sigmoid_grad"
    return x * (y * (one - y))


def op_extra(*ops):
    return sum(INEXACT.get(o, 0.0) for o in ops)


# ------------------------------------------------------------------------------------------------ checks
def key(entry, ca, cb):
    return "%s|%s-%s" % (entry, ca, cb)


def resolved_mode(mode):
    """the path the last call took (PATH_AUTO cases assert that one was reported)"""
    if mode != "auto":
        assert NAMES[L.last_path()] == mode, (mode, L.last_path())
        return mode
    got = L.last_path()
    assert got in NAMES and got != L.PATH_BF16, got
    return NAMES[got]


def check(tag, mode, entry, got, A, B, alpha, beta=0.0, C0=None, splits=1, bias=None, act="none", extra=0.0):
    """the reference of the path `mode` for got = act(alpha A B + beta C0 + bias); A (..., M, K), B (..., K, N) after the ops"""
    if mode != "simt":
        bound_and_check(tag, mode, entry, got, A, B, alpha, beta, C0, splits, bias, act, extra)
        return
    assert bias is None and act == "none"
    lead = got.shape[:-2]
    Ab = np.broadcast_to(np.asarray(A, f32), lead + A.shape[-2:])
    Bb = np.broadcast_to(np.asarray(B, f32), lead + B.shape[-2:])
    M, K, N = Ab.shape[-2], Ab.shape[-1], Bb.shape[-1]
    want = np.zeros(lead + (M, N), f32) if beta == 0.0 else np.array(np.broadcast_to(C0, lead + (M, N)), f32)
    for i in np.ndindex(*lead):
        w = np.ascontiguousarray(want[i])
        O.gemm_strided(M, N, K, alpha, np.ascontiguousarray(Ab[i]), K, 1, np.ascontiguousarray(Bb[i]), N, 1, beta, w, N, 1)
        want[i] = w
    if extra == 0.0:
        bad = got.view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), "%s: %d elements differ from the oracle, first at %s: got %r want %r" % (
            tag, int(bad.sum()), np.argwhere(bad)[0], got[bad][0], want[bad][0])
        return
    sab = np.abs(Ab).astype(f64) @ np.abs(Bb).astype(f64)
    bnd = abs(alpha) * (4 * 2.0 ** -23 + 2 * K * 2.0 ** -24) * sab + 2.0 ** -22 * np.abs(want.astype(f64))
    err = np.abs(got.astype(f64) - want)
    assert (err <= bnd).all(), "%s: worst err / bound %.3g against the oracle" % (tag, float((err / np.maximum(bnd, 1e-300)).max()))


def run_view(M, N, clayout, beta, c0, call, bf16=False):
    """C's buffer with sentinels around the view (C0 inside, or NaN with beta = 0); call(tensor, offset, rs, cs) twice on fresh
    copies -> the view of the first; checks that nothing outside the view changed and that both calls give the same bits"""
    size, off, rs, cs = c_view(M, N, clayout)
    idx = view_index(M, N, off, rs, cs) + 1
    if bf16:
        buf = np.full(size + 2, 0xC2FA, np.uint16)
        buf[idx] = f32_to_bf16_bits(c0).reshape(M, N) if beta != 0.0 else 0x7FC0
    else:
        buf = np.full(size + 2, -7777.0, f32)
        buf[idx] = c0 if beta != 0.0 else np.nan
    mask = np.ones(buf.size, bool)
    mask[idx.reshape(-1)] = False
    outs = []
    for _ in range(2):
        tc = dev(buf.view(np.int16) if bf16 else buf)
        call(tc, off + 1, rs, cs)
        sync()
        after = tc.cpu().numpy().view(buf.dtype)
        assert np.array_equal(after[mask], buf[mask]), "written outside the C view"
        outs.append(after[idx].copy())
    assert np.array_equal(outs[0], outs[1]), "a repeated call differs"
    return bf16_bits_to_f32(outs[0]) if bf16 else outs[0]


# ------------------------------------------------------------------------------------------------ layouts and classes
GEN = ["padded", "colslice", "negrow", "negcol", "misaligned", "both2"]
AS_A = {"row": K_MAJOR, "col": MN_MAJOR}      # the class each layout name stands for (every other name: general)
AS_B = {"row": MN_MAJOR, "col": K_MAJOR}


def intended(layout, side):
    return (AS_A if side == "A" else AS_B).get(layout, GENERAL)


def classify(esz, off, s_mn, s_k):
    """the library's own classification of an operand at element `off` of a 256-byte aligned buffer"""
    import ctypes
    return lib().laser_b200_debug_classify(esz, ctypes.c_void_p(0x7f0000000000 + off * esz), s_mn, s_k)


def library_class(layout, side, R, C, esz):
    _, off, rs, cs = embed(np.zeros((R, C), np.uint16 if esz == 2 else f32), layout)
    return classify(esz, off, rs, cs) if side == "A" else classify(esz, off, cs, rs)


def class_pairs(i):
    """(layout of A, layout of B): every class pair, every layout name on either side; rotated by i"""
    def g(k):
        return GEN[(k + i) % 6]
    return ([("row", "col"), ("row", "row"), ("row", g(0)), ("col", "col"), ("col", "row"), ("col", g(1)), (g(2), "col"),
             (g(3), "row")] + [(g(k), g(k + 1 + i % 5)) for k in range(6)])


# shapes at tile edges (128 x 128 tiles, 64 / 32-element k-tiles): multiples of 8 where an operand must stay K- or MN-major
# (16 bytes of bf16), 3 mod 4 where both are general (so that `padded`, a leading dimension of C + 3, never becomes aligned)
ALIGNED = [(136, 120, 72), (120, 264, 136), (264, 136, 200), (128, 256, 64), (8, 136, 520)]
ODD = [(131, 127, 67), (255, 259, 35), (3, 131, 127)]


def strided_cases():
    out = []
    for mi, mode in enumerate(("f16x3", "tf32x3", "tf32x1", "bf16", "simt")):
        for j, (la, lb) in enumerate(class_pairs(mi)):
            gen = la in GEN and lb in GEN
            shape = (ODD if gen else ALIGNED)[j % (3 if gen else 5)]
            out.append(("strided", mode, la, lb, shape, AB[j % 4], C_LAYOUTS[(j + mi) % 4], mode == "f16x3" and j % 5 == 4))
    for j, (la, lb) in enumerate(class_pairs(2)[::2]):
        out.append(("strided", "auto", la, lb, (ALIGNED + [(264, 264, 136)])[j % 6], AB[j % 4], C_LAYOUTS[j % 4], False))
    return out


def fused_cases():
    """j = 3q + r: A in class r with op q, B in class q % 3 with op (j + 2) % 6 -- every op on either side in every class, every
    class pair twice; aux in the operand's layout or the other one, bias per row / column with each activation, in turn"""
    out = []
    for mi, mode in enumerate(TC + ("simt",)):
        for j in range(18):
            ca, cb = j % 3, (j // 3) % 3
            la = ("row", "col", GEN[(j + mi) % 6])[ca]
            lb = ("col", "row", GEN[(j + mi + 3) % 6])[cb]
            shape = ALIGNED[(j + mi) % 5]
            epi = None if mode == "simt" else EPIS[(j + mi) % 8]
            out.append(("fused", mode, la, lb, OPS[j // 3], OPS[(j + 2) % 6], j % 2 == 1, epi, shape, AB[j % 4],
                        C_LAYOUTS[(j + mi) % 4], mode == "f16x3" and j % 7 == 6))
    for j in range(6):
        out.append(("fused", "auto", ("row", "col", "both2")[j % 3], ("col", "row", "negcol")[j // 2], OPS[j], OPS[5 - j],
                    j % 2 == 0, None, (ALIGNED + [(264, 264, 136)])[j], AB[j % 4], C_LAYOUTS[j % 4], False))
    return out


# batched operands: row (K-major for A), col (MN-major for A) or general, each problem at base + b * bs
BLAYOUTS = ("row", "col", "general")
BS_KINDS = ("own", "shared", "negative", "gap")
# (op of A, op of B, aux in the other layout)
BOPS = [(None, None, False), ("relu_grad", None, False), (None, "tanh_grad", True), ("sigmoid", "sigmoid_grad", False),
        ("tanh_grad", "relu", True), ("relu", "relu_grad", False)]
BSHAPES = [((5, 136, 120, 72), (3, 120, 136, 200), (4, 8, 264, 136)), ((3, 136, 120, 75), (5, 120, 136, 43), (4, 8, 264, 133))]


def batch_cases(entry):
    """every class pair per mode with each batch-stride kind on A and on B and each op variant in turn; the batch-reduced
    product with K not a multiple of 4 (segment boundaries off the 16-byte grid)"""
    out = []
    shapes = BSHAPES[entry == "batch_reduce"]
    for mi, mode in enumerate(TC + ("simt", "auto")):
        for j in range(9 if mode == "auto" else 12):
            ca, cb = j % 3, (j // 3) % 3 if j < 9 else (j + 1) % 3
            ka, kb = BS_KINDS[(j + mi) % 4], BS_KINDS[(j // 4 + j + 1 + mi) % 4]
            out.append((entry, mode, BLAYOUTS[ca], BLAYOUTS[cb], ka, kb, BOPS[(j + mi) % 6], shapes[j % 3], AB[(j + mi) % 4],
                        C_LAYOUTS[j % 4]))
    return out


CASES = {"strided": strided_cases(), "fused": fused_cases(), "batched": batch_cases("batched"),
         "batch_reduce": batch_cases("batch_reduce")}


def subset(cases):
    return [c for i, c in enumerate(cases) if FULL or i % 4 == 0]


def cid(c):
    return "-".join(str(x).replace(" ", "") for x in c[1:4]) + "-%d" % CASES[c[0]].index(c)


def work(mode, MNK):
    return (3.0 if mode in ("f16x3", "tf32x3", "auto") else 1.0) * float(np.prod(MNK))


# ------------------------------------------------------------------------------------------------ gemm_strided
def operands(rng, M, N, K, wide=False, bf16=False):
    a = signed(rng, (M, K), rows=True, wide=wide).astype(f32)
    b = signed(rng, (K, N), cols=True, wide=wide).astype(f32)
    c0 = rng.uniform(-1.0, 1.0, (M, N)).astype(f32)
    if bf16:
        a, b, c0 = (bf16_bits_to_f32(f32_to_bf16_bits(x)).reshape(x.shape) for x in (a, b, c0))
    return a, b, c0


def placed(x, layout, bf16=False):
    """(device tensor, offset, rs, cs) of x laid out as `layout`"""
    buf, off, rs, cs = embed(f32_to_bf16_bits(x).reshape(x.shape) if bf16 else x, layout)
    return dev(buf.view(np.int16) if bf16 else buf), off, rs, cs


@pytest.mark.parametrize("case", subset(CASES["strided"]), ids=cid)
def test_strided(case):
    _, mode, la, lb, (M, N, K), (alpha, beta), clayout, wide = case
    emu_budget(work(mode, (M, N, K)))
    bf16 = mode == "bf16"
    a, b, c0 = operands(np.random.default_rng(CASES["strided"].index(case)), M, N, K, wide, bf16)
    ta, oa, rsa, csa = placed(a, la, bf16)
    tb, ob, rsb, csb = placed(b, lb, bf16)
    name = "bf16" if bf16 else "f32"
    got = run_view(M, N, clayout, beta, c0, lambda tc, oc, rsc, csc: L.gemm_strided(
        M, N, K, alpha, at(ta, oa, name), rsa, csa, at(tb, ob, name), rsb, csb, beta, at(tc, oc, name), rsc, csc,
        path=PATHS[mode]), bf16)
    m = resolved_mode(mode)
    tag = "strided %s A=%s B=%s M=%d N=%d K=%d C=%s" % (mode, la, lb, M, N, K, clayout)
    check(tag, m, key("strided", CLS[intended(la, "A")], CLS[intended(lb, "B")]), got, a, b, alpha, beta, c0,
          plan(m, M, N, K)[0] if m != "simt" else 1)


# ------------------------------------------------------------------------------------------------ gemm_strided_fused
def other(layout):
    return "col" if layout == "row" else "row"


def fused_run(case, K=None, seed=None):
    """-> (launches, C, A and B after the ops, C0, bias broadcast or None, extra per-product error)"""
    _, mode, la, lb, op_a, op_b, aux_other, epi, (M, N, K0), (alpha, beta), clayout, wide = case
    K = K0 if K is None else K
    rng = np.random.default_rng(CASES["fused"].index(case) if seed is None else seed)
    a, b, c0 = operands(rng, M, N, K, wide)
    ya, yb = aux_values(rng, op_a, (M, K)), aux_values(rng, op_b, (K, N))
    bias = signed(rng, (1, M if epi and epi[0] else N)).astype(f32)[0]
    ta, oa, rsa, csa = placed(a, la)
    tb, ob, rsb, csb = placed(b, lb)
    keep = []                                    # the aux tensors, alive until the calls are done

    def spec(op, y, layout):
        if op not in AUX_OPS:
            return op
        t, o, rs, cs = placed(y, other(layout) if aux_other else layout)
        keep.append(t)
        return (op, at(t, o), rs, cs)
    sa, sb = spec(op_a, ya, la), spec(op_b, yb, lb)
    kw = {}
    if epi is not None:
        kw = dict(bias=dev(bias), bias_per_row=epi[0], activation=epi[1])
    out = {}
    n = launches(lambda: out.__setitem__("c", run_view(M, N, clayout, beta, c0, lambda tc, oc, rsc, csc: L.gemm_strided_fused(
        M, N, K, alpha, at(ta, oa), rsa, csa, at(tb, ob), rsb, csb, beta, at(tc, oc), rsc, csc, path=PATHS[mode], op_a=sa,
        op_b=sb, **kw))))
    A, B = apply_op(op_a, a, ya), apply_op(op_b, b, yb)
    bb = None
    if epi is not None:
        bb = np.broadcast_to((bias[:, None] if epi[0] else bias[None, :]).astype(f64), (M, N))
    return n // 2, out["c"], A, B, c0, bb, op_extra(op_a, op_b)


@pytest.mark.parametrize("case", subset(CASES["fused"]), ids=cid)
def test_fused(case):
    _, mode, la, lb, op_a, op_b, _, epi, (M, N, K), (alpha, beta), clayout, _ = case
    emu_budget(work(mode, (M, N, K)))
    _, got, A, B, c0, bias, extra = fused_run(case)
    m = resolved_mode(mode)
    tag = "fused %s A=%s:%s B=%s:%s epi=%s M=%d N=%d K=%d C=%s" % (mode, la, op_a, lb, op_b, epi, M, N, K, clayout)
    check(tag, m, key("fused", CLS[intended(la, "A")], CLS[intended(lb, "B")]), got, A, B, alpha, beta, c0,
          plan(m, M, N, K)[0] if m != "simt" else 1, bias, epi[1] if epi else "none", extra)


# ------------------------------------------------------------------------------------------------ batched operands
def stack_strides(layout, R, C):
    """(rs, cs, span of one problem) of an R x C matrix of a batch laid out as `layout`"""
    rs, cs = {"row": (up(C, 4), 1), "col": (1, up(R, 4)), "general": (2 * C, 2)}[layout]
    return rs, cs, (C * cs if layout == "col" else R * rs)


class Stack:
    """a batch of R x C matrices x (one matrix: shared) in one buffer, problem b's element (i, j) at base + b * bs + i * rs +
    j * cs; rows padded to 16 bytes, a gap of 5 floats (misaligned problems) for `gap`, stored last to first for `negative`"""

    def __init__(self, x, layout, kind):
        n, R, C = x.shape
        rs, cs, span = stack_strides(layout, R, C)
        self.rs, self.cs = rs, cs
        self.bs = {"own": span, "shared": 0, "negative": -(span + 4), "gap": span + 5}[kind]
        assert (n == 1) == (kind == "shared")
        per = abs(self.bs) or span
        buf = np.full(n * per + 8, 1.0e6, f32)
        self.base = (n - 1) * per if kind == "negative" else 0
        i, j = np.arange(R)[:, None], np.arange(C)[None, :]
        for b in range(n):
            buf[self.base + b * self.bs + i * rs + j * cs] = x[b]
        self.t = dev(buf)

    def ptr(self):
        return at(self.t, self.base)


def batch_data(rng, case, K=None):
    entry, mode, la, lb, ka, kb, (op_a, op_b, aux_other), (batch, M, N, K0), _, _ = case
    K = K0 if K is None else K
    na, nb = (1 if ka == "shared" else batch), (1 if kb == "shared" else batch)
    a = per_problem(rng, signed(rng, (na, M, K), rows=True)).astype(f32)
    b = per_problem(rng, signed(rng, (nb, K, N), cols=True)).astype(f32)
    ya, yb = aux_values(rng, op_a, (batch, M, K)), aux_values(rng, op_b, (batch, K, N))
    sa, sb = Stack(a, la, ka), Stack(b, lb, kb)

    def spec(op, y, layout, s):
        if op not in AUX_OPS:
            return op
        s.aux = Stack(y, other(layout) if aux_other else layout, "own")     # alive as long as the operand
        return (op, s.aux.ptr(), s.aux.rs, s.aux.cs, s.aux.bs)
    A = np.broadcast_to(apply_op(op_a, a, ya if op_a in AUX_OPS else None), (batch, M, K))
    B = np.broadcast_to(apply_op(op_b, b, yb if op_b in AUX_OPS else None), (batch, K, N))
    return sa, sb, spec(op_a, ya, la, sa), spec(op_b, yb, lb, sb), A, B, op_extra(op_a, op_b)


def batched_run(case, K=None, seed=None):
    """-> (launches of one call, C (batch, M, N), A, B after the ops, C0, extra)"""
    _, mode, la, lb, ka, kb, _, (batch, M, N, K0), (alpha, beta), clayout = case
    K = K0 if K is None else K
    rng = np.random.default_rng(1000 + CASES["batched"].index(case) if seed is None else seed)
    sa, sb, opa, opb, A, B, extra = batch_data(rng, case, K)
    ldc = N + 1 + C_LAYOUTS.index(clayout)
    bsc = M * ldc + 3
    c0 = rng.uniform(-1.0, 1.0, (batch, M, N)).astype(f32)
    buf = np.full(batch * bsc + 2, -7777.0, f32)
    idx = 1 + np.arange(batch)[:, None, None] * bsc + np.arange(M)[None, :, None] * ldc + np.arange(N)[None, None, :]
    buf[idx] = c0 if beta != 0.0 else np.nan
    mask = np.ones(buf.size, bool)
    mask[idx.reshape(-1)] = False
    outs = []
    n = 0
    for _ in range(2):
        tc = dev(buf)
        n = launches(lambda: L.gemm_strided_batched_fused(batch, M, N, K, alpha, sa.ptr(), sa.rs, sa.cs, sa.bs, sb.ptr(), sb.rs,
                                                          sb.cs, sb.bs, beta, at(tc, 1), ldc, 1, bsc, path=PATHS[mode],
                                                          op_a=opa, op_b=opb))
        after = tc.cpu().numpy()
        assert np.array_equal(after[mask].view(np.uint32), buf[mask].view(np.uint32)), "written outside the problems' C views"
        outs.append(after[idx].copy())
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "a repeated call differs"
    return n, outs[0], A, B, c0, extra


@pytest.mark.parametrize("case", subset(CASES["batched"]), ids=cid)
def test_batched(case):
    _, mode, la, lb, ka, kb, ops, (batch, M, N, K), (alpha, beta), _ = case
    emu_budget(work(mode, (batch, M, N, K)))
    _, got, A, B, c0, extra = batched_run(case)
    m = resolved_mode(mode)
    tag = "batched %s A=%s/%s B=%s/%s ops=%s batch=%d M=%d N=%d K=%d" % (mode, la, ka, lb, kb, ops, batch, M, N, K)
    check(tag, m, key("batched", la, lb), got, A, B, alpha, beta, c0, plan(m, M, N, K, batch)[0] if m != "simt" else 1,
          extra=extra)


def reduce_run(case, K=None, seed=None):
    """-> (launches of one call, C, A^ and B^ (the op'd problems concatenated along k), C0, extra)"""
    _, mode, la, lb, ka, kb, _, (batch, M, N, K0), (alpha, beta), clayout = case
    K = K0 if K is None else K
    rng = np.random.default_rng(2000 + CASES["batch_reduce"].index(case) if seed is None else seed)
    sa, sb, opa, opb, A, B, extra = batch_data(rng, case, K)
    c0 = rng.uniform(-1.0, 1.0, (M, N)).astype(f32)
    out = {}
    n = launches(lambda: out.__setitem__("c", run_view(M, N, clayout, beta, c0, lambda tc, oc, rsc, csc:
                                         L.gemm_strided_batch_reduce_fused(batch, M, N, K, alpha, sa.ptr(), sa.rs, sa.cs, sa.bs,
                                                                           sb.ptr(), sb.rs, sb.cs, sb.bs, beta, at(tc, oc),
                                                                           rsc, csc, path=PATHS[mode], op_a=opa, op_b=opb))))
    return n // 2, out["c"], np.concatenate(list(A), axis=1), np.concatenate(list(B), axis=0), c0, extra


@pytest.mark.parametrize("case", subset(CASES["batch_reduce"]), ids=cid)
def test_batch_reduce(case):
    _, mode, la, lb, ka, kb, ops, (batch, M, N, K), (alpha, beta), clayout = case
    emu_budget(work(mode, (batch, M, N, K)))
    _, got, A, B, c0, extra = reduce_run(case)
    m = resolved_mode(mode)
    tag = "batch_reduce %s A=%s/%s B=%s/%s ops=%s batch=%d M=%d N=%d K=%d C=%s" % (mode, la, ka, lb, kb, ops, batch, M, N, K,
                                                                                   clayout)
    check(tag, m, key("batch_reduce", la, lb), got, A, B, alpha, beta, c0, plan(m, M, N, batch * K)[0] if m != "simt" else 1,
          extra=extra)


# ------------------------------------------------------------------------------------------------ split-K classes
def split_cases():
    """cases of each entry whose plan splits K over few output tiles (every tile split)"""
    out = []
    for mi, mode in enumerate(("f16x3", "tf32x3")):
        for j, (la, lb) in enumerate((("col", "row"), ("padded", "col"))):
            out.append(("strided", mode, la, lb, (200, 104, 1536), AB[j + mi], C_LAYOUTS[j + 2 * mi], False))
            out.append(("fused", mode, la, lb, OPS[j + 3 * mi], OPS[5 - j], j == 1, (True, "relu"), (200, 104, 1536), AB[j + mi],
                        C_LAYOUTS[j], False))
            out.append(("batched", mode, BLAYOUTS[j + mi], BLAYOUTS[2 - j], BS_KINDS[j + 2 * mi], BS_KINDS[3 - j], BOPS[j + 1],
                        (2, 104, 96, 1536), AB[j], "even"))
            out.append(("batch_reduce", mode, BLAYOUTS[j], BLAYOUTS[1 + mi], BS_KINDS[2 * j + mi], BS_KINDS[j], BOPS[2 * j + mi],
                        (6, 104, 96, 259), AB[j], C_LAYOUTS[mi + j]))
    return out


@pytest.mark.parametrize("case", split_cases(), ids=lambda c: "%s-%s-%s-%s" % c[:4])
def test_split_k_classes(case):
    """the plan splits K: the call launches exactly one reduce kernel more than the same call at a K that never splits, with
    K's alignment kept (which decides whether an operand is read in place), and meets its path's rule"""
    entry, mode = case[0], case[1]
    if entry in ("strided", "fused"):
        M, N, K = case[4] if entry == "strided" else case[8]
        batch, Kp = 1, K
    else:
        batch, M, N, K = case[7]
        Kp = batch * K if entry == "batch_reduce" else K
    emu_budget(work(mode, (batch, M, N, K)))
    ks, nd = plan(mode, M, N, Kp, 1 if entry == "batch_reduce" else batch)
    assert ks >= 2 and nd == 0, (case, ks, nd)
    small = (64 + K % 64) if entry != "batch_reduce" else 4 + K % 4
    if entry == "strided":
        (alpha, beta), clayout = case[5], case[6]

        def one(k):
            a, b, c0 = operands(np.random.default_rng(3), M, N, k)
            ta, oa, rsa, csa = placed(a, case[2])
            tb, ob, rsb, csb = placed(b, case[3])
            out = {}
            n = launches(lambda: out.__setitem__("c", run_view(M, N, clayout, beta, c0, lambda tc, oc, rsc, csc: L.gemm_strided(
                M, N, k, alpha, at(ta, oa), rsa, csa, at(tb, ob), rsb, csb, beta, at(tc, oc), rsc, csc, path=PATHS[mode]))))
            return n // 2, out["c"], a, b, c0, None, 0.0
        n, got, A, B, c0, bias, extra = one(K)
        base = one(small)[0]
        act = "none"
    elif entry == "fused":
        n, got, A, B, c0, bias, extra = fused_run(case, seed=3)
        base = fused_run(case, K=small, seed=5)[0]
        (alpha, beta), act = case[9], case[7][1]
    else:
        runner = batched_run if entry == "batched" else reduce_run
        n, got, A, B, c0, extra = runner(case, seed=3)
        base = runner(case, K=small, seed=5)[0]
        bias, (alpha, beta), act = None, case[8], "none"
    if not CHILD:       # (under the 1 MB workspace cap of the child the batches run in more chunks: more launches)
        assert n == base + 1, (n, base, ks)
    check("split %s" % (case[:4],), mode, key(entry + "_split", case[2], case[3]), got, A, B, alpha, beta, c0, ks, bias, act,
          extra)


# ------------------------------------------------------------------------------------------------ pre-packs, host pointers
PACK_CASES = [("packed", "col", "colslice", (136, 120, 200)), ("packed", "negrow", "misaligned", (131, 127, 67)),
              ("packed", "misaligned", "negrow", (264, 136, 72)), ("packed", "colslice", "col", (8, 264, 136)),
              ("packedB", "col", "colslice", (120, 136, 520)), ("packedB", "row", "negrow", (131, 259, 35)),
              ("packedB", "misaligned", "misaligned", (255, 127, 129)), ("packedB", "negrow", "col", (128, 256, 64))]


@pytest.mark.parametrize("case", PACK_CASES, ids=lambda c: "%s-%s-%s" % c[:3])
def test_prepacked(case):
    """pre-packs of column-major, every-other-column, bottom-up and misaligned operands, gathered before the row pass"""
    entry, la, lb, (M, N, K) = case
    i = PACK_CASES.index(case)
    alpha, beta = AB[i % 4]
    a, b, c0 = operands(np.random.default_rng(3000 + i), M, N, K, wide=i % 4 == 3)
    ta, oa, rsa, csa = placed(a, la)
    tb, ob, rsb, csb = placed(b, lb)
    pa = L.alloc_packed(L.gemm_prepackA_mem_required(M, N, K))
    pb = L.alloc_packed(L.gemm_prepackB_mem_required(M, N, K))
    L.gemm_prepackA(pa, M, N, K, at(ta, oa), rsa, csa)
    L.gemm_prepackB(pb, M, N, K, at(tb, ob), rsb, csb)
    sync()

    def call(tc, oc, rsc, csc):
        if entry == "packed":
            L.gemm_packed(M, N, K, alpha, pa, pb, beta, at(tc, oc), rsc, csc)
        else:
            L.gemm_packedB(M, N, K, alpha, at(ta, oa), rsa, csa, pb, beta, at(tc, oc), rsc, csc)
    got = run_view(M, N, C_LAYOUTS[i % 4], beta, c0, call)
    check("%s A=%s B=%s M=%d N=%d K=%d" % (case[:3] + case[3]), "f16x3", key(entry, la, lb), got, a, b, alpha, beta, c0,
          plan("f16x3", M, N, K)[0])


HOST_CASES = [("f16x3", "row", "col", "padded", (300, 136, 72)), ("f16x3", "padded", "row", "row", (2100, 136, 72)),
              ("tf32x3", "row", "negcol", "negrow", (2100, 120, 136)), ("f16x3", "negrow", "row", "padded", (2049, 136, 200)),
              ("tf32x3", "col", "colslice", "col", (264, 136, 200))]


@pytest.mark.parametrize("case", HOST_CASES, ids=lambda c: "%s-%s-%s-M%d" % (c[:3] + (c[4][0],)))
def test_host_pointer_entry(case):
    """host buffers: the plain path and the pipelined one (M >= 2048, the last row panel shorter than a tile), every row of A
    at its own scale across the panels; the fp32 mode set with set_f32_mode"""
    mode, la, lb, lc, (M, N, K) = case
    emu_budget(work(mode, (M, N, K)))
    i = HOST_CASES.index(case)
    alpha, beta = AB[i % 4]
    a, b, c0 = operands(np.random.default_rng(4000 + i), M, N, K)
    ba, oa, rsa, csa = embed(a, la)
    bb, ob, rsb, csb = embed(b, lb)
    old = L.get_f32_mode()
    L.set_f32_mode(PATHS[mode])
    try:
        outs = []
        for _ in range(2):
            bc, oc, rsc, csc = embed(c0 if beta != 0.0 else np.full((M, N), np.nan, f32), lc)
            before = bc.copy()
            L.gemm_strided(M, N, K, alpha, ba[oa:], rsa, csa, bb[ob:], rsb, csb, beta, bc[oc:], rsc, csc)
            assert L.last_path() == PATHS[mode]
            idx = oc + np.arange(M)[:, None] * rsc + np.arange(N)[None, :] * csc
            mask = np.ones(bc.size, bool)
            mask[idx.reshape(-1)] = False
            assert np.array_equal(bc[mask], before[mask]), "written outside the C view"
            outs.append(bc[idx].copy())
    finally:
        L.set_f32_mode(old)
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "a repeated call differs"
    check("host %s A=%s B=%s C=%s M=%d N=%d K=%d" % (case[:4] + case[4]), mode, key("host", la, lb), outs[0], a, b, alpha, beta,
          c0, plan(mode, M, N, K)[0])


# ------------------------------------------------------------------------------------------------ convolutions
def conv_data(rng, ishape, kshape):
    """images scaled per image, input channel and spatial row; filters per output and input channel"""
    n, C, H, W = ishape
    x = rng.uniform(-1.0, 1.0, ishape) * (2.0 ** exps(rng, n))[:, None, None, None] * \
        (2.0 ** exps(rng, C))[None, :, None, None] * (2.0 ** exps(rng, H))[None, None, :, None]
    w = rng.uniform(-1.0, 1.0, kshape) * (2.0 ** exps(rng, kshape[0]))[:, None, None, None] * \
        (2.0 ** exps(rng, kshape[1]))[None, :, None, None]
    return x.astype(f32), w.astype(f32)


CONV = {"3x3_pad1_stride2": (((2, 8, 9, 9), (12, 8, 3, 3)) if EMU else ((4, 32, 15, 15), (48, 32, 3, 3)), (1, 1), (2, 2)),
        "1x1_in_place": (((2, 12, 4, 4), (8, 12, 1, 1)) if EMU else ((4, 40, 12, 12), (48, 40, 1, 1)), (0, 0), (1, 1)),
        "3x3_pad1_stride1": (((2, 6, 7, 7), (8, 6, 3, 3)) if EMU else ((3, 24, 14, 14), (40, 24, 3, 3)), (1, 1), (1, 1)),
        "3x3_stride2_tail": (((2, 4, 8, 8), (8, 4, 3, 3)) if EMU else ((5, 24, 8, 8), (40, 24, 3, 3)), (0, 0), (2, 2))}
CONV_CASES = ([("conv2d_fused", mode, g, act) for i, mode in enumerate(TC) for g, act in
               (("3x3_pad1_stride2", ("relu", "tanh", "sigmoid")[i]), ("1x1_in_place", ("none", "sigmoid", "relu")[i]))] +
              [("filter_grad", mode, g, op) for i, mode in enumerate(TC) for g, op in
               (("3x3_pad1_stride1", ("relu_grad", None, "relu_grad")[i]), ("1x1_in_place", ("relu_grad", "relu_grad", None)[i]))] +
              [("input_grad", mode, g, op) for i, mode in enumerate(TC) for g, op in
               (("3x3_pad1_stride1", (None, "relu_grad", "sigmoid_grad")[i]), ("3x3_stride2_tail", ("tanh_grad", None, "relu_grad")[i]),
                ("1x1_in_place", ("sigmoid_grad", "tanh_grad", None)[i]))])


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "%s-%s-%s-%s" % c)
def test_convolution(case):
    entry, mode, geom, var = case
    (ishape, kshape), padding, strides = CONV[geom]
    i = CONV_CASES.index(case)
    rng = np.random.default_rng(5000 + i)
    x, w = conv_data(rng, ishape, kshape)
    oshape = tuple(L.conv2d_out_shape(ishape, kshape, padding, strides))
    n, C = ishape[:2]
    co, P, Kc = kshape[0], oshape[2] * oshape[3], int(np.prod(kshape[1:]))
    emu_budget(3.0 * n * co * P * Kc)
    b_img, a_mat = conv_ref(x, w, padding, strides)             # B_n = im2col(x_n) (Kc, P), A = W (co, Kc)
    alpha, beta = AB[i % 4]
    outs = []
    if entry == "conv2d_fused":
        bias = signed(rng, (1, co)).astype(f32)[0]
        for _ in range(2):
            out = dev(np.full(n * co * P, np.nan, f32))
            L.conv2d_fused(out, dev(x), ishape, dev(w), kshape, padding, strides, bias=dev(bias), activation=var, path=PATHS[mode])
            sync()
            outs.append(out.cpu().numpy().reshape(n, co, P).copy())
        ks = plan(mode, co, P, Kc, n)[0]
        args = (np.broadcast_to(a_mat, (n,) + a_mat.shape), b_img, 1.0, 0.0, None, ks,
                np.broadcast_to(bias.astype(f64)[None, :, None], (n, co, P)), var)
    else:
        dy = (signed(rng, (n, co, P), rows=True) * (2.0 ** exps(rng, n))[:, None, None] *
              np.repeat(2.0 ** exps(rng, oshape[2]), oshape[3])[None, None, :]).astype(f32)
        y = aux_values(rng, var, dy.shape)
        g = apply_op(var, dy, y)
        if entry == "filter_grad":
            c0 = rng.uniform(-1.0, 1.0, (co, Kc)).astype(f32)
            for _ in range(2):
                dw = dev(c0 if beta != 0.0 else np.full((co, Kc), np.nan, f32))
                L.conv2d_filter_grad_fused(dw, dev(x), ishape, dev(dy), kshape, padding, strides, alpha, beta, op=var,
                                           aux=dev(y) if var else None, path=PATHS[mode])
                sync()
                outs.append(dw.cpu().numpy().reshape(co, Kc).copy())
            A, B = np.concatenate(list(g), axis=1), np.concatenate([bi.T for bi in b_img], axis=0)
            args = (A, B, alpha, beta, c0, plan(mode, co, Kc, n * P)[0], None, "none")
        else:
            c0 = rng.uniform(-1.0, 1.0, (n, C, ishape[2] * ishape[3])).astype(f32)
            for _ in range(2):
                dx = dev(c0 if beta != 0.0 else np.full(c0.shape, np.nan, f32))
                L.conv2d_input_grad_fused(dx, ishape, dev(dy), dev(w), kshape, padding, strides, alpha, beta, op=var,
                                          aux=dev(y) if var else None, path=PATHS[mode])
                sync()
                outs.append(dx.cpu().numpy().reshape(c0.shape).copy())
            kH, kW = kshape[2:]
            A = np.ascontiguousarray(w[:, :, ::-1, ::-1].transpose(1, 0, 2, 3)).reshape(C, co * kH * kW)
            B = transposed_windows(np.asarray(g, f64).reshape(oshape), ishape, kshape, padding, strides).transpose(0, 2, 1)
            args = (np.broadcast_to(A, (n,) + A.shape), B, alpha, beta, c0, plan(mode, C, c0.shape[2], A.shape[1], n)[0], None,
                    "none")
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "a repeated call differs"
    A, B, alpha, beta, c0, ks, bias, act = args
    bound_and_check("%s %s %s %s splits=%d" % (case + (ks,)), mode, key(entry, geom, var), outs[0], A, B, alpha, beta, c0, ks,
                    bias, act, op_extra(var))


# ------------------------------------------------------------------------------------------------ chunks, report
@pytest.mark.skipif(CHILD, reason="runs in the parent process only")
def test_batched_and_convolution_cases_in_1mb_workspace_chunks():
    """a 1 MB workspace cap splits the batches and images into chunks: the chunk offsets of data, aux and scale words cross
    the scaled problems, and every case still meets its rule"""
    e = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), LASER_B200_OPCLS_CHILD="1", LASER_B200_BATCH_WS_MB="1")
    sel = "batched or batch_reduce or convolution" + ("" if FULL else " and not auto and not simt")
    out = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_operand_classes.py"), "-m", "gpu", "-q",
                          "-p", "no:cacheprovider", "-k", sel], cwd=ROOT, env=e, capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and " passed" in out.stdout and "failed" not in out.stdout, out.stdout[-3000:] + out.stderr[-2000:]


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode, entry and class pair of this run (the last test of the file)"""
    mine = {k: v for k, v in RATIOS.items() if "|" in k[1]}
    if not mine:
        pytest.skip("no case ran")
    lines = ["largest err / bound per operand class pair on %d SMs (%s):" % (sm_count(), "host-emulated library" if EMU else "device")]
    for (mode, entry), r in sorted(mine.items()):
        lines.append("  %-7s %-44s %.3g" % (mode, entry, r))
    with capsys.disabled():
        print("\n" + "\n".join(lines))
