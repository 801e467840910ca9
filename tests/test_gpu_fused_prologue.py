"""GPU: fused prologue C <- act(alpha * opA(A) * opB(B) + beta * C + bias) -- an elementwise op (relu / tanh / sigmoid, or a
derivative with its aux tensor) applied to an operand while it is prepared (the reference's roadmap: fuse operations during
the prepacking, README.md:244-245).  Parity is the oracle on the op'd operands, restated step by step in float32."""
import ctypes

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, emu_budget, needs_gpu, sync

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402

OPS = ["relu", "tanh", "sigmoid", "relu_grad", "tanh_grad", "sigmoid_grad"]
PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
SHAPE = (130, 260, 150) if EMU else (300, 520, 700)     # straddles the 128-row / 128-column / 64-k tiles either way


def op_ref(name, x, y):
    """the header's formulas, float32 step by step"""
    one = np.float32(1)
    with np.errstate(all="ignore"):
        return {"relu": lambda: np.fmax(x, np.float32(0)), "tanh": lambda: np.tanh(x),
                "sigmoid": lambda: one / (one + np.exp(-x)), "relu_grad": lambda: np.where(y > 0, x, np.float32(0)),
                "tanh_grad": lambda: x * (one - y * y), "sigmoid_grad": lambda: x * (y * (one - y))}[name]().astype(np.float32)


def aux_for(name, shape, seed):
    """aux in the range each derivative sees: a signed pre-activation, a tanh output, a sigmoid output"""
    lo, hi = {"tanh_grad": (-1, 1), "sigmoid_grad": (0, 1)}.get(name, (-1, 1))
    return O.fill_uniform_f32(int(np.prod(shape)), seed, lo, hi).reshape(shape)


class Operand:
    """a logical rows x cols float32 matrix stored as `layout`: row (row-major), trans (column-major) or general (every
    other column of a wider row-major buffer, the B[:, ::2] of a strided view)"""

    def __init__(self, x, layout):
        R, Cc = x.shape
        self.x = x
        if layout == "row":
            self.buf, self.rs, self.cs = x.copy(), Cc, 1
        elif layout == "trans":
            self.buf, self.rs, self.cs = np.ascontiguousarray(x.T), 1, R
        else:
            wide = np.full((R, 2 * Cc), 5.0, np.float32); wide[:, ::2] = x
            self.buf, self.rs, self.cs = wide, 2 * Cc, 2
        self.t = dev(self.buf)


def aux_layout_of(layout, aux_layout):
    if aux_layout == "same":
        return layout
    return "trans" if layout == "row" else "row"


def run_case(path, M, N, K, opa, opb, a_layout="row", b_layout="row", aux_layout="same", alpha=0.5, beta=0.75, ldc_pad=3,
             lo=0.0, hi=1.0, epi=None):
    """one fused call against the oracle on the op'd operands; -> (got, want, path taken).  C starts in [lo, hi) too, so
    with U(0,1) inputs and beta > 0 every element of C is positive (the max-relative gate)."""
    A = O.fill_uniform_f32(M * K, 1, lo, hi).reshape(M, K); B = O.fill_uniform_f32(K * N, 2, lo, hi).reshape(K, N)
    C0 = O.fill_uniform_f32(M * N, 3, lo, hi).reshape(M, N)
    ta, tb = Operand(A, a_layout), Operand(B, b_layout)
    specs, Aop, Bop, keep = [None, None], A, B, []
    for i, (name, x, t, layout) in enumerate(((opa, A, ta, a_layout), (opb, B, tb, b_layout))):
        if name is None:
            continue
        y = aux_for(name, x.shape, 10 + i)
        if name.endswith("_grad"):
            aux = Operand(y, aux_layout_of(layout, aux_layout))
            keep.append(aux)
            specs[i] = (name, aux.t, aux.rs, aux.cs)
        else:
            specs[i] = name
        if i == 0:
            Aop = op_ref(name, x, y)
        else:
            Bop = op_ref(name, x, y)
    ldc = N + ldc_pad
    want = np.full((M, ldc), -7.0, np.float32); want[:, :N] = C0
    O.gemm_strided(M, N, K, alpha, Aop, K, 1, Bop, N, 1, beta, want, ldc, 1)
    kw = {}
    if epi is not None:
        bias, act = epi
        kw = dict(bias=dev(bias), activation=act)
    hbuf = np.full((M, ldc), -7.0, np.float32); hbuf[:, :N] = C0
    tc = dev(hbuf)
    L.gemm_strided_fused(M, N, K, alpha, ta.t, ta.rs, ta.cs, tb.t, tb.rs, tb.cs, beta, tc, ldc, 1, path=path,
                         op_a=specs[0], op_b=specs[1], **kw)
    sync()
    got = tc.cpu().numpy()
    assert np.all(got[:, N:] == -7.0)                    # the padding of C is not touched
    for o in [ta, tb] + keep:                             # inputs are read only
        assert np.array_equal(o.t.cpu().numpy().view(np.uint32), o.buf.view(np.uint32))
    return got[:, :N], want[:, :N], L.last_path()


def assert_gates(path_taken, got, want, names, positive=True):
    exact = all(n is None or n not in ("tanh", "sigmoid") for n in names)
    if path_taken == L.PATH_SIMT:
        if exact:
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        else:
            assert O.normwise_relative_error(got, want) <= 1e-6
    elif path_taken == L.PATH_TF32X1:
        assert O.normwise_relative_error(got, want) < 2e-3
    else:
        if positive:
            assert O.max_relative_error(got, want) < 1e-4, O.max_relative_error(got, want)
        assert O.normwise_relative_error(got, want) < 2e-6
        assert O.mean_relative_error(got, want) <= 1e-5


@pytest.mark.parametrize("where", ["A", "B", "both"])
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("path", list(PATHS))
def test_ops_on_every_path(path, op, where):
    """beta != 0, padded C; U(0,1) operands (the op'd operands stay non-negative: the max-relative gate applies)"""
    M, N, K = SHAPE
    opa = op if where in ("A", "both") else None
    opb = op if where in ("B", "both") else None
    got, want, taken = run_case(PATHS[path], M, N, K, opa, opb)
    if path != "auto":
        assert taken == PATHS[path]
    assert_gates(taken, got, want, (opa, opb))


@pytest.mark.parametrize("aux_layout", ["same", "other"])
@pytest.mark.parametrize("layouts", [("row", "row"), ("trans", "trans"), ("general", "general"), ("row", "general")])
@pytest.mark.parametrize("ops", [("relu_grad", "tanh_grad"), ("sigmoid", "sigmoid_grad")])
@pytest.mark.parametrize("path", list(PATHS))
def test_operand_and_aux_layouts(path, ops, layouts, aux_layout):
    """row-major, transposed and general (every other column) operands, aux in the operand's layout or another one"""
    M, N, K = SHAPE
    got, want, taken = run_case(PATHS[path], M, N, K, ops[0], ops[1], layouts[0], layouts[1], aux_layout)
    assert_gates(taken, got, want, ops)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
def test_signed_inputs_meet_the_fp32_gates(path):
    """U(-0.1, 0.1): normwise < 2e-6 and mean_relative_error <= 1e-5"""
    M, N, K = SHAPE
    got, want, taken = run_case(PATHS[path], M, N, K, "relu_grad", "tanh_grad", lo=-0.1, hi=0.1)
    assert_gates(taken, got, want, ("relu_grad", "tanh_grad"), positive=False)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "simt"])
def test_long_k_major_rows(path):
    """K-major rows of 2048 floats: without an op the ring kernel prepares them; with one, the register-only row kernel"""
    M, N, K = 192, 192, 2048
    emu_budget(M * N * K)
    got, want, taken = run_case(PATHS[path], M, N, K, "relu_grad", "sigmoid_grad", "row", "trans")
    assert_gates(taken, got, want, ("relu_grad", "sigmoid_grad"))


@pytest.mark.parametrize("b_layout", ["trans", "row"])
def test_scale_is_taken_after_the_op(b_layout):
    """F16X3: SIGMOID on rows of A (columns of B) whose raw values are all below 1e-20 (outputs ~0.5), TANH_GRAD with |aux|
    up to 300 (factors near -9e4).  A scale word taken over the raw values overflows the fp16 pieces."""
    M, N, K = SHAPE
    A = (O.fill_uniform_f32(M * K, 1, -1, 1) * 1e-21).reshape(M, K)
    B = (O.fill_uniform_f32(K * N, 2, -1, 1) * 1e-21).reshape(K, N)
    ta, tb = Operand(A, "row"), Operand(B, b_layout)
    want = np.zeros((M, N), np.float32)
    O.gemm_strided(M, N, K, 1.0, op_ref("sigmoid", A, None), K, 1, op_ref("sigmoid", B, None), N, 1, 0.0, want, N, 1)
    tc = dev(np.zeros((M, N), np.float32))
    L.gemm_strided_fused(M, N, K, 1.0, ta.t, ta.rs, ta.cs, tb.t, tb.rs, tb.cs, 0.0, tc, N, 1, path=L.PATH_F16X3,
                         op_a="sigmoid", op_b="sigmoid")
    sync()
    got = tc.cpu().numpy()
    assert O.max_relative_error(got, want) < 1e-4 and O.normwise_relative_error(got, want) < 2e-6
    X = O.fill_uniform_f32(M * K, 3, -1, 1).reshape(M, K); Y = O.fill_uniform_f32(M * K, 4, -300, 300).reshape(M, K)
    Xb = O.fill_uniform_f32(K * N, 5, -1, 1).reshape(K, N); Yb = O.fill_uniform_f32(K * N, 6, -300, 300).reshape(K, N)
    ta, tb, ya, yb = Operand(X, "row"), Operand(Xb, b_layout), Operand(Y, "row"), Operand(Yb, b_layout)
    want = np.zeros((M, N), np.float32)
    O.gemm_strided(M, N, K, 1.0, op_ref("tanh_grad", X, Y), K, 1, op_ref("tanh_grad", Xb, Yb), N, 1, 0.0, want, N, 1)
    tc = dev(np.zeros((M, N), np.float32))
    L.gemm_strided_fused(M, N, K, 1.0, ta.t, ta.rs, ta.cs, tb.t, tb.rs, tb.cs, 0.0, tc, N, 1, path=L.PATH_F16X3,
                         op_a=("tanh_grad", ya.t, ya.rs, ya.cs), op_b=("tanh_grad", yb.t, yb.rs, yb.cs))
    sync()
    assert O.normwise_relative_error(tc.cpu().numpy(), want) < 2e-6


@pytest.mark.parametrize("path", ["simt", "f16x3", "tf32x3"])
def test_prologue_and_epilogue_in_one_call(path):
    M, N, K = SHAPE
    bias = O.fill_uniform_f32(N, 4, -1, 1)
    got, base, taken = run_case(PATHS[path], M, N, K, "relu_grad", "sigmoid_grad", epi=(bias, "tanh"))
    want = np.tanh(base.astype(np.float64) + bias[None, :]).astype(np.float32)
    assert np.allclose(got, want, rtol=2e-5, atol=2e-6), np.abs(got - want).max()


def _call_raw(M, N, K, tA, tB, tC, opa, opb, epi, path):
    """the C entry itself (NULL pointers where the Python mirror would take the epilogue entry)"""
    sync()
    rc = _capi.lib().laser_b200_gemm_strided_f32_fused_dev(M, N, K, 1.0, tA.data_ptr(), K, 1, tB.data_ptr(), N, 1, 0.0,
                                                           tC.data_ptr(), N, 1, opa, opb, epi, path, G._current_stream())
    sync()
    return rc


@pytest.mark.parametrize("path", ["simt", "f16x3", "tf32x3", "tf32x1", "auto"])
def test_null_ops_are_the_plain_call(path):
    """opA = opB = epi = NULL: the same path, the same launches, a bit-identical C; and a plain call after a fused one
    gives what it gave before (the op lives in the call's arguments only)"""
    M, N, K = SHAPE
    A = O.fill_uniform_f32(M * K, 1, -1, 1).reshape(M, K); B = O.fill_uniform_f32(K * N, 2, -1, 1).reshape(K, N)
    tA, tB = dev(A), dev(B)
    c1, c2, c3 = dev(np.zeros((M, N), np.float32)), dev(np.zeros((M, N), np.float32)), dev(np.zeros((M, N), np.float32))
    n0 = L.launch_count()
    L.gemm_strided(M, N, K, 1.0, tA, K, 1, tB, N, 1, 0.0, c1, N, 1, path=PATHS[path]); sync()
    n1 = L.launch_count(); p1 = L.last_path()
    assert _call_raw(M, N, K, tA, tB, c2, None, None, None, PATHS[path]) == 0
    n2 = L.launch_count()
    assert L.last_path() == p1 and n2 - n1 == n1 - n0
    assert np.array_equal(c1.cpu().numpy().view(np.uint32), c2.cpu().numpy().view(np.uint32))
    aux = dev(aux_for("tanh_grad", (M, K), 9))
    L.gemm_strided_fused(M, N, K, 1.0, tA, K, 1, tB, N, 1, 0.0, c3, N, 1, path=PATHS[path], op_a=("tanh_grad", aux, K, 1),
                         op_b="relu")
    L.gemm_strided(M, N, K, 1.0, tA, K, 1, tB, N, 1, 0.0, c3, N, 1, path=PATHS[path]); sync()
    assert np.array_equal(c1.cpu().numpy().view(np.uint32), c3.cpu().numpy().view(np.uint32))


def test_invalid_ops_launch_nothing():
    M, N, K = SHAPE
    tA, tB = dev(np.ones((M, K), np.float32)), dev(np.ones((K, N), np.float32))
    tC = dev(np.full((M, N), 3.0, np.float32))
    for op, aux in ((7, None), (-1, None), (_capi.OP_RELU_GRAD, None), (_capi.OP_TANH_GRAD, None), (_capi.OP_SIGMOID_GRAD, None)):
        spec = _capi.OperandOp(op=op, aux=aux, auxRowStride=K, auxColStride=1)
        for opa, opb in ((ctypes.byref(spec), None), (None, ctypes.byref(spec))):
            n0 = L.launch_count()
            assert _call_raw(M, N, K, tA, tB, tC, opa, opb, None, L.PATH_AUTO) == _capi.E_INVAL
            assert L.launch_count() == n0
    assert np.all(tC.cpu().numpy() == 3.0)
    with pytest.raises(L.LaserB200Error):
        L.gemm_strided_fused(M, N, K, 1.0, tA, K, 1, tB, N, 1, 0.0, tC, N, 1, op_a=("relu_grad",))


def test_auto_never_takes_the_gemv_shortcut_with_an_op():
    """N = 3, M = 4096: PATH_AUTO sends a plain call to the warp-shuffle GEMV, which has no op: a call with an op must not
    go there (a wrong dispatch is a wrong result)"""
    M, N, K = 4096, 3, 256
    got, want, taken = run_case(L.PATH_AUTO, M, N, K, "relu_grad", None, alpha=1.0, beta=0.0, ldc_pad=0)
    assert_gates(taken, got, want, ("relu_grad", None))


@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("case", ["A_kmajor_aux", "A_kmajor_noaux", "B_mnmajor_aux", "B_kmajor_aux"])
def test_the_fusion_adds_no_launch(path, case):
    """an op on a K-major or MN-major operand with same-layout aux, or with none, adds zero launches over the plain call"""
    M, N, K = SHAPE
    opa = {"A_kmajor_aux": "relu_grad", "A_kmajor_noaux": "tanh"}.get(case)
    opb = {"B_mnmajor_aux": "sigmoid_grad", "B_kmajor_aux": "tanh_grad"}.get(case)
    b_layout = "trans" if case == "B_kmajor_aux" else "row"
    B = O.fill_uniform_f32(K * N, 2, 0, 1).reshape(K, N)
    tb = Operand(B, b_layout)
    tA = dev(O.fill_uniform_f32(M * K, 1, 0, 1).reshape(M, K))
    tc = dev(np.zeros((M, N), np.float32))
    n0 = L.launch_count()
    L.gemm_strided(M, N, K, 1.0, tA, K, 1, tb.t, tb.rs, tb.cs, 0.0, tc, N, 1, path=PATHS[path]); sync()
    plain = L.launch_count() - n0
    got, want, taken = run_case(PATHS[path], M, N, K, opa, opb, "row", b_layout, alpha=1.0, beta=0.0, ldc_pad=0)
    n1 = L.launch_count()
    ya = Operand(aux_for("relu_grad", (M, K), 10), "row")
    yb = Operand(aux_for("tanh_grad", (K, N), 11), b_layout)
    L.gemm_strided_fused(M, N, K, 1.0, tA, K, 1, tb.t, tb.rs, tb.cs, 0.0, tc, N, 1, path=PATHS[path],
                         op_a=None if opa is None else (opa if opa == "tanh" else (opa, ya.t, ya.rs, ya.cs)),
                         op_b=None if opb is None else (opb, yb.t, yb.rs, yb.cs))
    sync()
    assert L.launch_count() - n1 == plain
    assert_gates(taken, got, want, (opa, opb))


@needs_gpu
def test_full_size_backward_product():
    """8192^3, F16X3, RELU_GRAD on A and TANH_GRAD on B, gated over the whole C against the exact kernel on op'd operands
    (materialised by torch: one rounding per operation, as in the header's formulas)"""
    import torch
    from test_gpu_parity import _gates_on_device
    M = N = K = 8192
    tA = torch.empty(M * K, dtype=torch.float32, device="cuda"); tZ = torch.empty_like(tA)
    tB = torch.empty(K * N, dtype=torch.float32, device="cuda"); tY = torch.empty_like(tB)
    L.fill_uniform_f32(tA, M * K, 42, 0, 1); L.fill_uniform_f32(tZ, M * K, 44, -1, 1)
    L.fill_uniform_f32(tB, K * N, 43, 0, 1); L.fill_uniform_f32(tY, K * N, 45, -1, 1)
    got = torch.full((M, N), float("nan"), dtype=torch.float32, device="cuda")
    L.gemm_strided_fused(M, N, K, 1.0, tA, K, 1, tB, N, 1, 0.0, got, N, 1, path=L.PATH_F16X3,
                         op_a=("relu_grad", tZ, K, 1), op_b=("tanh_grad", tY, N, 1))
    assert L.last_path() == L.PATH_F16X3
    Aop = torch.where(tZ > 0, tA, torch.zeros_like(tA))
    Bop = tB * (1 - tY * tY)
    ref = torch.full((M, N), float("nan"), dtype=torch.float32, device="cuda")
    L.gemm_strided(M, N, K, 1.0, Aop, K, 1, Bop, N, 1, 0.0, ref, N, 1, path=L.PATH_SIMT)
    torch.cuda.synchronize()
    assert not torch.isnan(got).any()
    max_rel, normwise, mre = _gates_on_device(got, ref, True)
    assert max_rel < 1e-4 and normwise < 2e-6 and mre <= 1e-5, (max_rel, normwise, mre)
