"""GPU: the batched fused product laser_b200_gemm_strided_batched_f32_fused_dev -- every problem of a batch prepared in the
launches of one problem and multiplied in one GEMM launch.  Each problem must equal the single fused call on its own views
bit for bit, on every path; the launch count must not grow with the batch."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, emu_budget, needs_gpu, sync

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
# straddles the 128-row / 128-column tiles and the 64-element k-tile; K <= 768 keeps split-K off in both calls
SHAPE, BATCH = ((130, 140, 100), 3) if EMU else ((200, 260, 300), 5)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def at(t, off):
    """device address `off` float32 elements into t"""
    return L.DevPtr(t.data_ptr() + 4 * off, "f32")


class Batched:
    """batch matrices of R x Cc float32 in one buffer: problem b's element (i, j) at base + b * bs + i * rs + j * cs.
    layout: row, trans (column-major) or general (every other column of wider rows); share: bs = 0; neg: bs < 0."""

    def __init__(self, batch, R, Cc, layout, seed, lo=0.0, hi=1.0, share=False, neg=False, gap=8):
        rs, cs, span = {"row": (Cc, 1, R * Cc), "trans": (1, R, R * Cc), "general": (2 * Cc, 2, 2 * R * Cc)}[layout]
        self.rs, self.cs = rs, cs
        per = span + gap
        self.bs = 0 if share else (-per if neg else per)
        n = 1 if share else batch
        self.base = (n - 1) * per if neg else 0
        buf = np.full(n * per, 5.0, np.float32)
        self.x = O.fill_uniform_f32(n * R * Cc, seed, lo, hi).reshape(n, R, Cc)
        i, j = np.arange(R)[:, None], np.arange(Cc)[None, :]
        for b in range(n):
            buf[self.base + (0 if share else b * self.bs) + i * rs + j * cs] = self.x[b]
        self.buf = buf
        self.t = dev(buf)

    def off(self, b):
        return self.base + b * self.bs

    def ptr(self, b=0):
        return at(self.t, self.off(b))


def c_buffer(batch, M, N, ldc, gap, nan):
    bsC = M * ldc + gap
    c0 = np.full(batch * bsC, -7.0, np.float32)
    i, j = np.arange(M)[:, None], np.arange(N)[None, :]
    for b in range(batch):
        c0[b * bsC + i * ldc + j] = np.nan if nan else O.fill_uniform_f32(M * N, 3 + b, 0, 1).reshape(M, N)
    return c0, bsC


def spec(op, aux, b=None):
    """op_a / op_b argument: batched (b None) or the single call's for problem b"""
    if op is None:
        return None
    if aux is None:
        return op
    if b is None:
        return (op, aux.ptr(), aux.rs, aux.cs, aux.bs)
    return (op, aux.ptr(b), aux.rs, aux.cs)


def run_pair(path, batch=BATCH, shape=SHAPE, la="row", lb="row", share_a=False, share_b=False, neg=False, opa=None, opb=None,
             aux_b_layout=None, alpha=0.5, beta=0.75, nan_c=False, ldc_pad=3, gap_c=6, epi=None):
    """the batched call and the single fused calls problem by problem, on copies of one C buffer -> (batched C, single C,
    launches of the batched call)"""
    M, N, K = shape
    A = Batched(batch, M, K, la, 1, share=share_a, neg=neg)
    B = Batched(batch, K, N, lb, 2, share=share_b, neg=neg)
    auxa = Batched(batch, M, K, la, 11, -1, 1, neg=neg) if opa == "relu_grad" else None
    auxb = Batched(batch, K, N, aux_b_layout or lb, 12, -1, 1) if opb == "tanh_grad" else None
    ldc = N + ldc_pad
    c0, bsC = c_buffer(batch, M, N, ldc, gap_c, nan_c)
    kw = {}
    if epi is not None:
        kw = dict(bias=dev(O.fill_uniform_f32(N, 4, -1, 1)), activation=epi)
    tcb, tcs = dev(c0), dev(c0)
    sync()
    n0 = L.launch_count()
    L.gemm_strided_batched_fused(batch, M, N, K, alpha, A.ptr(), A.rs, A.cs, A.bs, B.ptr(), B.rs, B.cs, B.bs, beta, tcb, ldc, 1,
                                 bsC, path=path, op_a=spec(opa, auxa), op_b=spec(opb, auxb), **kw)
    sync()
    launches = L.launch_count() - n0
    for b in range(batch):
        L.gemm_strided_fused(M, N, K, alpha, A.ptr(b), A.rs, A.cs, B.ptr(b), B.rs, B.cs, beta, at(tcs, b * bsC), ldc, 1, path=path,
                             op_a=spec(opa, auxa, b), op_b=spec(opb, auxb, b), **kw)
    sync()
    return tcb.cpu().numpy().copy(), tcs.cpu().numpy().copy(), launches


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


@pytest.mark.parametrize("layouts", [("row", "row"), ("trans", "trans"), ("general", "general"), ("row", "trans")])
@pytest.mark.parametrize("path", list(PATHS))
def test_layouts_bit_identical_to_single_calls(path, layouts):
    got, want, _ = run_pair(PATHS[path], la=layouts[0], lb=layouts[1])
    assert_bits(got, want)


@pytest.mark.parametrize("case", ["share_a", "share_b", "negative"])
@pytest.mark.parametrize("path", list(PATHS))
def test_shared_and_negative_batch_strides(path, case):
    got, want, _ = run_pair(PATHS[path], share_a=case == "share_a", share_b=case == "share_b", neg=case == "negative")
    assert_bits(got, want)


@pytest.mark.parametrize("case", ["relu_grad_A", "tanh_grad_B_other_layout", "both_shared_A"])
@pytest.mark.parametrize("path", list(PATHS))
def test_operand_ops(path, case):
    """relu' on A with per-problem aux, tanh' on B with aux in another layout; A shared with a per-problem aux"""
    if case == "relu_grad_A":
        got, want, _ = run_pair(PATHS[path], opa="relu_grad")
    elif case == "tanh_grad_B_other_layout":
        got, want, _ = run_pair(PATHS[path], opb="tanh_grad", aux_b_layout="trans")
    else:
        got, want, _ = run_pair(PATHS[path], share_a=True, opa="relu_grad", opb="tanh_grad", lb="trans")
    assert_bits(got, want)


@pytest.mark.parametrize("path", list(PATHS))
def test_epilogue_scalars_and_c_layout(path):
    """bias + activation; beta = 0 over a NaN-filled C (never read); an odd guard between the problems' C (no paired stores)"""
    got, want, _ = run_pair(PATHS[path], epi="tanh", alpha=1.5, beta=0.25)
    assert_bits(got, want)
    got, want, _ = run_pair(PATHS[path], beta=0.0, nan_c=True, ldc_pad=0, gap_c=5)
    assert_bits(got, want)
    assert not np.isnan(got[:SHAPE[0] * SHAPE[1]]).any()


@pytest.mark.parametrize("layouts", [("row", "row"), ("trans", "trans"), ("general", "general"), ("row", "trans")])
@pytest.mark.parametrize("path", list(PATHS))
def test_launch_count_does_not_grow_with_the_batch(path, layouts):
    shape, big = ((64, 72, 80), 16) if EMU else ((200, 260, 300), 64)
    _, _, one = run_pair(PATHS[path], batch=1, shape=shape, la=layouts[0], lb=layouts[1])
    got, want, many = run_pair(PATHS[path], batch=big, shape=shape, la=layouts[0], lb=layouts[1], opa="relu_grad")
    _, _, one_op = run_pair(PATHS[path], batch=1, shape=shape, la=layouts[0], lb=layouts[1], opa="relu_grad")
    assert many == one_op
    assert_bits(got, want)
    _, _, many = run_pair(PATHS[path], batch=big, shape=shape, la=layouts[0], lb=layouts[1])
    assert many == one


def _raw(batch, strides, opa=None, path=L.PATH_AUTO):
    M, N, K = 8, 8, 8
    tA, tB, tC = dev(np.ones(64, np.float32)), dev(np.ones(64, np.float32)), dev(np.full(64, 3.0, np.float32))
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_gemm_strided_batched_f32_fused_dev(
        batch, M, N, K, 1.0, tA.data_ptr(), K, 1, tB.data_ptr(), N, 1, 0.0, tC.data_ptr(), N, 1, strides, opa, None, None, path,
        G._current_stream())
    sync()
    assert np.all(tC.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_errors_launch_nothing():
    ok = ctypes.byref(_capi.BatchStrides(0, 0, 64, 0, 0))
    assert _raw(-1, ok) == (_capi.E_INVAL, 0)
    assert _raw(2, None) == (_capi.E_INVAL, 0)
    assert _raw(2, ctypes.byref(_capi.BatchStrides(0, 0, 0, 0, 0))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, ctypes.byref(_capi.OperandOp(op=9))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, path=5) == (_capi.E_INVAL, 0)
    assert _raw(0, ok) == (_capi.E_OK, 0)
    assert _raw(0, None) == (_capi.E_OK, 0)
    with pytest.raises(ValueError):
        L.gemm_strided_batched_fused(2, 8, 8, 8, 1.0, dev(np.ones(64, np.float32)), 8, 1, 0, dev(np.ones(64, np.float32)), 8, 1,
                                     0, 0.0, dev(np.zeros(128, np.float32)), 8, 1, 64, op_a=("relu_grad", None, 8, 1))


LONG_K = ((64, 64, 2048), 2) if EMU else ((200, 260, 2048), 3)


def test_long_k_with_split_k_meets_the_fp32_gates():
    """few tiles and a long K: split-K planes and the reduce kernel over the batch, against the oracle per problem"""
    (M, N, K), batch = LONG_K
    A, B = Batched(batch, M, K, "row", 1), Batched(batch, K, N, "row", 2)
    c0, bsC = c_buffer(batch, M, N, N, 4, False)
    tc = dev(c0)
    L.gemm_strided_batched_fused(batch, M, N, K, 1.0, A.ptr(), K, 1, A.bs, B.ptr(), N, 1, B.bs, 0.5, tc, N, 1, bsC,
                                 path=L.PATH_F16X3)
    sync()
    got = tc.cpu().numpy()
    for b in range(batch):
        want = c0[b * bsC:b * bsC + M * N].reshape(M, N).copy()
        O.gemm_strided(M, N, K, 1.0, A.x[b], K, 1, B.x[b], N, 1, 0.5, want, N, 1)
        g = got[b * bsC:b * bsC + M * N].reshape(M, N)
        assert O.max_relative_error(g, want) < 1e-4
        assert O.normwise_relative_error(g, want) < 2e-6 and O.mean_relative_error(g, want) <= 1e-5
    assert np.all(got[M * N:bsC] == -7.0)


def _subprocess(code, **env):
    e = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]), **env)
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=e, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout


_SUB = """
import numpy as np, test_gpu_batched_fused as T, laser_b200 as L
got, want, n = T.run_pair(L.PATH_F16X3, batch=%d, shape=%r)
assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
np.save(%r, got)
print("LAUNCHES", n)
"""


def test_long_k_without_split_k_is_bit_identical(tmp_path):
    (M, N, K), batch = LONG_K
    _subprocess(_SUB % (batch, (M, N, K), str(tmp_path / "c.npy")), LASER_B200_SPLITK="0")


def test_chunks_are_bit_identical_to_one_launch(tmp_path):
    """a 1 MB workspace cap holds one problem at a time: 3 chunks for 3 problems, each with the launches of one chunk"""
    shape = (192, 192, 192)
    got, want, n_whole = run_pair(L.PATH_F16X3, batch=3, shape=shape)
    launches = {}
    for batch in (2, 3):
        f = str(tmp_path / ("c%d.npy" % batch))
        out = _subprocess(_SUB % (batch, shape, f), LASER_B200_BATCH_WS_MB="1")
        launches[batch] = int(out.split("LAUNCHES")[1].split()[0])
    assert launches[3] % 3 == 0 and launches[3] // 3 == launches[2] // 2 and launches[2] % 2 == 0
    assert launches[3] == 3 * n_whole
    assert np.array_equal(np.load(str(tmp_path / "c3.npy")).view(np.uint32), got.view(np.uint32))


@needs_gpu
def test_32_problems_of_1024_cubed_against_float64():
    import torch
    batch, n = 32, 1024
    emu_budget(batch * n ** 3)
    tA = torch.empty(batch * n * n, dtype=torch.float32, device="cuda"); tB = torch.empty_like(tA)
    L.fill_uniform_f32(tA, tA.numel(), 42, -1, 1); L.fill_uniform_f32(tB, tB.numel(), 43, -1, 1)
    got = torch.full((batch, n, n), float("nan"), dtype=torch.float32, device="cuda")
    L.gemm_strided_batched_fused(batch, n, n, n, 1.0, tA, n, 1, n * n, tB, n, 1, n * n, 0.0, got, n, 1, n * n)
    torch.cuda.synchronize()
    assert L.last_path() == L.PATH_F16X3
    ref = torch.bmm(tA.view(batch, n, n).double(), tB.view(batch, n, n).double())
    d = (got.double() - ref)
    normwise = (torch.linalg.norm(d) / torch.linalg.norm(ref)).item()
    den = torch.maximum(got.double().abs(), ref.abs())
    mre = torch.where(den > 0, d.abs() / den, torch.zeros_like(d)).mean().item()
    assert normwise < 2e-6 and mre <= 1e-5, (normwise, mre)
