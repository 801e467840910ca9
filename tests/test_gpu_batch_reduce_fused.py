"""GPU: the batch-reduced fused product laser_b200_gemm_strided_batch_reduce_f32_fused_dev -- C <- act(alpha * sum_b
opA(A_b) * opB(B_b) + beta * C + bias) as one fused product over the operands concatenated along K.  C must equal, bit for bit
and on every path, the fused call over the materialised concatenation A^ = [A_0 | .. | A_{n-1}], B^ = [B_0; ..; B_{n-1}]
(aux tensors concatenated the same way); the exact path equals the CPU oracle over A^, B^; the tensor-core paths meet the
per-element bound of tests/test_gpu_error_bounds.py with K' = n * K; the preparation launches do not grow with the batch."""
import ctypes

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, emu_budget, sync
from test_gpu_batched_fused import Batched, assert_bits, at
from test_gpu_error_bounds import bound_and_check, plan, scaled

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
TC_NAMES = {L.PATH_F16X3: "f16x3", L.PATH_TF32X3: "tf32x3", L.PATH_TF32X1: "tf32x1"}
# M and N straddle the 128-row / 128-column tiles; K = 75 is not a multiple of 4, so every segment boundary but the first
# lies off the 16-byte grid; n * K <= 768 keeps split-K off
SHAPE, BATCH = ((130, 140, 75), 4) if EMU else ((200, 260, 150), 5)
ACTS = ["none", "relu", "tanh", "sigmoid"]


def concat(X, batch, axis):
    """the problems' matrices of a Batched laid end to end (axis 1: along columns, A^; axis 0: along rows, B^)"""
    return np.ascontiguousarray(np.concatenate([X.x[0 if X.bs == 0 else b] for b in range(batch)], axis=axis))


def op_spec(op, aux, batched):
    if op is None:
        return None
    if aux is None:
        return op
    return (op, aux.ptr(), aux.rs, aux.cs, aux.bs) if batched else (op, aux[0], aux[1], aux[2])


def run_pair(path, batch=BATCH, shape=SHAPE, la="row", lb="row", share_a=False, share_b=False, neg=False, opa=None, opb=None,
             aux_b_layout=None, alpha=0.5, beta=0.75, nan_c=False, act=None, bias_per_row=False):
    """the batch-reduced call, and the fused call over the materialised concatenation, on copies of one C -> (reduced C, fused
    C, launches of the reduced call, launches of the fused call, (A^, B^, C0) as float32 arrays)"""
    M, N, K = shape
    A = Batched(batch, M, K, la, 1, -1, 1, share=share_a, neg=neg)
    B = Batched(batch, K, N, lb, 2, -1, 1, share=share_b, neg=neg)
    auxa = Batched(batch, M, K, la, 11, -1, 1, neg=neg) if opa == "relu_grad" else None
    auxb = Batched(batch, K, N, aux_b_layout or lb, 12, -1, 1) if opb in ("tanh_grad", "sigmoid_grad") else None
    Ah, Bh = concat(A, batch, 1), concat(B, batch, 0)
    ldc = N + 3
    c0 = np.full(M * ldc, np.nan if nan_c else 0.0, np.float32)
    if not nan_c:
        c0[:] = O.fill_uniform_f32(M * ldc, 3, -1, 1)
    kw = {}
    if act is not None:
        kw = dict(bias=dev(O.fill_uniform_f32(M if bias_per_row else N, 4, -1, 1)), bias_per_row=bias_per_row, activation=act)
    tr, tf = dev(c0), dev(c0)
    tAh, tBh = dev(Ah), dev(Bh)
    aux_a_h = (dev(concat(auxa, batch, 1)), batch * K, 1) if auxa else None
    aux_b_h = (dev(concat(auxb, batch, 0)), N, 1) if auxb else None
    sync()
    n0 = L.launch_count()
    L.gemm_strided_batch_reduce_fused(batch, M, N, K, alpha, A.ptr(), A.rs, A.cs, A.bs, B.ptr(), B.rs, B.cs, B.bs, beta, tr, ldc, 1,
                                      path=path, op_a=op_spec(opa, auxa, True), op_b=op_spec(opb, auxb, True), **kw)
    sync()
    n1 = L.launch_count()
    L.gemm_strided_fused(M, N, batch * K, alpha, tAh, batch * K, 1, tBh, N, 1, beta, tf, ldc, 1, path=path,
                         op_a=op_spec(opa, aux_a_h, False), op_b=op_spec(opb, aux_b_h, False), **kw)
    sync()
    n2 = L.launch_count()
    return tr.cpu().numpy().copy(), tf.cpu().numpy().copy(), n1 - n0, n2 - n1, (Ah, Bh, c0)


@pytest.mark.parametrize("layouts", [("row", "row"), ("trans", "trans"), ("general", "general"), ("row", "trans")])
@pytest.mark.parametrize("path", list(PATHS))
def test_layouts_bit_identical_to_the_concatenated_call(path, layouts):
    got, want, _, _, _ = run_pair(PATHS[path], la=layouts[0], lb=layouts[1])
    assert_bits(got, want)


@pytest.mark.parametrize("case", ["share_a", "share_b", "negative", "trans_negative"])
@pytest.mark.parametrize("path", list(PATHS))
def test_shared_negative_and_padded_batch_strides(path, case):
    """a stride of 0: the same matrix in every K segment; negative strides; every Batched is padded between its problems"""
    trans = case == "trans_negative"
    got, want, _, _, _ = run_pair(PATHS[path], share_a=case == "share_a", share_b=case == "share_b", neg=case.endswith("negative"),
                                  la="trans" if trans else "row", lb="trans" if trans else "row")
    assert_bits(got, want)


@pytest.mark.parametrize("case", ["relu_grad_A", "tanh_grad_B_other_layout", "sigmoid_grad_B_shared_A", "relu_A_tanh_B"])
@pytest.mark.parametrize("path", list(PATHS))
def test_operand_ops_with_batched_aux(path, case):
    """relu' on A with its own aux per problem; tanh' on B with aux in another layout (the gather); sigmoid' on B with A shared;
    ops without aux on both"""
    kw = {"relu_grad_A": dict(opa="relu_grad"), "tanh_grad_B_other_layout": dict(opb="tanh_grad", aux_b_layout="trans"),
          "sigmoid_grad_B_shared_A": dict(opb="sigmoid_grad", share_a=True, lb="trans"),
          "relu_A_tanh_B": dict(opa="relu", opb="tanh")}[case]
    got, want, _, _, _ = run_pair(PATHS[path], **kw)
    assert_bits(got, want)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("path", list(PATHS))
def test_bias_activation_and_scalars(path, act):
    """the bias per row (relu, sigmoid) or per column, the activation applied once to the whole sum; beta = 0 over a NaN-filled
    C (never read)"""
    got, want, _, _, _ = run_pair(PATHS[path], act=act, bias_per_row=act in ("relu", "sigmoid"), alpha=-1.5, beta=0.25)
    assert_bits(got, want)
    got, want, _, _, _ = run_pair(PATHS[path], act=act, beta=0.0, nan_c=True)
    assert_bits(got, want)
    M, N, _ = SHAPE
    assert not np.isnan(got.reshape(M, N + 3)[:, :N]).any()


SPLIT = ((64, 64, 512), 4) if EMU else ((128, 128, 2048), 16)   # n * K = 2048 / 32768 over one output tile


@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
def test_split_k_is_bit_identical_and_within_the_bound(path):
    """few output tiles and a long K': the plan splits K (the reduce kernel is one more launch than the preparation and the
    GEMM), and the result is the concatenated call's bit for bit and within the per-element bound"""
    (M, N, K), batch = SPLIT
    ks, _ = plan(path, M, N, batch * K)
    assert ks >= 2, "the shape must split K"
    got, want, n_red, n_fused, (Ah, Bh, c0) = run_pair(PATHS[path], batch=batch, shape=(M, N, K), alpha=1.0, beta=0.5)
    assert_bits(got, want)
    # A row-major: one concatenating row pass; B row-major (MN-major): f16x3 column words, then the split -- tf32x3 one gather;
    # then the GEMM and the reduce
    assert n_red == {"f16x3": 3, "tf32x3": 2}[path] + 2 and n_fused == n_red
    ldc = N + 3
    g = got.reshape(M, ldc)[:, :N]
    bound_and_check("batch_reduce split", path, "batch_reduce", g, Ah, Bh, 1.0, 0.5, c0.reshape(M, ldc)[:, :N], splits=ks)


def test_exact_path_matches_the_oracle_over_the_concatenation():
    M, N, K = SHAPE
    got, _, _, _, (Ah, Bh, c0) = run_pair(L.PATH_SIMT, la="general", lb="trans", neg=True)
    ldc = N + 3
    want = c0.copy()
    O.gemm_strided(M, N, BATCH * K, 0.5, Ah, BATCH * K, 1, Bh, N, 1, 0.75, want, ldc, 1)
    assert_bits(got, want)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound(path):
    """signed data, every row of each A_b and column of each B_b and every problem at its own power-of-two scale"""
    (M, N, K), batch = ((130, 140, 96), 6) if EMU else ((257, 255, 384), 12)
    rng = np.random.default_rng(7)
    a = np.stack([scaled(rng, (M, K), rows=True) * np.float32(2.0 ** rng.integers(-6, 7)) for _ in range(batch)])
    b = np.stack([scaled(rng, (K, N), cols=True) * np.float32(2.0 ** rng.integers(-6, 7)) for _ in range(batch)])
    tA, tB = dev(a.reshape(-1)), dev(b.reshape(-1))
    C = dev(np.full(M * N, np.nan, np.float32))
    L.gemm_strided_batch_reduce_fused(batch, M, N, K, 1.0, tA, K, 1, M * K, tB, N, 1, K * N, 0.0, C, N, 1, path=PATHS[path])
    sync()
    ks, _ = plan(path, M, N, batch * K)
    bound_and_check("batch_reduce", path, "batch_reduce", C.cpu().numpy().reshape(M, N), np.concatenate(list(a), axis=1),
                    np.concatenate(list(b), axis=0), 1.0, splits=ks)


def test_convolution_filter_gradient():
    """dW = sum_n dY_n * cols_n^T: dY in NCHW ([c_out][outH*outW] per image), cols from laser_b200_im2col_f32_dev
    ([C*kH*kW][outH*outW] per image, read transposed), against torch.nn.grad.conv2d_weight in float64"""
    torch = pytest.importorskip("torch")
    imgs, C, H, W, Cout, k = (3, 4, 12, 12, 8, 3) if EMU else (8, 16, 28, 28, 32, 3)
    ishape, kshape = (imgs, C, H, W), (Cout, C, k, k)
    _, _, oh, ow = L.conv2d_out_shape(ishape, kshape, (1, 1), (1, 1))
    Kc, P = C * k * k, oh * ow
    x = O.fill_uniform_f32(imgs * C * H * W, 21, -1, 1)
    dy = O.fill_uniform_f32(imgs * Cout * P, 22, -1, 1)
    tx, tdy = dev(x), dev(dy)
    cols = dev(np.zeros(imgs * Kc * P, np.float32))
    L.im2col(cols, tx, ishape, kshape, (1, 1), (1, 1), images=imgs)
    dw = dev(np.full(Cout * Kc, np.nan, np.float32))
    # A_n = dY_n (Cout x P), B_n = cols_n^T (P x Kc): element (p, q) of B_n at cols_n[q][p]
    L.gemm_strided_batch_reduce_fused(imgs, Cout, Kc, P, 1.0, tdy, P, 1, Cout * P, cols, 1, P, Kc * P, 0.0, dw, Kc, 1,
                                      path=L.PATH_F16X3)
    sync()
    ref = torch.nn.grad.conv2d_weight(torch.from_numpy(x.astype(np.float64)).reshape(ishape), kshape,
                                      torch.from_numpy(dy.astype(np.float64)).reshape(imgs, Cout, oh, ow), padding=1).numpy()
    got = dw.cpu().numpy().reshape(Cout, Kc)
    colsn = cols.cpu().numpy().reshape(imgs, Kc, P)
    Ah = np.concatenate(list(dy.reshape(imgs, Cout, P)), axis=1)
    Bh = np.concatenate([colsn[n].T for n in range(imgs)], axis=0)
    # the concatenated operands are the filter gradient's: their float64 product is torch's
    np.testing.assert_allclose(Ah.astype(np.float64) @ Bh.astype(np.float64), ref.reshape(Cout, Kc), rtol=0,
                               atol=1e-12 * np.abs(ref).max())
    ks, _ = plan("f16x3", Cout, Kc, imgs * P)
    bound_and_check("filter gradient", "f16x3", "batch_reduce", got, Ah, Bh, 1.0, splits=ks)


@pytest.mark.parametrize("layouts", [("row", "row"), ("trans", "trans"), ("general", "general"), ("row", "trans")])
@pytest.mark.parametrize("path", list(PATHS))
def test_launch_count_does_not_grow_with_the_batch(path, layouts):
    # (M * N * 2K above 128^3: PATH_AUTO takes a tensor-core path for both batches)
    shape = (96, 96, 128) if EMU else (200, 260, 128)
    few = run_pair(PATHS[path], batch=2, shape=shape, la=layouts[0], lb=layouts[1], opa="relu_grad")
    many = run_pair(PATHS[path], batch=6, shape=shape, la=layouts[0], lb=layouts[1], opa="relu_grad")
    assert few[2] == many[2]
    assert_bits(many[0], many[1])


def test_batch_one_is_the_fused_call():
    got, want, n_red, n_fused, _ = run_pair(L.PATH_F16X3, batch=1, opa="relu_grad")
    assert_bits(got, want)
    assert n_red == n_fused


def _raw(batch, strides, opa=None, path=L.PATH_AUTO, M=8, N=8, K=8):
    tA, tB, tC = dev(np.ones(64, np.float32)), dev(np.ones(64, np.float32)), dev(np.full(64, 3.0, np.float32))
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_gemm_strided_batch_reduce_f32_fused_dev(
        batch, M, N, K, 1.0, tA.data_ptr(), K, 1, tB.data_ptr(), N, 1, 0.0, tC.data_ptr(), N, 1, strides, opa, None, None, path,
        G._current_stream())
    sync()
    assert np.all(tC.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_errors_launch_nothing():
    ok = ctypes.byref(_capi.BatchStrides(0, 0, 0, 0, 0))
    assert _raw(-1, ok) == (_capi.E_INVAL, 0)
    assert _raw(2, None) == (_capi.E_INVAL, 0)
    assert _raw(2, ctypes.byref(_capi.BatchStrides(0, 0, 64, 0, 0))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, ctypes.byref(_capi.OperandOp(op=9))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))) == (_capi.E_INVAL, 0)
    assert _raw(2, ok, path=5) == (_capi.E_INVAL, 0)
    assert _raw(0, ok) == (_capi.E_OK, 0)
    assert _raw(0, None) == (_capi.E_OK, 0)
    assert _raw(2, ok, K=0) == (_capi.E_OK, 0)
    # n * K past int32 on a tensor-core path (nothing is read: the check comes first)
    assert _raw(2 ** 20, ok, K=2 ** 12, path=L.PATH_F16X3) == (_capi.E_UNSUPPORTED, 0)


def test_big_sum_against_float64():
    """64 products of 512^3 summed, on the default path"""
    emu_budget(64 * 512 ** 3)
    batch, n = 64, 512
    import torch
    tA = torch.empty(batch * n * n, dtype=torch.float32, device="cuda"); tB = torch.empty_like(tA)
    L.fill_uniform_f32(tA, tA.numel(), 42, -1, 1); L.fill_uniform_f32(tB, tB.numel(), 43, -1, 1)
    got = torch.full((n, n), float("nan"), dtype=torch.float32, device="cuda")
    L.gemm_strided_batch_reduce_fused(batch, n, n, n, 1.0, tA, n, 1, n * n, tB, n, 1, n * n, 0.0, got, n, 1)
    torch.cuda.synchronize()
    assert L.last_path() == L.PATH_F16X3
    ref = torch.einsum("bmk,bkn->mn", tA.view(batch, n, n).double(), tB.view(batch, n, n).double())
    d = got.double() - ref
    assert (torch.linalg.norm(d) / torch.linalg.norm(ref)).item() < 2e-6
