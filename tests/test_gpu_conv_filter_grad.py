"""GPU: the fused convolution's filter gradient laser_b200_conv2d_filter_grad_f32_fused_dev -- dW <- alpha * sum_n
op(dY_n) * im2col(X_n)^T + beta * dW as one batch-reduced product whose B operand is prepared straight from the images.  On
every path dW must equal, bit for bit, the batch-reduced product over the im2col matrices materialised by laser_b200_im2col_f32_dev
and read transposed; the exact path equals the CPU oracle over the concatenation; the tensor-core paths meet the per-element
bound of tests/test_gpu_error_bounds.py with K' = n * outH * outW against torch.nn.grad.conv2d_weight in float64; the launch
count does not grow with the images, and no im2col matrix is written."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, sync
from test_gpu_error_bounds import bound_and_check, plan

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
# (ishape, kshape, padding, strides); n * outH * outW is not a multiple of 4 for stride2, non_square_3x5 and odd_batch_7x7
GEOMS = {
    "pad1": ((3, 8, 10, 10), (16, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 16, 20, 20), (48, 16, 3, 3), (1, 1), (1, 1)),
    "stride2": ((3, 4, 9, 8), (8, 4, 3, 3), (1, 1), (2, 2)) if EMU else ((5, 12, 17, 15), (40, 12, 3, 3), (1, 1), (2, 2)),
    "non_square_3x5": ((2, 3, 8, 9), (8, 3, 3, 5), (1, 2), (1, 1)) if EMU else ((3, 8, 16, 19), (32, 8, 3, 5), (1, 2), (1, 1)),
    "one_by_one_stride2": ((3, 6, 7, 7), (8, 6, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 32, 15, 15), (64, 32, 1, 1), (0, 0), (2, 2)),
    "odd_batch_7x7": ((3, 2, 9, 9), (8, 2, 3, 3), (0, 0), (1, 1)) if EMU else ((5, 16, 9, 9), (32, 16, 3, 3), (0, 0), (1, 1)),
    "single_image": ((1, 4, 8, 8), (8, 4, 3, 3), (1, 1), (1, 1)) if EMU else ((1, 16, 24, 24), (32, 16, 3, 3), (1, 1), (1, 1)),
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dW (never read), beta != 0 over a seeded one
VARIANTS = {"plain": (None, 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 1.0, 1.25)}


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


class Grad:
    """one filter gradient's data: images X, output gradients dY, the forward output Z an op's aux is taken from, and dW0"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, x=None, dy=None):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        n, C = ishape[:2]
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        self.P = self.oshape[2] * self.oshape[3]
        self.Kc = C * kshape[2] * kshape[3]
        self.x = O.fill_uniform_f32(int(np.prod(ishape)), seed, -1, 1).reshape(ishape) if x is None else x
        self.dy = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 1, -1, 1).reshape(self.oshape) if dy is None else dy
        z = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 2, -2, 2).reshape(self.oshape)
        self.aux = {"relu_grad": np.maximum(z, 0), "tanh_grad": np.tanh(z), "sigmoid_grad": 1 / (1 + np.exp(-z))}
        self.w0 = O.fill_uniform_f32(kshape[0] * self.Kc, seed + 3, -1, 1)
        self.tx, self.tdy = dev(self.x), dev(self.dy)
        self.taux = {k: dev(v.astype(np.float32)) for k, v in self.aux.items()}

    def dw0(self, beta):
        return dev(self.w0 if beta != 0.0 else np.full(self.w0.shape, np.nan, np.float32))

    def fused(self, path, op=None, alpha=1.0, beta=0.0):
        """-> (dW, launches)"""
        dw = self.dw0(beta)
        sync()
        n0 = L.launch_count()
        L.conv2d_filter_grad_fused(dw, self.tx, self.ishape, self.tdy, self.kshape, self.padding, self.strides, alpha, beta, op=op,
                                   aux=self.taux.get(op), path=path)
        sync()
        return dw.cpu().numpy().copy(), L.launch_count() - n0

    def op_a(self, op):
        if op is None or op not in self.taux:
            return op
        cout = self.kshape[0]
        return (op, self.taux[op], self.P, 1, cout * self.P)

    def unfused(self, path, op=None, alpha=1.0, beta=0.0):
        """the batch-reduced product over the im2col matrices ([Kc][P] per image) read transposed"""
        n, cout = self.ishape[0], self.kshape[0]
        cols = dev(np.zeros(n * self.Kc * self.P, np.float32))
        L.im2col(cols, self.tx, self.ishape, self.kshape, self.padding, self.strides, images=n)
        dw = self.dw0(beta)
        L.gemm_strided_batch_reduce_fused(n, cout, self.Kc, self.P, alpha, self.tdy, self.P, 1, cout * self.P, cols, 1, self.P,
                                          self.Kc * self.P, beta, dw, self.Kc, 1, path=path, op_a=self.op_a(op))
        sync()
        return dw.cpu().numpy().copy()

    def concatenated(self, op=None):
        """(A^, B^) as multiplied: [op(dY_0) | .. | op(dY_{n-1})] (Cout x nP) and [cols_0^T; ..; cols_{n-1}^T] (nP x Kc)"""
        n, cout = self.ishape[0], self.kshape[0]
        a = self.dy.reshape(n, cout, self.P).astype(np.float32)
        if op == "relu_grad":
            a = np.where(self.aux[op].reshape(a.shape) > 0, a, np.float32(0))
        Ah = np.ascontiguousarray(np.concatenate(list(a), axis=1))
        Bh = np.ascontiguousarray(np.concatenate([O.im2col(np.ascontiguousarray(self.x[b]), self.ishape, self.kshape, self.padding,
                                                           self.strides).T for b in range(n)], axis=0))
        return Ah, Bh


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_batch_reduced_product_over_im2col(path, geom):
    """each geometry with one variant (they take turns), so that every variant meets several geometries"""
    op, alpha, beta = list(VARIANTS.values())[list(GEOMS).index(geom) % len(VARIANTS)]
    g = Grad(*GEOMS[geom])
    got, _ = g.fused(PATHS[path], op, alpha, beta)
    assert_bits(got, g.unfused(PATHS[path], op, alpha, beta))
    if beta == 0.0:
        assert not np.isnan(got).any()


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("path", list(PATHS))
def test_ops_and_scalars_bit_identical(path, variant):
    """every op with the forward output as aux (relu', tanh', sigmoid'), alpha != 1, beta = 1.25 over a seeded dW and beta = 0
    over a NaN-filled one"""
    g = Grad(*GEOMS["stride2"], seed=5)
    got, _ = g.fused(PATHS[path], *VARIANTS[variant])
    assert_bits(got, g.unfused(PATHS[path], *VARIANTS[variant]))


def test_exact_path_matches_the_oracle_over_the_concatenation():
    g = Grad(*GEOMS["non_square_3x5"], seed=9)
    got, _ = g.fused(L.PATH_SIMT, "relu_grad", 0.5, 0.75)
    Ah, Bh = g.concatenated("relu_grad")
    cout, K = g.kshape[0], Ah.shape[1]
    want = g.w0.copy()
    O.gemm_strided(cout, g.Kc, K, 0.5, Ah, K, 1, Bh, g.Kc, 1, 0.75, want, g.Kc, 1)
    assert_bits(got, want)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound_against_torch(path):
    """signed data, every image and channel of X and every output channel of dY at its own power-of-two scale; the concatenated
    operands' float64 product is torch.nn.grad.conv2d_weight's"""
    torch = pytest.importorskip("torch")
    ishape, kshape = ((2, 4, 10, 10), (16, 4, 3, 3)) if EMU else ((8, 32, 28, 28), (64, 32, 3, 3))
    rng = np.random.default_rng(11)
    n, C = ishape[:2]
    x = rng.uniform(-1, 1, ishape) * 2.0 ** rng.integers(-6, 7, n)[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, C)[None, :, None, None]
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, (1, 1), (1, 1)))
    dy = rng.uniform(-1, 1, oshape) * 2.0 ** rng.integers(-6, 7, kshape[0])[None, :, None, None]
    g = Grad(ishape, kshape, (1, 1), (1, 1), x=x.astype(np.float32), dy=dy.astype(np.float32))
    got, _ = g.fused(PATHS[path])
    Ah, Bh = g.concatenated()
    ref = torch.nn.grad.conv2d_weight(torch.from_numpy(g.x.astype(np.float64)), kshape, torch.from_numpy(g.dy.astype(np.float64)),
                                      padding=1).numpy().reshape(kshape[0], g.Kc)
    np.testing.assert_allclose(Ah.astype(np.float64) @ Bh.astype(np.float64), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    ks, _ = plan(path, kshape[0], g.Kc, Ah.shape[1])
    bound_and_check("conv filter gradient", path, "conv_filter_grad", got.reshape(kshape[0], g.Kc), Ah, Bh, 1.0, splits=ks)


@pytest.mark.skipif(EMU, reason="a K' long enough to split is slow on the CPU build")
@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
def test_layer_shape_splits_k(path):
    """Cout 64 x Kc 576 is five output tiles: the plan splits the 25088-long K', the reduce kernel is one more launch"""
    g = Grad((32, 64, 28, 28), (64, 64, 3, 3), (1, 1), (1, 1), seed=13)
    ks, _ = plan(path, 64, 576, 32 * 784)
    assert ks >= 2, "the shape must split K"
    got, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.5)
    # A: one concatenating row pass; B: f16x3 the abs-max and the split pass, tf32x3 one pass; the GEMM; the reduce
    assert n == {"f16x3": 3, "tf32x3": 2}[path] + 2
    assert_bits(got, g.unfused(PATHS[path], "relu_grad", 1.0, 0.5))


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1", "simt"])
def test_launch_count_does_not_grow_with_the_images(path):
    ishape, kshape, padding, strides = GEOMS["pad1"]
    counts = []
    for imgs in (1, 4 if EMU else 16):
        g = Grad((imgs,) + ishape[1:], kshape, padding, strides)
        _, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.0)
        P = g.P
        ks = plan(path, kshape[0], g.Kc, imgs * P)[0] if path != "simt" else 1
        counts.append(n - (1 if ks > 1 else 0))   # (a split adds the reduce kernel)
    # the gradients' row pass (a gather when P is not a multiple of 4), the images' tap-row passes (f16x3: abs-max and split),
    # the product
    assert counts[0] == counts[1] == {"f16x3": 4, "tf32x3": 3, "tf32x1": 3, "simt": 3}[path], counts


# the profiler session runs in a process of its own: the check does not depend on what ran before it in the test process,
# and the test process keeps one CUDA profiler session only (tests/test_gpu_conv_fused.py's)
_PROFILE = """
import torch, test_gpu_conv_filter_grad as T, laser_b200 as L
g = T.Grad(*T.GEOMS["pad1"])
g.fused(L.PATH_F16X3)
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    g.fused(L.PATH_F16X3)
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print("KERNEL", e.name)
"""


@pytest.mark.skipif(EMU, reason="torch.profiler needs the GPU")
def test_no_im2col_kernel_is_launched():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]))
    out = subprocess.run([sys.executable, "-c", _PROFILE], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    names = [line[len("KERNEL "):] for line in out.stdout.splitlines() if line.startswith("KERNEL ")]
    assert any("im2col_tap_rows_kernel" in n for n in names), names
    assert not any("im2col_kernel" in n or "im2col_rows_kernel" in n for n in names), names


@pytest.mark.parametrize("path", list(PATHS))
def test_one_by_one_reads_the_images_in_place(path):
    """a 1 x 1 kernel with unit strides and no padding is the batch-reduced product over the images themselves"""
    ishape, kshape = ((3, 8, 6, 6), (16, 8, 1, 1)) if EMU else ((4, 64, 14, 14), (128, 64, 1, 1))
    g = Grad(ishape, kshape, (0, 0), (1, 1), seed=17)
    got, n_fused = g.fused(PATHS[path], "sigmoid_grad", 1.5, 1.25)
    n, C, cout, P = ishape[0], ishape[1], kshape[0], g.P
    dw = g.dw0(1.25)
    sync()
    n0 = L.launch_count()
    L.gemm_strided_batch_reduce_fused(n, cout, C, P, 1.5, g.tdy, P, 1, cout * P, g.tx, 1, P, C * P, 1.25, dw, C, 1,
                                      path=PATHS[path], op_a=g.op_a("sigmoid_grad"))
    sync()
    assert n_fused == L.launch_count() - n0
    assert_bits(got, dw.cpu().numpy())


def _raw(ishape=(2, 2, 5, 5), kshape=(3, 2, 3, 3), padding=(1, 1), strides=(1, 1), op=None, path=L.PATH_AUTO, null=None):
    dw = dev(np.full(3 * 2 * 9, 3.0, np.float32))
    x, dy = dev(np.ones(2 * 2 * 25, np.float32)), dev(np.ones(2 * 3 * 25, np.float32))
    ptrs = {"dw": dw.data_ptr(), "x": x.data_ptr(), "dy": dy.data_ptr()}
    if null:
        ptrs[null] = None
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_conv2d_filter_grad_f32_fused_dev(ptrs["dw"], ptrs["x"], i4(*ishape), ptrs["dy"], i4(*kshape),
                                                                 i2(*padding), i2(*strides), 1.0, 0.0, op, path,
                                                                 G._current_stream())
    sync()
    assert np.all(dw.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    aux = dev(np.ones(2 * 3 * 25, np.float32))
    relu_grad = lambda rs, cs: ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD, aux=aux.data_ptr(), auxRowStride=rs,
                                                            auxColStride=cs))
    for kw in (dict(path=5), dict(path=-1), dict(op=ctypes.byref(_capi.OperandOp(op=9))),
               dict(op=ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))), dict(op=relu_grad(26, 1)), dict(op=relu_grad(25, 2)),
               dict(op=relu_grad(1, 25)), dict(kshape=(3, 1, 3, 3)), dict(strides=(0, 1)), dict(padding=(-1, 0)),
               dict(kshape=(3, 2, 8, 3)), dict(null="dw"), dict(null="x"), dict(null="dy")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    assert _raw(ishape=(0, 2, 5, 5)) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 2, 5, 5), null="dw") == (_capi.E_OK, 0)
    # n * outH * outW = 2^30 * 4 past int32 on a tensor-core path (nothing is read: the check comes first)
    assert _raw(ishape=(2 ** 30, 2, 4, 4), padding=(0, 0), path=L.PATH_F16X3) == (_capi.E_UNSUPPORTED, 0)
