"""GPU: the channels-last convolution's filter gradient laser_b200_conv2d_nhwc_filter_grad_f32_fused_dev -- NHWC images x and
output gradients dY, the filter matrix dWmat [kH * kW * c_in][c_out] written through its strides, ONE product
dWmat^T <- alpha * op(dY)^T * T^T + beta * dWmat^T whose B (the tap rows T [K][n * P], the NHWC forward's windows transposed) is
prepared straight from the images.  On every path dW must equal, bit for bit, the fused GEMM over T materialised in numpy with
the same A view, op and C strides; the exact path equals the CPU oracle and the NCHW filter-gradient entry on the same data,
permuted; the tensor-core paths meet the per-element bound of tests/test_gpu_error_bounds.py against
torch.nn.grad.conv2d_weight in float64; a layer shape splits K'; the launch count does not grow with the images; no im2col or
transpose kernel runs; argument errors launch nothing."""
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
# (ishape (n, c, h, w), kshape (c_out, c_in, kH, kW), padding, strides): the NHWC forward test's geometries and a single image
GEOMS = {
    "pad1": ((2, 8, 8, 8), (16, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 64, 20, 20), (64, 64, 3, 3), (1, 1), (1, 1)),
    "stride2": ((2, 4, 9, 9), (12, 4, 3, 3), (0, 0), (2, 2)) if EMU else ((5, 32, 17, 17), (48, 32, 3, 3), (0, 0), (2, 2)),
    "non_square": ((2, 4, 7, 9), (8, 4, 3, 5), (1, 2), (1, 2)) if EMU else ((3, 16, 16, 19), (32, 16, 3, 5), (1, 2), (2, 1)),
    # c = 3: the scalar path (K = 27, below one tile of taps)
    "rgb_c3": ((2, 3, 10, 10), (16, 3, 3, 3), (1, 1), (2, 2)) if EMU else ((4, 3, 32, 32), (64, 3, 3, 3), (1, 1), (2, 2)),
    # c = 5 (scalar path), c_out odd: A = dY^T is not a 16-byte-strided view and is gathered
    "c5_cout_odd": ((2, 5, 7, 6), (9, 5, 3, 2), (1, 0), (1, 1)) if EMU else ((3, 5, 15, 14), (15, 5, 3, 2), (1, 0), (1, 1)),
    "one_by_one_stride2": ((2, 8, 7, 7), (12, 8, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 32, 15, 15), (64, 32, 1, 1), (0, 0), (2, 2)),
    # K = 1152
    "long_k": ((1, 128, 4, 4), (8, 128, 3, 3), (1, 1), (1, 1)) if EMU else ((2, 128, 12, 12), (64, 128, 3, 3), (1, 1), (1, 1)),
    "single_image": ((1, 4, 8, 8), (8, 4, 3, 3), (1, 1), (1, 1)) if EMU else ((1, 16, 24, 24), (32, 16, 3, 3), (1, 1), (1, 1)),
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dW (never read), beta != 0 over a seeded one
VARIANTS = {"plain": (None, 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 1.0, 1.25)}
# the filter matrix's two layouts: kernel_to_hwcc's [kH][kW][C_in][C_out] and torch's channels_last weight [c_out][kH][kW][c_in]
LAYOUTS = ["hwio", "ohwi"]


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def up(x, m):
    return -(-x // m) * m


def tap_rows(x, ishape, kshape, padding, strides):
    """[kH * kW * c][n * outH * outW]: the NHWC forward's window rows of the images x, transposed"""
    n, C, H, W = ishape
    kH, kW = kshape[2:]
    (pH, pW), (sH, sW) = padding, strides
    oh, ow = 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW
    xp = np.zeros((n, H + 2 * pH, W + 2 * pW, C), x.dtype)
    xp[:, pH:pH + H, pW:pW + W] = x
    hi = (np.arange(oh) * sH)[:, None] + np.arange(kH)[None, :]
    wi = (np.arange(ow) * sW)[:, None] + np.arange(kW)[None, :]
    return np.ascontiguousarray(xp[:, hi[:, None, :, None], wi[None, :, None, :], :].reshape(n * oh * ow, kH * kW * C).T)


class Grad:
    """one filter gradient's data: NHWC images x [n][h][w][c], NHWC output gradients dy [n * P][c_out], the forward output z an
    op's aux is taken from (NHWC like dy), and dW0 as the filter matrix [K][c_out]"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, x=None, dy=None):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        n, C, H, W = ishape
        co, _, kH, kW = kshape
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        self.P, self.K, self.co = self.oshape[2] * self.oshape[3], kH * kW * C, co
        self.J = n * self.P
        self.x = O.fill_uniform_f32(n * H * W * C, seed, -1, 1).reshape(n, H, W, C) if x is None else x
        self.dy = O.fill_uniform_f32(self.J * co, seed + 1, -1, 1).reshape(self.J, co) if dy is None else dy
        z = O.fill_uniform_f32(self.J * co, seed + 2, -2, 2).reshape(self.J, co)
        self.aux = {"relu_grad": np.maximum(z, 0), "tanh_grad": np.tanh(z), "sigmoid_grad": 1 / (1 + np.exp(-z))}
        self.w0 = O.fill_uniform_f32(self.K * co, seed + 3, -1, 1).reshape(self.K, co)
        self.tx, self.tdy = dev(self.x), dev(self.dy)
        self.taux = {k: dev(v.astype(np.float32)) for k, v in self.aux.items()}

    def dw0(self, beta, layout):
        """-> (the device buffer, the [K][c_out] view the entry takes, its element strides)"""
        w = self.w0 if beta != 0.0 else np.full(self.w0.shape, np.nan, np.float32)
        if layout == "hwio":
            buf = dev(w)
            return buf, buf, (self.co, 1)
        buf = dev(np.ascontiguousarray(w.T))   # [c_out][K]
        return buf, (buf if EMU else buf.t()), (1, self.K)

    def as_wmat(self, buf, layout):
        h = buf.cpu().numpy().copy()
        return h.reshape(self.K, self.co) if layout == "hwio" else np.ascontiguousarray(h.reshape(self.co, self.K).T)

    def fused(self, path, op=None, alpha=1.0, beta=0.0, layout="hwio"):
        """-> (dWmat [K][c_out], launches)"""
        buf, view, st = self.dw0(beta, layout)
        sync()
        n0 = L.launch_count()
        L.conv2d_nhwc_filter_grad_fused(view, self.tx, self.ishape, self.tdy, self.kshape, self.padding, self.strides, alpha, beta,
                                        op=op, aux=self.taux.get(op), path=path, kernel_strides=st if EMU else None)
        sync()
        return self.as_wmat(buf, layout), L.launch_count() - n0

    def op_a(self, op):
        if op is None or op not in self.taux:
            return op
        return (op, self.taux[op], 1, self.co)

    def taps(self):
        return tap_rows(self.x, self.ishape, self.kshape, self.padding, self.strides)

    def gemm(self, path, op=None, alpha=1.0, beta=0.0, layout="hwio"):
        """the fused GEMM over the tap rows materialised in numpy, [K][round_up(n * P, 4)], with the same A view and C strides"""
        ld = up(self.J, 4)
        t = np.zeros((self.K, ld), np.float32)
        t[:, :self.J] = self.taps()
        buf, _, (rs, cs) = self.dw0(beta, layout)
        G.gemm_strided_fused(self.co, self.K, self.J, alpha, self.tdy, 1, self.co, dev(t), 1, ld, beta, buf, cs, rs, path=path,
                             op_a=self.op_a(op))
        sync()
        return self.as_wmat(buf, layout)

    def a_rows(self, op=None):
        """op(dY)^T as multiplied, [c_out][n * P]"""
        a = self.dy.astype(np.float32)
        if op == "relu_grad":
            a = np.where(self.aux[op] > 0, a, np.float32(0))
        return np.ascontiguousarray(a.T)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_gemm_over_the_tap_rows(path, geom, layout):
    """each geometry with one variant (they take turns); PATH_AUTO: the GEMM on the path the entry resolved"""
    op, alpha, beta = list(VARIANTS.values())[list(GEOMS).index(geom) % len(VARIANTS)]
    g = Grad(*GEOMS[geom])
    got, _ = g.fused(PATHS[path], op, alpha, beta, layout)
    resolved = L.last_path()
    if path != "auto":
        assert resolved == PATHS[path]
    if beta == 0.0:
        assert not np.isnan(got).any()
    assert_bits(got, g.gemm(resolved, op, alpha, beta, layout))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("path", list(PATHS))
def test_ops_and_scalars_bit_identical(path, variant):
    """every op with the forward output as aux (relu', tanh', sigmoid'), alpha != 1, beta = 1.25 over a seeded dW and beta = 0
    over a NaN-filled one"""
    g = Grad(*GEOMS["stride2"], seed=5)
    got, _ = g.fused(PATHS[path], *VARIANTS[variant], layout="ohwi")
    assert_bits(got, g.gemm(L.last_path(), *VARIANTS[variant], layout="ohwi"))


@pytest.mark.parametrize("geom", list(GEOMS))
def test_auto_takes_the_path_of_the_nchw_entry(geom):
    g = Grad(*GEOMS[geom], seed=3)
    g.fused(L.PATH_AUTO)
    nhwc = L.last_path()
    dw = dev(np.zeros(g.co * g.K, np.float32))
    L.conv2d_filter_grad_fused(dw, dev(np.ascontiguousarray(g.x.transpose(0, 3, 1, 2))), g.ishape,
                               dev(np.ascontiguousarray(g.dy.reshape(g.ishape[0], g.P, g.co).transpose(0, 2, 1))), g.kshape,
                               g.padding, g.strides, path=L.PATH_AUTO)
    sync()
    assert nhwc == L.last_path()


def nchw_filter_grad(g, path, op, alpha, beta):
    """the NCHW filter-gradient entry on NCHW copies of the same data -> its dW permuted to the filter matrix [K][c_out]"""
    n, C, H, W = g.ishape
    co, _, kH, kW = g.kshape
    to_nchw = lambda a: np.ascontiguousarray(a.reshape(n, g.P, co).transpose(0, 2, 1))
    w0 = np.ascontiguousarray(g.w0.reshape(kH, kW, C, co).transpose(3, 2, 0, 1))
    dw = dev(w0 if beta != 0.0 else np.full(w0.shape, np.nan, np.float32))
    L.conv2d_filter_grad_fused(dw, dev(np.ascontiguousarray(g.x.transpose(0, 3, 1, 2))), g.ishape, dev(to_nchw(g.dy)), g.kshape,
                               g.padding, g.strides, alpha, beta, op=op, aux=dev(to_nchw(g.aux[op])) if op else None, path=path)
    sync()
    return np.ascontiguousarray(dw.cpu().numpy().reshape(co, C, kH, kW).transpose(2, 3, 1, 0).reshape(g.K, co))


@pytest.mark.parametrize("geom", ["non_square", "rgb_c3", "c5_cout_odd"])
def test_exact_path_matches_the_oracle_and_the_nchw_entry(geom):
    """the CPU oracle over (op(dY)^T, T^T); and the NCHW entry's exact path on the same data, permuted: the same values summed
    in the same order over n * P + p, bit for bit"""
    g = Grad(*GEOMS[geom], seed=9)
    got, _ = g.fused(L.PATH_SIMT, "relu_grad", 0.5, 0.75, layout="ohwi")
    a, t = g.a_rows("relu_grad"), g.taps()
    want = g.w0.copy()   # C[co][k] at k * c_out + co
    O.gemm_strided(g.co, g.K, g.J, 0.5, a, g.J, 1, t, 1, g.J, 0.75, want, 1, g.co)
    assert_bits(got, want)
    assert_bits(got, nchw_filter_grad(g, L.PATH_SIMT, "relu_grad", 0.5, 0.75))


def scaled_grad(ishape, kshape, padding, strides, seed):
    """signed data: every image and channel of x and every output channel of dY at its own power of two"""
    n, C, H, W = ishape
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, H, W, C)) * 2.0 ** rng.integers(-6, 7, n)[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, C)[None, None, None, :]
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
    dy = rng.uniform(-1, 1, (n * oshape[2] * oshape[3], kshape[0])) * 2.0 ** rng.integers(-6, 7, kshape[0])[None, :]
    return Grad(ishape, kshape, padding, strides, x=x.astype(np.float32), dy=dy.astype(np.float32))


BOUND_GEOMS = {"layer": ((2, 4, 10, 10), (16, 4, 3, 3), (1, 1), (1, 1)) if EMU else ((8, 32, 28, 28), (64, 32, 3, 3), (1, 1), (1, 1)),
               "rgb_c3": GEOMS["rgb_c3"], "c5_cout_odd": GEOMS["c5_cout_odd"]}


@pytest.mark.parametrize("geom", list(BOUND_GEOMS))
@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound_against_torch(path, geom):
    """the operands' float64 product is torch.nn.grad.conv2d_weight's, permuted to the filter matrix"""
    ishape, kshape, padding, strides = BOUND_GEOMS[geom]
    g = scaled_grad(ishape, kshape, padding, strides, 11)
    got, _ = g.fused(PATHS[path], layout="ohwi")
    A, B = g.a_rows(), np.ascontiguousarray(g.taps().T)
    if not EMU:
        torch = pytest.importorskip("torch")
        n, C, H, W = ishape
        co, _, kH, kW = kshape
        ref = torch.nn.grad.conv2d_weight(torch.from_numpy(g.x.astype(np.float64)).permute(0, 3, 1, 2), kshape,
                                          torch.from_numpy(g.dy.astype(np.float64)).reshape(n, g.oshape[2], g.oshape[3], co)
                                          .permute(0, 3, 1, 2), stride=strides, padding=padding)
        ref = ref.permute(0, 2, 3, 1).reshape(co, g.K).numpy()
        np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    ks, _ = plan(path, g.co, g.K, g.J)
    bound_and_check("conv nhwc filter gradient", path, "conv_nhwc_filter_grad", np.ascontiguousarray(got.T), A, B, 1.0, splits=ks)


@pytest.mark.skipif(EMU, reason="a K' long enough to split is slow on the CPU build")
@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
def test_layer_shape_splits_k(path):
    """c_out 64 x K 576 is five output tiles: the plan splits the 25088-long K', the reduce kernel is one more launch"""
    g = Grad((32, 64, 28, 28), (64, 64, 3, 3), (1, 1), (1, 1), seed=13)
    ks, _ = plan(path, 64, 576, 32 * 784)
    assert ks >= 2, "the shape must split K"
    got, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.5)
    # A = dY^T, MN-major: f16x3 its column abs-max and split passes in place, tf32x3 one gather; B: f16x3 the abs-max and the
    # split pass, tf32x3 one pass; the GEMM; the reduce
    assert n == {"f16x3": 6, "tf32x3": 4}[path]
    assert_bits(got, g.gemm(PATHS[path], "relu_grad", 1.0, 0.5))


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1", "simt"])
def test_launch_count_does_not_grow_with_the_images(path):
    ishape, kshape, padding, strides = GEOMS["pad1"]
    counts = []
    for imgs in (1, 3 if EMU else 16):
        g = Grad((imgs,) + ishape[1:], kshape, padding, strides)
        _, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.0)
        ks = plan(path, g.co, g.K, g.J)[0] if path != "simt" else 1
        counts.append(n - (1 if ks > 1 else 0))   # (a split adds the reduce kernel)
    # A: f16x3 two passes over dY in place, otherwise one gather applying the op; B: the tap-row passes (f16x3: abs-max and
    # split); the product
    assert counts[0] == counts[1] == {"f16x3": 5, "tf32x3": 3, "tf32x1": 3, "simt": 3}[path], counts


# the profiler session runs in a process of its own: the check does not depend on what ran before it in the test process
_PROFILE = """
import torch, test_gpu_conv_nhwc_filter_grad as T, laser_b200 as L
g = T.Grad(*T.GEOMS["pad1"])
for path in (L.PATH_F16X3, L.PATH_TF32X3):
    g.fused(path, "relu_grad")
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for path in (L.PATH_F16X3, L.PATH_TF32X3):
        g.fused(path, "relu_grad")
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print("KERNEL", e.name)
"""


@pytest.mark.skipif(EMU, reason="torch.profiler needs the GPU")
def test_no_im2col_or_transpose_kernel_is_launched():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]))
    out = subprocess.run([sys.executable, "-c", _PROFILE], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    names = [line[len("KERNEL "):] for line in out.stdout.splitlines() if line.startswith("KERNEL ")]
    assert any("im2col_nhwc_tap_rows_kernel" in n for n in names), names
    assert not any("im2col_kernel" in n or "im2col_rows_kernel" in n or "transpose" in n.lower() for n in names), names


@pytest.mark.parametrize("path", list(PATHS))
def test_one_by_one_reads_the_images_in_place(path):
    """1 x 1, unit strides, no padding: the fused GEMM over the images read in place as [c][n * h * w] -- same bits, same
    launches (no tap-row pass)"""
    ishape, kshape = ((2, 8, 6, 6), (12, 8, 1, 1)) if EMU else ((4, 64, 14, 14), (128, 64, 1, 1))
    g = Grad(ishape, kshape, (0, 0), (1, 1), seed=17)
    got, n_fused = g.fused(PATHS[path], "sigmoid_grad", 1.5, 1.25, layout="ohwi")
    resolved = L.last_path()
    buf, _, (rs, cs) = g.dw0(1.25, "ohwi")
    sync()
    n0 = L.launch_count()
    G.gemm_strided_fused(g.co, g.K, g.J, 1.5, g.tdy, 1, g.co, g.tx, g.K, 1, 1.25, buf, cs, rs, path=resolved,
                         op_a=g.op_a("sigmoid_grad"))
    sync()
    assert n_fused == L.launch_count() - n0
    assert_bits(got, g.as_wmat(buf, "ohwi"))


def _raw(ishape=(2, 2, 5, 5), kshape=(3, 2, 3, 3), padding=(1, 1), strides=(1, 1), kstrides=(3, 1), op=None, path=L.PATH_AUTO,
         null=None):
    dw = dev(np.full(18 * 3, 3.0, np.float32))
    x, dy = dev(np.ones(2 * 25 * 2, np.float32)), dev(np.ones(2 * 25 * 3, np.float32))
    ptrs = {"dw": dw.data_ptr(), "x": x.data_ptr(), "dy": dy.data_ptr()}
    if null:
        ptrs[null] = None
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    fn = _capi.lib().laser_b200_conv2d_nhwc_filter_grad_f32_fused_dev
    if kstrides is None:   # a NULL kernelStrides: the same symbol through a handle whose argtypes take a plain pointer there
        fn = ctypes.CDLL(_capi.lib()._name).laser_b200_conv2d_nhwc_filter_grad_f32_fused_dev
        fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, i4, ctypes.c_void_p, i4, ctypes.c_void_p, i2, i2, ctypes.c_float,
                       ctypes.c_float, ctypes.POINTER(_capi.OperandOp), ctypes.c_int, ctypes.c_void_p]
    rc = fn(ptrs["dw"], ptrs["x"], i4(*ishape), ptrs["dy"], i4(*kshape), i2(*kstrides) if kstrides else None, i2(*padding),
            i2(*strides), 1.0, 0.0, op, path, G._current_stream())
    sync()
    assert np.all(dw.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    aux = dev(np.ones(2 * 25 * 3, np.float32))
    relu_grad = lambda rs, cs: ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD, aux=aux.data_ptr(), auxRowStride=rs,
                                                            auxColStride=cs))
    for kw in (dict(path=5), dict(path=-1), dict(op=ctypes.byref(_capi.OperandOp(op=9))),
               dict(op=ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))), dict(op=relu_grad(3, 1)), dict(op=relu_grad(1, 4)),
               dict(op=relu_grad(25, 1)), dict(kstrides=None), dict(kshape=(3, 1, 3, 3)), dict(strides=(0, 1)),
               dict(padding=(-1, 0)), dict(kshape=(3, 2, 8, 3)), dict(null="dw"), dict(null="x"), dict(null="dy")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    assert _raw(ishape=(0, 2, 5, 5)) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 2, 5, 5), null="dw") == (_capi.E_OK, 0)
    # n * outH * outW = 2^30 * 4 past int32 on a tensor-core path (nothing is read: the check comes first)
    assert _raw(ishape=(2 ** 30, 2, 4, 4), padding=(0, 0), path=L.PATH_F16X3) == (_capi.E_UNSUPPORTED, 0)


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode of this file's bound checks (the last test of the file)"""
    from test_gpu_error_bounds import RATIOS
    mine = {k: r for k, r in RATIOS.items() if k[1] == "conv_nhwc_filter_grad"}
    if not mine:
        pytest.skip("no case ran")
    with capsys.disabled():
        print("\nlargest err / bound of the NHWC filter gradient:\n" +
              "\n".join("  %-7s %.3g" % (m, r) for (m, _), r in sorted(mine.items())))
