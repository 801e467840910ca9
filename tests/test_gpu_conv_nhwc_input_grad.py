"""GPU: the channels-last convolution's input gradient laser_b200_conv2d_nhwc_input_grad_f32_fused_dev -- NHWC output gradients
dY, the filter matrix Wmat [kH * kW * c_in][c_out] read through its strides, ONE product dX <- alpha * R * W'^T + beta * dX per
chunk of whole images, whose A (the input pixels' windows R over op(dY) zero-dilated by the strides, in (kh', kw', co) order) is
prepared straight from dY.  On every path dX must equal, bit for bit, the fused GEMM over R materialised in numpy (holes 0) and
W'^T; at stride 1 with pH <= kH - 1 the NHWC forward entry over (dY, W'^T, kH - 1 - pH); the exact path equals the CPU oracle;
the tensor-core paths meet the per-element bound of tests/test_gpu_error_bounds.py against torch.nn.grad.conv2d_input in
float64; a channels-last layer's whole backward pass matches torch autograd; 1 x 1 kernels read dY in place; the launch count
does not grow with the images, and chunks give the bits of one; argument errors launch nothing."""
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
# forward geometries (ishape (n, c_in, h, w), kshape (c_out, c_in, kH, kW), padding, strides)
GEOMS = {
    "pad1": ((3, 8, 10, 10), (16, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 48, 20, 20), (64, 48, 3, 3), (1, 1), (1, 1)),
    # (8 - 3) mod 2 = 1: the last input row and column lie in no window
    "stride2_tail": ((2, 4, 8, 8), (8, 4, 3, 3), (0, 0), (2, 2)) if EMU else ((5, 24, 8, 8), (40, 24, 3, 3), (0, 0), (2, 2)),
    "non_square_3x5": ((2, 3, 8, 9), (8, 3, 3, 5), (1, 2), (1, 2)) if EMU else ((3, 16, 16, 19), (32, 16, 3, 5), (1, 2), (1, 2)),
    "one_by_one_stride2": ((3, 6, 7, 7), (8, 6, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 32, 15, 15), (64, 32, 1, 1), (0, 0), (2, 2)),
    # p' = kH - 1 - pH = -1
    "one_by_one_pad1": ((2, 6, 5, 6), (8, 6, 1, 1), (1, 1), (1, 1)) if EMU else ((3, 32, 14, 13), (64, 32, 1, 1), (1, 1), (1, 1)),
    # c_out = 3 and 5: the scalar path
    "cout3": ((2, 4, 7, 7), (3, 4, 3, 3), (1, 1), (2, 2)) if EMU else ((4, 32, 15, 15), (3, 32, 3, 3), (1, 1), (2, 2)),
    "cout5": ((2, 4, 7, 6), (5, 4, 3, 2), (1, 0), (1, 1)) if EMU else ((3, 16, 15, 14), (5, 16, 3, 2), (1, 0), (1, 1)),
    "single_image": ((1, 4, 8, 8), (8, 4, 3, 3), (1, 1), (1, 1)) if EMU else ((1, 16, 24, 24), (32, 16, 3, 3), (1, 1), (1, 1)),
    # n * H * W = 147 / 405: not a multiple of 4
    "odd_pixels": ((3, 2, 7, 7), (8, 2, 3, 3), (0, 0), (1, 1)) if EMU else ((5, 16, 9, 9), (32, 16, 3, 3), (0, 0), (1, 1)),
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dX (never read), beta != 0 over a seeded one
VARIANTS = {"plain": (None, 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 1.0, 1.25), "sigmoid": ("sigmoid", 0.75, 0.0), "relu": ("relu", 1.0, 1.25),
            "tanh": ("tanh", 1.5, 0.0)}
# the filter matrix's two layouts: kernel_to_hwcc's [kH][kW][C_in][C_out] and torch's channels_last weight [c_out][kH][kW][c_in]
LAYOUTS = ["hwio", "ohwi"]


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def up(x, m):
    return -(-x // m) * m


def tconv_rows(z, ishape, kshape, padding, strides):
    """[n * H * W][kH * kW * c_out] rows over z [n][outH][outW][c_out]: input pixel (ih, iw)'s window zero-dilated by the strides
    and padded by kH - 1 - pH, in (kh', kw', co) order; 0 wherever a tap falls between, before or past z's rows and columns"""
    n, _, H, W = ishape
    co, _, kH, kW = kshape
    oh, ow = z.shape[1:3]

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, padding[0], strides[0], oh)
    wq, vw = axis(W, kW, padding[1], strides[1], ow)
    g = z[:, hq[:, None, :, None], wq[None, :, None, :], :]
    ok = (vh[:, None, :, None] & vw[None, :, None, :])[None, :, :, :, :, None]
    return np.ascontiguousarray(np.where(ok, g, np.zeros((), z.dtype)).reshape(n * H * W, kH * kW * co))


def lib_op(name, x, aux=None):
    """op(x) elementwise with the library's own op (aux: a derivative's): the exact path's product of op(x) with the identity"""
    flat = np.ascontiguousarray(x.reshape(-1, x.shape[-1]), np.float32)
    R, Cc = flat.shape
    out = dev(np.zeros_like(flat))
    op = name if aux is None else (name, dev(np.ascontiguousarray(aux.reshape(R, Cc), np.float32)), Cc, 1)
    G.gemm_strided_fused(R, Cc, Cc, 1.0, dev(flat), Cc, 1, dev(np.eye(Cc, dtype=np.float32)), Cc, 1, 0.0, out, Cc, 1,
                         path=L.PATH_SIMT, op_a=op)
    sync()
    return out.cpu().numpy().reshape(x.shape).copy()


class Grad:
    """one input gradient's data: the filter matrix Wmat [K][c_out], NHWC output gradients dy [n][outH][outW][c_out], the
    forward output z an op's aux is taken from (NHWC like dy), and dX0 [n * H * W][c_in]"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, wmat=None, dy=None):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        n, C, H, W = ishape
        co, _, kH, kW = kshape
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        oh, ow = self.oshape[2:]
        self.C, self.co, self.T, self.K = C, co, kH * kW, kH * kW * C
        self.Kp, self.R = kH * kW * co, n * H * W
        self.wmat = O.fill_uniform_f32(self.K * co, seed, -1, 1).reshape(self.K, co) if wmat is None else wmat
        self.dy = O.fill_uniform_f32(n * oh * ow * co, seed + 1, -1, 1).reshape(n, oh, ow, co) if dy is None else dy
        z = O.fill_uniform_f32(n * oh * ow * co, seed + 2, -2, 2).reshape(n, oh, ow, co)
        self.aux = {"relu_grad": np.maximum(z, 0), "tanh_grad": np.tanh(z), "sigmoid_grad": 1 / (1 + np.exp(-z))}
        self.aux = {k: v.astype(np.float32) for k, v in self.aux.items()}
        self.x0 = O.fill_uniform_f32(self.R * C, seed + 3, -1, 1).reshape(self.R, C)
        self.tdy = dev(self.dy)
        self.taux = {k: dev(v) for k, v in self.aux.items()}

    def kernel(self, layout):
        """-> (the device buffer, the [K][c_out] view the entry takes, its element strides)"""
        if layout == "hwio":
            buf = dev(self.wmat)
            return buf, buf, (self.co, 1)
        buf = dev(np.ascontiguousarray(self.wmat.T))   # [c_out][K]
        return buf, (buf if EMU else buf.t()), (1, self.K)

    def wt(self):
        """W'^T [c_in][K']: W'^T[ci][t * c_out + co] = Wmat[(T - 1 - t) * c_in + ci][co]"""
        w = self.wmat.reshape(self.T, self.C, self.co)[::-1]
        return np.ascontiguousarray(w.transpose(1, 0, 2).reshape(self.C, self.Kp))

    def dx0(self, beta):
        return dev(self.x0 if beta != 0.0 else np.full(self.x0.shape, np.nan, np.float32))

    def fused(self, path, op=None, alpha=1.0, beta=0.0, layout="hwio"):
        """-> (dX [n * H * W][c_in], launches)"""
        dx = self.dx0(beta)
        _, view, st = self.kernel(layout)
        sync()
        n0 = L.launch_count()
        L.conv2d_nhwc_input_grad_fused(dx, self.ishape, self.tdy, view, self.kshape, self.padding, self.strides, alpha, beta, op=op,
                                       aux=self.taux.get(op), path=path, kernel_strides=st)
        sync()
        return dx.cpu().numpy().reshape(self.R, self.C).copy(), L.launch_count() - n0

    def rows(self, z):
        return tconv_rows(z, self.ishape, self.kshape, self.padding, self.strides)

    def a_rows(self, op=None):
        """R as multiplied: op(dY) with the library's own op at the source positions, holes 0"""
        z = self.dy if op is None else lib_op(op, self.dy, self.aux.get(op))
        return self.rows(z)

    def gemm(self, path, op=None, alpha=1.0, beta=0.0):
        """the fused GEMM over R materialised (op applied by the library, holes 0), [n * H * W][round_up(K', 4)], B = W'^T read
        K-major, C = dX with strides (c_in, 1)"""
        ld = up(self.Kp, 4)
        a = np.zeros((self.R, ld), np.float32)
        a[:, :self.Kp] = self.a_rows(op)
        b = np.zeros((self.C, ld), np.float32)
        b[:, :self.Kp] = self.wt()
        dx = self.dx0(beta)
        G.gemm_strided_fused(self.R, self.C, self.Kp, alpha, dev(a), ld, 1, dev(b), 1, ld, beta, dx, self.C, 1, path=path)
        sync()
        return dx.cpu().numpy().reshape(self.R, self.C).copy()


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_gemm_over_the_windows(path, geom, layout):
    """each geometry with one variant (they take turns); PATH_AUTO: the GEMM on the path the entry resolved"""
    op, alpha, beta = list(VARIANTS.values())[list(GEOMS).index(geom) % len(VARIANTS)]
    g = Grad(*GEOMS[geom])
    got, _ = g.fused(PATHS[path], op, alpha, beta, layout)
    resolved = L.last_path()
    if path != "auto":
        assert resolved == PATHS[path]
    if beta == 0.0:
        assert not np.isnan(got).any()
    assert_bits(got, g.gemm(resolved, op, alpha, beta))


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("path", ["simt", "f16x3", "tf32x3", "tf32x1"])
def test_ops_and_scalars_bit_identical(path, variant):
    """every op (derivatives with the forward output as aux), alpha != 1, beta = 1.25 over a seeded dX and beta = 0 over a
    NaN-filled one -- at stride 2, where the last row and column get beta * dX0 (or 0) only"""
    g = Grad(*GEOMS["stride2_tail"], seed=5)
    got, _ = g.fused(PATHS[path], *VARIANTS[variant], layout="ohwi")
    assert_bits(got, g.gemm(PATHS[path], *VARIANTS[variant]))
    n, C, H, W = g.ishape
    op, alpha, beta = VARIANTS[variant]
    tail = got.reshape(n, H, W, C)[:, H - 1]
    np.testing.assert_array_equal(tail, np.float32(beta) * g.x0.reshape(n, H, W, C)[:, H - 1] if beta else 0.0)


@pytest.mark.parametrize("geom", list(GEOMS))
def test_auto_takes_the_path_of_the_nchw_entry(geom):
    g = Grad(*GEOMS[geom], seed=3)
    g.fused(L.PATH_AUTO)
    nhwc = L.last_path()
    co, C, kH, kW = g.kshape
    w = np.ascontiguousarray(g.wmat.reshape(kH, kW, C, co).transpose(3, 2, 0, 1))
    dx = dev(np.zeros(g.R * C, np.float32))
    L.conv2d_input_grad_fused(dx, g.ishape, dev(np.ascontiguousarray(g.dy.transpose(0, 3, 1, 2))), dev(w), g.kshape, g.padding,
                              g.strides, path=L.PATH_AUTO)
    sync()
    assert nhwc == L.last_path()


@pytest.mark.parametrize("geom", ["pad1", "single_image", "odd_pixels", "cout5"])
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_nhwc_forward_entry(path, geom):
    """stride 1, pH <= kH - 1, no op: the forward call over (dY, W'^T as a [c_in][K'] buffer with kernelStrides (1, K'),
    padding kH - 1 - pH) is the same product"""
    ishape, kshape, padding, strides = GEOMS[geom]
    assert strides == (1, 1) and padding[0] <= kshape[2] - 1 and padding[1] <= kshape[3] - 1
    g = Grad(ishape, kshape, padding, strides, seed=7)
    got, _ = g.fused(PATHS[path])
    co, C, kH, kW = g.kshape
    out = dev(np.full(g.R * C, np.nan, np.float32))
    wt = dev(g.wt())
    L.conv2d_nhwc_fused(out, g.tdy, g.oshape, wt if EMU else wt.t(), (C, co, kH, kW), (kH - 1 - padding[0], kW - 1 - padding[1]),
                        (1, 1), path=PATHS[path], kernel_strides=(1, g.Kp))
    sync()
    assert_bits(got, out.cpu().numpy().reshape(g.R, C))


def f64_bound(A, B):
    """the float64 product and a bound for any fp32 summation order of it: (K + 1) * 2^-24 * |A| |B| (K the reduction length)"""
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    return A64 @ B64, (A.shape[1] + 1) * 2.0 ** -24 * (np.abs(A64) @ np.abs(B64)) + 1e-30


@pytest.mark.parametrize("geom", ["stride2_tail", "non_square_3x5", "cout5"])
def test_exact_path_matches_the_oracle(geom):
    """the CPU oracle over (R, W'^T), bit for bit.  The NCHW entry sums K' in (co, tap) order, this one in (tap, co) order: the
    two meet the same float64 bound, not each other's bits"""
    g = Grad(*GEOMS[geom], seed=9)
    got, _ = g.fused(L.PATH_SIMT, "relu_grad", 0.5, 0.75, layout="ohwi")
    a = np.ascontiguousarray(g.a_rows("relu_grad"))
    wt = g.wt()
    want = g.x0.copy()
    O.gemm_strided(g.R, g.C, g.Kp, 0.5, a, g.Kp, 1, wt, 1, g.Kp, 0.75, want, g.C, 1)
    assert_bits(got, want)
    n, C, H, W = g.ishape
    co, _, kH, kW = g.kshape
    w = np.ascontiguousarray(g.wmat.reshape(kH, kW, C, co).transpose(3, 2, 0, 1))
    dx = dev(np.ascontiguousarray(g.x0.reshape(n, H, W, C).transpose(0, 3, 1, 2)))
    L.conv2d_input_grad_fused(dx, g.ishape, dev(np.ascontiguousarray(g.dy.transpose(0, 3, 1, 2))), dev(w), g.kshape, g.padding,
                              g.strides, 0.5, 0.75, op="relu_grad", aux=dev(np.ascontiguousarray(g.aux["relu_grad"].transpose(0, 3, 1, 2))),
                              path=L.PATH_SIMT)
    sync()
    nchw = dx.cpu().numpy().reshape(n, C, H, W).transpose(0, 2, 3, 1).reshape(g.R, C)
    ab, bound = f64_bound(a, wt.T)
    ref = 0.5 * ab + 0.75 * g.x0.astype(np.float64)
    bound = 0.5 * bound + 2.0 ** -22 * (np.abs(0.5 * ab) + np.abs(0.75 * g.x0.astype(np.float64)))   # (+ the alpha, beta roundings)
    for res in (got, nchw):
        assert np.all(np.abs(res.astype(np.float64) - ref) <= bound)


def scaled_case(ishape, kshape, padding, strides, seed):
    """signed data: every image and channel of dY and every input channel of Wmat at its own power-of-two scale"""
    rng = np.random.default_rng(seed)
    n = ishape[0]
    co, C, kH, kW = kshape
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
    dy = rng.uniform(-1, 1, (n, oshape[2], oshape[3], co)) * 2.0 ** rng.integers(-6, 7, n)[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, co)[None, None, None, :]
    w = rng.uniform(-1, 1, (kH * kW, C, co)) * 2.0 ** rng.integers(-6, 7, C)[None, :, None]
    return Grad(ishape, kshape, padding, strides, wmat=w.reshape(kH * kW * C, co).astype(np.float32), dy=dy.astype(np.float32))


BOUND_GEOMS = ["pad1", "stride2_tail", "cout3"]


def torch_input_grad(g, dy):
    """torch.nn.grad.conv2d_input in float64 -> [n * H * W][c_in]"""
    torch = pytest.importorskip("torch")
    n, C, H, W = g.ishape
    co, _, kH, kW = g.kshape
    w = torch.from_numpy(g.wmat.astype(np.float64)).reshape(kH, kW, C, co).permute(3, 2, 0, 1)
    ref = torch.nn.grad.conv2d_input(g.ishape, w, torch.from_numpy(dy.astype(np.float64)).permute(0, 3, 1, 2), stride=g.strides,
                                     padding=g.padding)
    return ref.permute(0, 2, 3, 1).reshape(g.R, C).numpy()


@pytest.mark.parametrize("geom", BOUND_GEOMS)
@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound_against_torch(path, geom):
    g = scaled_case(*GEOMS[geom], seed=11)
    got, _ = g.fused(PATHS[path], layout="ohwi")
    A, B = g.a_rows(), np.ascontiguousarray(g.wt().T)
    if not EMU:
        ref = torch_input_grad(g, g.dy)
        np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    ks, _ = plan(path, g.R, g.C, g.Kp)
    bound_and_check("conv nhwc input gradient", path, "conv_nhwc_input_grad", got, A, B, 1.0, splits=ks)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_layer_backward_pass_against_torch_autograd(path):
    """conv2d_nhwc_fused with bias and relu, then dW and dX with relu_grad and the forward output as aux: against torch
    autograd of the convolution in float64 with the same relu mask, each within the bound"""
    torch = pytest.importorskip("torch")
    ishape, kshape, padding, strides = GEOMS["stride2_tail"]
    n, C, H, W = ishape
    co, _, kH, kW = kshape
    rng = np.random.default_rng(21)
    x = rng.uniform(-1, 1, (n, H, W, C)).astype(np.float32)
    wmat = rng.uniform(-1, 1, (kH * kW * C, co)).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, co).astype(np.float32)
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
    oh, ow = oshape[2:]
    dy = rng.uniform(-1, 1, (n, oh, ow, co)).astype(np.float32)
    tz = dev(np.zeros(n * oh * ow * co, np.float32))
    tw = dev(wmat)
    L.conv2d_nhwc_fused(tz, dev(x), ishape, tw, kshape, padding, strides, bias=dev(bias), activation="relu", path=PATHS[path],
                        kernel_strides=(co, 1))
    sync()
    z = tz.cpu().numpy().reshape(n, oh, ow, co).copy()
    g = Grad(ishape, kshape, padding, strides, wmat=wmat, dy=dy)
    dx = dev(np.full(g.R * C, np.nan, np.float32))
    dw = dev(np.full(g.K * co, np.nan, np.float32))
    L.conv2d_nhwc_input_grad_fused(dx, ishape, g.tdy, tw, kshape, padding, strides, op="relu_grad", aux=tz, path=PATHS[path],
                                   kernel_strides=(co, 1))
    L.conv2d_nhwc_filter_grad_fused(dw, dev(x), ishape, g.tdy, kshape, padding, strides, op="relu_grad", aux=tz, path=PATHS[path],
                                    kernel_strides=(co, 1))
    sync()
    gz = np.where(z > 0, dy, np.float32(0)).astype(np.float32)
    tx = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2).contiguous().requires_grad_()
    tk = torch.from_numpy(wmat.astype(np.float64)).reshape(kH, kW, C, co).permute(3, 2, 0, 1).contiguous().requires_grad_()
    y = torch.nn.functional.conv2d(tx, tk, torch.from_numpy(bias.astype(np.float64)), stride=strides, padding=padding)
    y.backward(torch.from_numpy(gz.astype(np.float64)).permute(0, 3, 1, 2))
    gx = tx.grad.permute(0, 2, 3, 1).reshape(g.R, C).numpy()
    gw = tk.grad.permute(2, 3, 1, 0).reshape(g.K, co).numpy()
    A, B = g.rows(gz), np.ascontiguousarray(g.wt().T)
    np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), gx, rtol=0, atol=1e-12 * np.abs(gx).max())
    bound_and_check("conv nhwc input gradient", path, "conv_nhwc_input_grad", dx.cpu().numpy().reshape(g.R, C), A, B, 1.0,
                    splits=plan(path, g.R, C, g.Kp)[0])
    J = n * oh * ow
    xp = np.zeros((n, H + 2 * padding[0], W + 2 * padding[1], C), np.float32)
    xp[:, padding[0]:padding[0] + H, padding[1]:padding[1] + W] = x
    hi = (np.arange(oh) * strides[0])[:, None] + np.arange(kH)[None, :]
    wi = (np.arange(ow) * strides[1])[:, None] + np.arange(kW)[None, :]
    taps = np.ascontiguousarray(xp[:, hi[:, None, :, None], wi[None, :, None, :], :].reshape(J, g.K))
    Ah = np.ascontiguousarray(gz.reshape(J, co).T)
    np.testing.assert_allclose(Ah.astype(np.float64) @ taps.astype(np.float64), gw.T, rtol=0, atol=1e-12 * np.abs(gw).max())
    bound_and_check("conv nhwc filter gradient", path, "conv_nhwc_filter_grad", np.ascontiguousarray(dw.cpu().numpy().reshape(g.K, co).T),
                    Ah, taps, 1.0, splits=plan(path, co, g.K, J)[0])


@pytest.mark.parametrize("path", list(PATHS))
def test_one_by_one_reads_the_gradients_in_place(path):
    """a 1 x 1 kernel with unit strides and no padding is the plain product op(dY) * Wmat^T over dY read in place and Wmat
    through its strides: same bits, same launches (no window pass, no copy)"""
    ishape, kshape = ((3, 8, 6, 6), (16, 8, 1, 1)) if EMU else ((4, 64, 14, 14), (128, 64, 1, 1))
    g = Grad(ishape, kshape, (0, 0), (1, 1), seed=17)
    got, n_fused = g.fused(PATHS[path], "sigmoid_grad", 1.5, 1.25, layout="ohwi")
    resolved = L.last_path()
    buf, _, (ks0, ks1) = g.kernel("ohwi")
    dx = g.dx0(1.25)
    sync()
    n0 = L.launch_count()
    G.gemm_strided_fused(g.R, g.C, g.co, 1.5, g.tdy, g.co, 1, buf, ks1, ks0, 1.25, dx, g.C, 1, path=resolved,
                         op_a=("sigmoid_grad", g.taux["sigmoid_grad"], g.co, 1))
    sync()
    assert n_fused == L.launch_count() - n0
    assert_bits(got, dx.cpu().numpy().reshape(g.R, g.C))


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1", "simt"])
def test_launch_count_does_not_grow_with_the_images(path):
    ishape, kshape, padding, strides = GEOMS["pad1"]
    counts = []
    for imgs in (1, 4 if EMU else 16):
        g = Grad((imgs,) + ishape[1:], kshape, padding, strides)
        _, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.0)
        ks = plan(path, g.R, g.C, g.Kp)[0] if path != "simt" else 1
        counts.append(n - (1 if ks > 1 else 0))   # (a split adds the reduce kernel)
    # the copy of W'^T; A's window pass; B's preparation (tf32x1 and the exact path: none, W'^T is read in place); the product
    assert counts[0] == counts[1] == {"f16x3": 4, "tf32x3": 4, "tf32x1": 3, "simt": 3}[path], counts


# the profiler session and the small workspace cap run in processes of their own: the checks do not depend on what ran
# before them in the test process, and LASER_B200_BATCH_WS_MB is read once per process
_PROFILE = """
import torch, test_gpu_conv_nhwc_input_grad as T, laser_b200 as L
g = T.Grad(*T.GEOMS["stride2_tail"])
g.fused(L.PATH_F16X3, "relu_grad")
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    g.fused(L.PATH_F16X3, "relu_grad")
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print("KERNEL", e.name)
"""

_CHUNKS = """
import hashlib, sys, test_gpu_conv_nhwc_input_grad as T, laser_b200 as L
g = T.Grad((3, 4, 16, 16), (64, 4, 3, 3), (1, 1), (1, 1), seed=23)
dx, n = g.fused(int(sys.argv[1]), "tanh_grad", 0.5, 1.25)
print("RESULT", n, hashlib.sha256(dx.tobytes()).hexdigest())
"""


def _subprocess(code, *args, env=None):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), **(env or {}))
    out = subprocess.run([sys.executable, "-c", code] + list(args), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout.splitlines()


@pytest.mark.skipif(EMU, reason="torch.profiler needs the GPU")
def test_the_window_pass_is_the_rows_kernel():
    names = [line[len("KERNEL "):] for line in _subprocess(_PROFILE) if line.startswith("KERNEL ")]
    assert any("im2col_rows_kernel" in n for n in names), names
    assert any("copy_strided_kernel" in n for n in names), names
    assert not any("im2col_kernel" in n or "tap_rows_kernel" in n or "transpose" in n.lower() for n in names), names


@pytest.mark.parametrize("path", ["f16x3", "simt"])
def test_chunks_give_the_bits_of_one_chunk(path):
    """LASER_B200_BATCH_WS_MB=1 holds one image per chunk (K' = 576, H * W = 256): more launches, the same dX"""
    one = [line for line in _subprocess(_CHUNKS, str(PATHS[path])) if line.startswith("RESULT")][0].split()
    many = [line for line in _subprocess(_CHUNKS, str(PATHS[path]), env={"LASER_B200_BATCH_WS_MB": "1"})
            if line.startswith("RESULT")][0].split()
    assert int(many[1]) > int(one[1]), (one, many)
    assert many[2] == one[2]


def _raw(ishape=(2, 2, 5, 5), kshape=(3, 2, 3, 3), padding=(1, 1), strides=(1, 1), kstrides=(3, 1), op=None, path=L.PATH_AUTO,
         null=None):
    dx = dev(np.full(2 * 25 * 2, 3.0, np.float32))
    w, dy = dev(np.ones(18 * 3, np.float32)), dev(np.ones(2 * 25 * 3, np.float32))
    ptrs = {"dx": dx.data_ptr(), "w": w.data_ptr(), "dy": dy.data_ptr()}
    if null:
        ptrs[null] = None
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    fn = _capi.lib().laser_b200_conv2d_nhwc_input_grad_f32_fused_dev
    if kstrides is None:   # a NULL kernelStrides: the same symbol through a handle whose argtypes take a plain pointer there
        fn = ctypes.CDLL(_capi.lib()._name).laser_b200_conv2d_nhwc_input_grad_f32_fused_dev
        fn.argtypes = [ctypes.c_void_p, i4, ctypes.c_void_p, ctypes.c_void_p, i4, ctypes.c_void_p, i2, i2, ctypes.c_float,
                       ctypes.c_float, ctypes.POINTER(_capi.OperandOp), ctypes.c_int, ctypes.c_void_p]
    rc = fn(ptrs["dx"], i4(*ishape), ptrs["dy"], ptrs["w"], i4(*kshape), i2(*kstrides) if kstrides else None, i2(*padding),
            i2(*strides), 1.0, 0.0, op, path, G._current_stream())
    sync()
    assert np.all(dx.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    aux = dev(np.ones(2 * 25 * 3, np.float32))
    relu_grad = lambda rs, cs: ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD, aux=aux.data_ptr(), auxRowStride=rs,
                                                            auxColStride=cs))
    for kw in (dict(path=5), dict(path=-1), dict(op=ctypes.byref(_capi.OperandOp(op=9))),
               dict(op=ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))), dict(op=relu_grad(1, 3)), dict(op=relu_grad(4, 1)),
               dict(op=relu_grad(25, 1)), dict(kstrides=None), dict(kshape=(3, 1, 3, 3)), dict(strides=(0, 1)),
               dict(padding=(-1, 0)), dict(kshape=(3, 2, 8, 3)), dict(null="dx"), dict(null="w"), dict(null="dy")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    assert _raw(ishape=(0, 2, 5, 5)) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 2, 5, 5), null="dx") == (_capi.E_OK, 0)
    # K' = c_out * kH * kW = 2^29 * 9 past int32 (nothing is read: the check comes first)
    assert _raw(kshape=(2 ** 29, 2, 3, 3)) == (_capi.E_UNSUPPORTED, 0)
    # n * H * W = 2^30 * 16 past int32 on a tensor-core path
    assert _raw(ishape=(2 ** 30, 2, 4, 4), padding=(0, 0), path=L.PATH_F16X3) == (_capi.E_UNSUPPORTED, 0)


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode of this file's bound checks (the last test of the file)"""
    from test_gpu_error_bounds import RATIOS
    mine = {k: r for k, r in RATIOS.items() if k[1] == "conv_nhwc_input_grad"}
    if not mine:
        pytest.skip("no case ran")
    with capsys.disabled():
        print("\nlargest err / bound of the NHWC input gradient:\n" +
              "\n".join("  %-7s %.3g" % (m, r) for (m, _), r in sorted(mine.items())))
