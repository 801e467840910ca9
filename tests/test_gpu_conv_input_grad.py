"""GPU: the fused convolution's input gradient laser_b200_conv2d_input_grad_f32_fused_dev -- dX_n <- alpha * W' * B_n + beta *
dX_n, the forward call's product over the rotated filters W' and B_n the input pixels' windows over op(dY_n) zero-dilated by
the strides.  On every path dX must equal, bit for bit, the batched fused product over W' and the transposed windows
materialised in numpy (holes 0), and at stride 1 with pH <= kH - 1 the forward entry over (dY, W', kH - 1 - pH); the exact
path equals the CPU oracle; the tensor-core paths meet the per-element bound of tests/test_gpu_error_bounds.py against
torch.nn.grad.conv2d_input in float64; the launch count does not grow with the images, and chunks give the bits of one."""
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
# forward geometries (ishape, kshape, padding, strides)
GEOMS = {
    "pad1": ((3, 8, 10, 10), (16, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 48, 20, 20), (64, 48, 3, 3), (1, 1), (1, 1)),
    # (8 - 3) mod 2 = 1: the last input row and column lie in no window
    "stride2_tail": ((2, 4, 8, 8), (8, 4, 3, 3), (0, 0), (2, 2)) if EMU else ((5, 24, 8, 8), (40, 24, 3, 3), (0, 0), (2, 2)),
    "non_square_3x5": ((2, 3, 8, 9), (8, 3, 3, 5), (1, 2), (1, 1)) if EMU else ((3, 16, 16, 19), (32, 16, 3, 5), (1, 2), (1, 1)),
    "one_by_one_stride2": ((3, 6, 7, 7), (8, 6, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 32, 15, 15), (64, 32, 1, 1), (0, 0), (2, 2)),
    # p' = kH - 1 - pH = -1
    "one_by_one_pad1": ((2, 6, 5, 6), (8, 6, 1, 1), (1, 1), (1, 1)) if EMU else ((3, 32, 14, 13), (64, 32, 1, 1), (1, 1), (1, 1)),
    "single_image": ((1, 4, 8, 8), (8, 4, 3, 3), (1, 1), (1, 1)) if EMU else ((1, 16, 24, 24), (32, 16, 3, 3), (1, 1), (1, 1)),
    # n * H * W = 147 / 405: not a multiple of 4
    "odd_pixels": ((3, 2, 7, 7), (8, 2, 3, 3), (0, 0), (1, 1)) if EMU else ((5, 16, 9, 9), (32, 16, 3, 3), (0, 0), (1, 1)),
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dX (never read), beta != 0 over a seeded one
VARIANTS = {"plain": (None, 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 1.0, 1.25), "sigmoid": ("sigmoid", 0.75, 0.0), "relu": ("relu", 1.0, 1.25)}


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def up(x, m):
    return -(-x // m) * m


def transposed_windows(z, ishape, kshape, padding, strides):
    """[n][H * W][K'] rows: input pixel (ih, iw)'s window over z [n][c_out][outH][outW] zero-dilated by the strides and padded by
    kH - 1 - pH, in the order (co, kh', kw'); 0 wherever a tap falls between, before or past z's rows and columns"""
    n, _, H, W = ishape
    co, _, kH, kW = kshape
    oh, ow = z.shape[2:]

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, padding[0], strides[0], oh)
    wq, vw = axis(W, kW, padding[1], strides[1], ow)
    g = z[:, :, hq[:, :, None, None], wq[None, None, :, :]]
    g = np.where((vh[:, :, None, None] & vw[None, None, :, :])[None, None], g, np.zeros((), z.dtype))
    return np.ascontiguousarray(g.transpose(0, 2, 4, 1, 3, 5).reshape(n, H * W, co * kH * kW))


def lib_op(name, x):
    """op(x) elementwise with the library's own op: the exact path's product of op(x) with the identity"""
    flat = np.ascontiguousarray(x.reshape(-1, x.shape[-1]), np.float32)
    R, Cc = flat.shape
    out = dev(np.zeros_like(flat))
    G.gemm_strided_fused(R, Cc, Cc, 1.0, dev(flat), Cc, 1, dev(np.eye(Cc, dtype=np.float32)), Cc, 1, 0.0, out, Cc, 1,
                         path=L.PATH_SIMT, op_a=name)
    sync()
    return out.cpu().numpy().reshape(x.shape).copy()


class Grad:
    """one input gradient's data: filters W, output gradients dY, the forward output Z an op's aux is taken from, and dX0"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, w=None, dy=None):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        n, C, H, W = ishape
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        self.HW, self.Kp = H * W, kshape[0] * kshape[2] * kshape[3]
        self.w = O.fill_uniform_f32(int(np.prod(kshape)), seed, -1, 1).reshape(kshape) if w is None else w
        self.dy = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 1, -1, 1).reshape(self.oshape) if dy is None else dy
        z = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 2, -2, 2).reshape(self.oshape)
        self.aux = {"relu_grad": np.maximum(z, 0), "tanh_grad": np.tanh(z), "sigmoid_grad": 1 / (1 + np.exp(-z))}
        self.x0 = O.fill_uniform_f32(int(np.prod(ishape)), seed + 3, -1, 1)
        self.tw, self.tdy = dev(self.w), dev(self.dy)
        self.taux = {k: dev(v.astype(np.float32)) for k, v in self.aux.items()}

    def wrot(self):
        """W'[ci][co][kh'][kw'] = W[co][ci][kH-1-kh'][kW-1-kw']"""
        return np.ascontiguousarray(self.w[:, :, ::-1, ::-1].transpose(1, 0, 2, 3))

    def dx0(self, beta):
        return dev(self.x0 if beta != 0.0 else np.full(self.x0.shape, np.nan, np.float32))

    def fused(self, path, op=None, alpha=1.0, beta=0.0):
        """-> (dX, launches)"""
        dx = self.dx0(beta)
        sync()
        n0 = L.launch_count()
        L.conv2d_input_grad_fused(dx, self.ishape, self.tdy, self.tw, self.kshape, self.padding, self.strides, alpha, beta, op=op,
                                  aux=self.taux.get(op), path=path)
        sync()
        return dx.cpu().numpy().copy(), L.launch_count() - n0

    def rows(self, z):
        return transposed_windows(z, self.ishape, self.kshape, self.padding, self.strides)

    def batched(self, path, op=None, alpha=1.0, beta=0.0):
        """the batched fused product over A = W' (shared) and B_n = the materialised transposed windows read transposed, op_b
        applied by the library on both sides (sigmoid, not 0 at 0: op(dY) materialised with the library's own op)"""
        n, C = self.ishape[:2]
        K, ld = self.Kp, up(self.Kp, 4)
        a = np.zeros((C, ld), np.float32)
        a[:, :K] = self.wrot().reshape(C, K)
        b = np.zeros((n, self.HW, ld), np.float32)
        op_b = op
        if op == "sigmoid":
            b[:, :, :K] = self.rows(lib_op("sigmoid", self.dy))
            op_b = None
        else:
            b[:, :, :K] = self.rows(self.dy)
        if op in self.aux:
            y = np.zeros((n, self.HW, ld), np.float32)
            y[:, :, :K] = self.rows(self.aux[op].astype(np.float32))
            op_b = (op, dev(y), 1, ld, self.HW * ld)
        dx = self.dx0(beta)
        G.gemm_strided_batched_fused(n, C, self.HW, K, alpha, dev(a), ld, 1, 0, dev(b), 1, ld, self.HW * ld, beta, dx, self.HW, 1,
                                     C * self.HW, path=path, op_b=op_b)
        sync()
        return dx.cpu().numpy().copy()


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_batched_product_over_the_windows(path, geom):
    """each geometry with one variant (they take turns), so that every variant meets several geometries; PATH_AUTO: the batched
    product on the path the entry resolved"""
    op, alpha, beta = list(VARIANTS.values())[list(GEOMS).index(geom) % len(VARIANTS)]
    g = Grad(*GEOMS[geom])
    got, _ = g.fused(PATHS[path], op, alpha, beta)
    resolved = L.last_path()
    if path != "auto":
        assert resolved == PATHS[path]
    assert_bits(got, g.batched(resolved, op, alpha, beta))
    if beta == 0.0:
        assert not np.isnan(got).any()


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("path", ["simt", "f16x3", "tf32x3", "tf32x1"])
def test_ops_and_scalars_bit_identical(path, variant):
    """every op (derivatives with the forward output as aux), alpha != 1, beta = 1.25 over a seeded dX and beta = 0 over a
    NaN-filled one -- at stride 2, where the last row and column get beta * dX0 (or 0) only"""
    g = Grad(*GEOMS["stride2_tail"], seed=5)
    got, _ = g.fused(PATHS[path], *VARIANTS[variant])
    assert_bits(got, g.batched(PATHS[path], *VARIANTS[variant]))
    n, C, H, W = g.ishape
    op, alpha, beta = VARIANTS[variant]
    tail = got.reshape(n, C, H, W)[:, :, H - 1, :]
    np.testing.assert_array_equal(tail, np.float32(beta) * g.x0.reshape(n, C, H, W)[:, :, H - 1, :] if beta else 0.0)


@pytest.mark.parametrize("geom", ["pad1", "non_square_3x5", "single_image", "odd_pixels"])
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_forward_entry(path, geom):
    """stride 1, pH <= kH - 1: the forward call over (dY, W', kH - 1 - pH) is the same product"""
    g = Grad(*GEOMS[geom], seed=7)
    got, _ = g.fused(PATHS[path])
    kH, kW = g.kshape[2:]
    out = dev(np.full(int(np.prod(g.ishape)), np.nan, np.float32))
    L.conv2d_fused(out, g.tdy, g.oshape, dev(g.wrot()), (g.ishape[1], g.kshape[0], kH, kW),
                   (kH - 1 - g.padding[0], kW - 1 - g.padding[1]), (1, 1), path=PATHS[path])
    sync()
    assert_bits(got, out.cpu().numpy())


def test_exact_path_matches_the_oracle():
    g = Grad(*GEOMS["stride2_tail"], seed=9)
    got, _ = g.fused(L.PATH_SIMT, "relu_grad", 0.5, 0.75)
    z = np.where(g.aux["relu_grad"] > 0, g.dy, np.float32(0)).astype(np.float32)
    rows = g.rows(z)
    n, C = g.ishape[:2]
    a = np.ascontiguousarray(g.wrot().reshape(C, g.Kp))
    want = g.x0.reshape(n, C, g.HW).copy()
    for b in range(n):
        wb = np.ascontiguousarray(want[b])
        O.gemm_strided(C, g.HW, g.Kp, 0.5, a, g.Kp, 1, np.ascontiguousarray(rows[b]), 1, g.Kp, 0.75, wb, g.HW, 1)
        want[b] = wb
    assert_bits(got, want.reshape(-1))


def scaled_case(ishape, kshape, padding, strides, seed):
    """signed data: every image and channel of dY and every input channel of W at its own power-of-two scale"""
    rng = np.random.default_rng(seed)
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
    dy = rng.uniform(-1, 1, oshape) * 2.0 ** rng.integers(-6, 7, oshape[0])[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, oshape[1])[None, :, None, None]
    w = rng.uniform(-1, 1, kshape) * 2.0 ** rng.integers(-6, 7, kshape[1])[None, :, None, None]
    return Grad(ishape, kshape, padding, strides, w=w.astype(np.float32), dy=dy.astype(np.float32))


@pytest.mark.parametrize("geom", ["pad1", "stride2_tail"])
@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound_against_torch(path, geom):
    torch = pytest.importorskip("torch")
    g = scaled_case(*GEOMS[geom], seed=11)
    got, _ = g.fused(PATHS[path])
    n, C = g.ishape[:2]
    A = g.wrot().reshape(C, g.Kp)
    B = g.rows(g.dy).transpose(0, 2, 1)
    ref = torch.nn.grad.conv2d_input(g.ishape, torch.from_numpy(g.w.astype(np.float64)), torch.from_numpy(g.dy.astype(np.float64)),
                                     stride=g.strides, padding=g.padding).numpy().reshape(n, C, g.HW)
    np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    ks, _ = plan(path, C, g.HW, g.Kp, batch=n)
    bound_and_check("conv input gradient", path, "conv_input_grad", got.reshape(n, C, g.HW), np.broadcast_to(A, (n, C, g.Kp)), B,
                    1.0, splits=ks)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_layer_backward_pass_against_torch_autograd(path):
    """conv2d_fused with bias and relu, then the input and filter gradients with relu_grad and the forward output as aux:
    against torch autograd of the convolution in float64 with the same relu mask, each within the bound"""
    torch = pytest.importorskip("torch")
    ishape, kshape, padding, strides = GEOMS["stride2_tail"]
    n, C, H, W = ishape
    co = kshape[0]
    rng = np.random.default_rng(21)
    x = rng.uniform(-1, 1, ishape).astype(np.float32)
    w = rng.uniform(-1, 1, kshape).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, co).astype(np.float32)
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
    dy = rng.uniform(-1, 1, oshape).astype(np.float32)
    tz = dev(np.zeros(int(np.prod(oshape)), np.float32))
    L.conv2d_fused(tz, dev(x), ishape, dev(w), kshape, padding, strides, bias=dev(bias), activation="relu", path=PATHS[path])
    sync()
    z = tz.cpu().numpy().reshape(oshape).copy()
    g = Grad(ishape, kshape, padding, strides, w=w, dy=dy)
    dx = dev(np.full(int(np.prod(ishape)), np.nan, np.float32))
    dw = dev(np.full(int(np.prod(kshape)), np.nan, np.float32))
    L.conv2d_input_grad_fused(dx, ishape, g.tdy, g.tw, kshape, padding, strides, op="relu_grad", aux=tz, path=PATHS[path])
    L.conv2d_filter_grad_fused(dw, dev(x), ishape, g.tdy, kshape, padding, strides, op="relu_grad", aux=tz, path=PATHS[path])
    sync()
    gz = np.where(z > 0, dy, np.float32(0)).astype(np.float32)
    tx = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    tw = torch.from_numpy(w.astype(np.float64)).requires_grad_()
    y = torch.nn.functional.conv2d(tx, tw, torch.from_numpy(bias.astype(np.float64)), stride=strides, padding=padding)
    y.backward(torch.from_numpy(gz.astype(np.float64)))
    A = g.wrot().reshape(C, g.Kp)
    B = g.rows(gz).transpose(0, 2, 1)
    np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), tx.grad.numpy().reshape(n, C, H * W), rtol=0,
                               atol=1e-12 * np.abs(tx.grad.numpy()).max())
    bound_and_check("conv input gradient", path, "conv_input_grad", dx.cpu().numpy().reshape(n, C, H * W),
                    np.broadcast_to(A, (n, C, g.Kp)), B, 1.0, splits=plan(path, C, H * W, g.Kp, batch=n)[0])
    P, Kc = oshape[2] * oshape[3], C * kshape[2] * kshape[3]
    Ah = np.ascontiguousarray(np.concatenate(list(gz.reshape(n, co, P)), axis=1))
    Bh = np.ascontiguousarray(np.concatenate([O.im2col(np.ascontiguousarray(x[b]), ishape, kshape, padding, strides).T
                                              for b in range(n)], axis=0))
    np.testing.assert_allclose(Ah.astype(np.float64) @ Bh.astype(np.float64), tw.grad.numpy().reshape(co, Kc), rtol=0,
                               atol=1e-12 * np.abs(tw.grad.numpy()).max())
    bound_and_check("conv filter gradient", path, "conv_filter_grad", dw.cpu().numpy().reshape(co, Kc), Ah, Bh, 1.0,
                    splits=plan(path, co, Kc, n * P)[0])


@pytest.mark.parametrize("path", list(PATHS))
def test_one_by_one_reads_the_gradients_in_place(path):
    """a 1 x 1 kernel with unit strides and no padding is the batched product W^T * dY_n over dY itself: same bits, same
    launches"""
    ishape, kshape = ((3, 8, 6, 6), (16, 8, 1, 1)) if EMU else ((4, 64, 14, 14), (128, 64, 1, 1))
    g = Grad(ishape, kshape, (0, 0), (1, 1), seed=17)
    got, n_fused = g.fused(PATHS[path], "sigmoid_grad", 1.5, 1.25)
    n, C, co, P = ishape[0], ishape[1], kshape[0], g.HW
    dx = g.dx0(1.25)
    sync()
    n0 = L.launch_count()
    G.gemm_strided_batched_fused(n, C, P, co, 1.5, g.tw, 1, C, 0, g.tdy, P, 1, co * P, 1.25, dx, P, 1, C * P, path=PATHS[path],
                                 op_b=("sigmoid_grad", g.taux["sigmoid_grad"], P, 1, co * P))
    sync()
    assert n_fused == L.launch_count() - n0
    assert_bits(got, dx.cpu().numpy())


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1", "simt"])
def test_launch_count_does_not_grow_with_the_images(path):
    ishape, kshape, padding, strides = GEOMS["pad1"]
    counts = []
    for imgs in (1, 4 if EMU else 16):
        g = Grad((imgs,) + ishape[1:], kshape, padding, strides)
        _, n = g.fused(PATHS[path], "relu_grad", 1.0, 0.0)
        ks = plan(path, kshape[1], g.HW, g.Kp, batch=imgs)[0] if path != "simt" else 1
        counts.append(n - (1 if ks > 1 else 0))   # (a split adds the reduce kernel)
    # the filter rotation; A's preparation (tf32x1 and the exact path: none); B's window pass; the product
    assert counts[0] == counts[1] == {"f16x3": 4, "tf32x3": 4, "tf32x1": 3, "simt": 3}[path], counts


# the profiler session and the small workspace cap run in processes of their own: the checks do not depend on what ran
# before them in the test process, and LASER_B200_BATCH_WS_MB is read once per process
_PROFILE = """
import torch, test_gpu_conv_input_grad as T, laser_b200 as L
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
import hashlib, sys, test_gpu_conv_input_grad as T, laser_b200 as L
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
    assert not any("im2col_kernel" in n or "im2col_tap_rows_kernel" in n for n in names), names


@pytest.mark.parametrize("path", ["f16x3", "simt"])
def test_chunks_give_the_bits_of_one_chunk(path):
    """LASER_B200_BATCH_WS_MB=1 holds one image per chunk (K' = 576, H * W = 256): more launches, the same dX"""
    one = [line for line in _subprocess(_CHUNKS, str(PATHS[path])) if line.startswith("RESULT")][0].split()
    many = [line for line in _subprocess(_CHUNKS, str(PATHS[path]), env={"LASER_B200_BATCH_WS_MB": "1"})
            if line.startswith("RESULT")][0].split()
    assert int(many[1]) > int(one[1]), (one, many)
    assert many[2] == one[2]


def _raw(ishape=(2, 2, 5, 5), kshape=(3, 2, 3, 3), padding=(1, 1), strides=(1, 1), op=None, path=L.PATH_AUTO, null=None):
    dx = dev(np.full(2 * 2 * 25, 3.0, np.float32))
    w, dy = dev(np.ones(3 * 2 * 9, np.float32)), dev(np.ones(2 * 3 * 25, np.float32))
    ptrs = {"dx": dx.data_ptr(), "w": w.data_ptr(), "dy": dy.data_ptr()}
    if null:
        ptrs[null] = None
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_conv2d_input_grad_f32_fused_dev(ptrs["dx"], i4(*ishape), ptrs["dy"], ptrs["w"], i4(*kshape),
                                                                i2(*padding), i2(*strides), 1.0, 0.0, op, path,
                                                                G._current_stream())
    sync()
    assert np.all(dx.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    aux = dev(np.ones(2 * 3 * 25, np.float32))
    relu_grad = lambda rs, cs: ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD, aux=aux.data_ptr(), auxRowStride=rs,
                                                            auxColStride=cs))
    for kw in (dict(path=5), dict(path=-1), dict(op=ctypes.byref(_capi.OperandOp(op=9))),
               dict(op=ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))), dict(op=relu_grad(26, 1)), dict(op=relu_grad(25, 2)),
               dict(op=relu_grad(1, 25)), dict(kshape=(3, 1, 3, 3)), dict(strides=(0, 1)), dict(padding=(-1, 0)),
               dict(kshape=(3, 2, 8, 3)), dict(null="dx"), dict(null="w"), dict(null="dy")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    assert _raw(ishape=(0, 2, 5, 5)) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 2, 5, 5), null="dx") == (_capi.E_OK, 0)
    # K' = c_out * kH * kW = 2^29 * 9 past int32 (nothing is read: the check comes first)
    assert _raw(kshape=(2 ** 29, 2, 3, 3)) == (_capi.E_UNSUPPORTED, 0)


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode of this file's bound checks (the last test of the file)"""
    from test_gpu_error_bounds import RATIOS
    mine = {k: r for k, r in RATIOS.items() if k[1] == "conv_input_grad"}
    if not mine:
        pytest.skip("no case ran")
    with capsys.disabled():
        print("\nlargest err / bound of the input gradient:\n" + "\n".join("  %-7s %.3g" % (m, r) for (m, _), r in sorted(mine.items())))
