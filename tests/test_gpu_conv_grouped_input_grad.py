"""GPU: the grouped convolution's input gradient laser_b200_conv2d_grouped_input_grad_f32_fused_dev
(torch.nn.grad.conv2d_input(groups=G)).  The exact path is the direct CUDA-core kernel over the transposed geometry: one launch,
no filter copy, and dX bit for bit G conv2d_input_grad_fused calls on PATH_SIMT over contiguous per-group copies (the oracle's
gemm_strided(W'_g, rows_{n,g}, alpha, beta) per image and group).  The tensor-core paths are one filter copy and one batched
GEMM per chunk whose rotated filters repeat every G problems: the bits of the per-group calls while K' <= 896 (no split along K
on either side), the per-element float64 bound, and a launch count that does not grow with n or G.  groups == 1 is
conv2d_input_grad_fused itself."""
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

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
TC = ["f16x3", "tf32x3", "tf32x1"]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# forward geometries (ishape, kshape = (c_out, c_in / G, kH, kW), padding, strides, groups)
NARROW = {
    "depthwise": ((2, 8, 9, 9), (8, 1, 3, 3), (1, 1), (1, 1), 8),
    "multiplier2": ((2, 4, 7, 7), (8, 1, 3, 3), (1, 1), (1, 1), 4),
    "depthwise_stride2": ((2, 6, 12, 10), (6, 1, 3, 3), (1, 1), (2, 2), 6),
    "stride21_non_square": ((2, 6, 12, 9), (6, 1, 3, 2), (1, 0), (2, 1), 6),
    "depthwise_7x7_pad3": ((2, 4, 10, 10), (4, 1, 7, 7), (3, 3), (1, 1), 4),
    "cg4": ((2, 16, 8, 8), (16, 4, 3, 3), (1, 1), (1, 1), 4),
    "mg64_kc_flush": ((1, 8, 5, 5), (128, 4, 3, 3), (1, 1), (1, 1), 2),       # K' = 576 > 512
    "grouped_1x1": ((2, 8, 6, 6), (12, 2, 1, 1), (0, 0), (1, 1), 4),
    "grouped_1x1_stride2": ((2, 8, 7, 7), (8, 2, 1, 1), (0, 0), (2, 2), 4),
    "tail_rows": ((2, 4, 8, 8), (4, 1, 3, 3), (0, 0), (2, 2), 4),             # row and column 7 in no window
    "odd_in_w": ((2, 6, 6, 13), (6, 2, 3, 3), (1, 1), (1, 2), 3),
    "wide_in_w": ((1, 2, 4, 150), (2, 1, 3, 3), (1, 1), (1, 1), 2),           # two column tiles
}
# groups wide enough for the tensor cores on PATH_AUTO (Cg >= 64, K' >= 64), K' <= 896
WIDE = {
    "g2": ((2, 128, 8, 8), (16, 64, 3, 3), (1, 1), (1, 1), 2),
    "g4_stride2": ((2, 256, 9, 9), (32, 64, 3, 3), (1, 1), (2, 2), 4),
} if EMU else {
    "g4": ((4, 256, 14, 14), (64, 64, 3, 3), (1, 1), (1, 1), 4),                # K' = 144
    "g8_stride2": ((3, 512, 15, 15), (128, 64, 3, 3), (1, 1), (2, 2), 8),       # K' = 144
    "g2_k864": ((2, 128, 12, 12), (192, 64, 3, 3), (1, 1), (1, 1), 2),          # K' = 864: the largest without a split
    "g2_1x1": ((2, 128, 14, 14), (128, 64, 1, 1), (0, 0), (1, 1), 2),
}
# (op, alpha, beta): beta = 0 runs over a NaN-filled dX (never read), beta != 0 over a seeded one
VARIANTS = {"plain": (None, 1.0, 0.0), "relu_grad": ("relu_grad", -0.5, 1.25), "tanh_grad": ("tanh_grad", 2.0, 0.0),
            "sigmoid_grad": ("sigmoid_grad", 2.0, 0.0), "sigmoid": ("sigmoid", 0.75, 1.0)}


def assert_bits(got, want):
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def launches(fn):
    sync()
    n0 = L.launch_count()
    fn()
    sync()
    return L.launch_count() - n0


def windows(z, ishape, kshape, padding, strides):
    """[n][H * W][K'] rows: input pixel (ih, iw)'s window over z [n][c][outH][outW] zero-dilated by the strides and padded by
    kH - 1 - pH, in the order (c, kh', kw'); 0 wherever a tap falls between, before or past z's rows and columns"""
    n, _, H, W = ishape
    _, _, kH, kW = kshape
    oh, ow = z.shape[2:]

    def axis(size, k, pad, s, out):
        d = np.arange(size)[:, None] - (k - 1 - pad) + np.arange(k)[None, :]
        ok = (d >= 0) & (d % s == 0) & (d // s < out)
        return np.where(ok, d // s, 0), ok
    hq, vh = axis(H, kH, padding[0], strides[0], oh)
    wq, vw = axis(W, kW, padding[1], strides[1], ow)
    g = z[:, :, hq[:, :, None, None], wq[None, None, :, :]]
    g = np.where((vh[:, :, None, None] & vw[None, None, :, :])[None, None], g, np.zeros((), z.dtype))
    return np.ascontiguousarray(g.transpose(0, 2, 4, 1, 3, 5).reshape(n, H * W, z.shape[1] * kH * kW))


class GGrad:
    """one grouped input gradient's data: filters W [c_out][Cg][kH][kW], dY, the forward output Z the aux is taken from, dX0"""

    def __init__(self, ishape, kshape, padding, strides, groups, seed=1, w=None, dy=None):
        self.ishape, self.kshape, self.padding, self.strides, self.groups = ishape, kshape, padding, strides, groups
        n, C, H, W = ishape
        self.Cg, self.Mg = C // groups, kshape[0] // groups
        o = O.conv2d_out_shape((n, self.Cg, H, W), (self.Mg,) + tuple(kshape[1:]), padding, strides)
        self.oshape = (n, kshape[0], o[2], o[3])
        self.HW, self.T = H * W, kshape[2] * kshape[3]
        self.Kp = self.Mg * self.T
        self.w = O.fill_uniform_f32(int(np.prod(kshape)), seed, -1, 1).reshape(kshape) if w is None else w
        self.dy = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 1, -1, 1).reshape(self.oshape) if dy is None else dy
        z = O.fill_uniform_f32(int(np.prod(self.oshape)), seed + 2, -2, 2).reshape(self.oshape)
        self.aux = {"relu_grad": np.maximum(z, 0), "tanh_grad": np.tanh(z), "sigmoid_grad": 1 / (1 + np.exp(-z))}
        self.aux = {k: v.astype(np.float32) for k, v in self.aux.items()}
        self.x0 = O.fill_uniform_f32(int(np.prod(ishape)), seed + 3, -1, 1).reshape(ishape)
        self.tw, self.tdy = dev(self.w), dev(self.dy)
        self.taux = {k: dev(v) for k, v in self.aux.items()}

    def dx0(self, beta, x0=None):
        x0 = self.x0 if x0 is None else x0
        return dev(x0 if beta != 0.0 else np.full(x0.shape, np.nan, np.float32))

    def grouped(self, path, op=None, alpha=1.0, beta=0.0, groups=None):
        """-> (dX, launches)"""
        dx = self.dx0(beta)
        sync()
        n0 = L.launch_count()
        L.conv2d_grouped_input_grad_fused(dx, self.ishape, self.tdy, self.tw, self.kshape, self.padding, self.strides,
                                          self.groups if groups is None else groups, alpha, beta, op=op, aux=self.taux.get(op),
                                          path=path)
        sync()
        return dx.cpu().numpy().copy(), L.launch_count() - n0

    def per_group_calls(self, path, op=None, alpha=1.0, beta=0.0):
        """G conv2d_input_grad_fused calls on contiguous per-group copies"""
        n, C, H, W = self.ishape
        out = np.empty(self.ishape, np.float32)
        for g in range(self.groups):
            cs, ms = slice(g * self.Cg, (g + 1) * self.Cg), slice(g * self.Mg, (g + 1) * self.Mg)
            dx = self.dx0(beta, np.ascontiguousarray(self.x0[:, cs]))
            aux = dev(np.ascontiguousarray(self.aux[op][:, ms])) if op in self.aux else None
            L.conv2d_input_grad_fused(dx, (n, self.Cg, H, W), dev(np.ascontiguousarray(self.dy[:, ms])),
                                      dev(np.ascontiguousarray(self.w[ms])), (self.Mg,) + tuple(self.kshape[1:]), self.padding,
                                      self.strides, alpha, beta, op=op, aux=aux, path=path)
            sync()
            out[:, cs] = dx.cpu().numpy().reshape(n, self.Cg, H, W)
        return out

    def wrot(self, g):
        """W'_g [Cg][K'] = kernel[g * Mg + co][ci][T - 1 - t] at (ci, co * T + t)"""
        ms = slice(g * self.Mg, (g + 1) * self.Mg)
        return np.ascontiguousarray(self.w[ms, :, ::-1, ::-1].transpose(1, 0, 2, 3).reshape(self.Cg, self.Kp))

    def operands(self, z):
        """A [n][G][Cg][K'] and B [n][G][K'][H * W] as multiplied, B the windows over z (op(dY))"""
        n = self.ishape[0]
        A = np.broadcast_to(np.stack([self.wrot(g) for g in range(self.groups)]), (n, self.groups, self.Cg, self.Kp))
        B = np.stack([windows(np.ascontiguousarray(z[:, g * self.Mg:(g + 1) * self.Mg]), self.ishape, self.kshape, self.padding,
                              self.strides) for g in range(self.groups)], axis=1)
        return A, np.ascontiguousarray(B.transpose(0, 1, 3, 2))


# ---- exact path: the direct kernel over the transposed geometry ------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("geom", list(NARROW))
def test_exact_path_equals_per_group_calls(geom, variant):
    c = GGrad(*NARROW[geom])
    got, n = c.grouped(L.PATH_SIMT, *VARIANTS[variant])
    assert n == 1 and L.last_path() == L.PATH_SIMT     # one launch: no filter copy, no window pass
    assert_bits(got, c.per_group_calls(L.PATH_SIMT, *VARIANTS[variant]))
    if VARIANTS[variant][2] == 0.0:
        assert not np.isnan(got).any()


@pytest.mark.parametrize("geom", ["depthwise_stride2", "cg4", "mg64_kc_flush", "tail_rows"])
def test_exact_path_matches_the_oracle(geom):
    """gemm_strided(W'_g, rows_{n,g}, alpha, beta) of the oracle per image and group, rows over relu_grad(dY) built in numpy"""
    c = GGrad(*NARROW[geom], seed=9)
    got, _ = c.grouped(L.PATH_SIMT, "relu_grad", 0.5, 0.75)
    z = np.where(c.aux["relu_grad"] > 0, c.dy, np.float32(0)).astype(np.float32)
    A, B = c.operands(z)
    n, C, H, W = c.ishape
    want = c.x0.reshape(n, C, c.HW).copy()
    for i in range(n):
        for g in range(c.groups):
            wb = np.ascontiguousarray(want[i, g * c.Cg:(g + 1) * c.Cg])
            O.gemm_strided(c.Cg, c.HW, c.Kp, 0.5, np.ascontiguousarray(A[i, g]), c.Kp, 1, np.ascontiguousarray(B[i, g]), c.HW, 1, 0.75,
                           wb, c.HW, 1)
            want[i, g * c.Cg:(g + 1) * c.Cg] = wb
    assert_bits(got, want.reshape(c.ishape))


def test_rows_no_window_covers_get_beta_dx_only():
    c = GGrad(*NARROW["tail_rows"], seed=5)
    got, _ = c.grouped(L.PATH_SIMT, "relu_grad", -0.5, 1.25)
    np.testing.assert_array_equal(got[:, :, -1, :], np.float32(1.25) * c.x0[:, :, -1, :])


def test_inf_filter_tap_in_the_padding_gives_nan_where_the_oracle_does():
    c = GGrad(*NARROW["cg4"])
    c.w[5, 2, 0, 0] = np.inf          # output channel 5 (group 1), top-left tap: W'_1's last tap, past the bottom / right edge
    c.tw = dev(c.w)
    got, _ = c.grouped(L.PATH_SIMT)
    want = c.per_group_calls(L.PATH_SIMT)
    nan = np.isnan(want)
    assert nan.any() and not nan.all()
    assert np.array_equal(np.isnan(got), nan)
    assert_bits(got[~nan], want[~nan])


# ---- tensor-core paths: one filter copy, one batched GEMM per chunk with the filters repeating every G problems -----------
@pytest.mark.parametrize("variant", ["plain", "relu_grad", "sigmoid"])
@pytest.mark.parametrize("geom", list(WIDE) + ["cg4", "multiplier2", "grouped_1x1", "depthwise_stride2"])
@pytest.mark.parametrize("path", TC)
def test_tensor_core_paths_equal_per_group_calls(path, geom, variant):
    c = GGrad(*(WIDE[geom] if geom in WIDE else NARROW[geom]))
    assert c.Kp <= 896
    got, _ = c.grouped(PATHS[path], *VARIANTS[variant])
    assert L.last_path() == PATHS[path]
    assert_bits(got, c.per_group_calls(PATHS[path], *VARIANTS[variant]))


def scaled_case(ishape, kshape, padding, strides, groups, seed):
    """signed data: every image and channel of dY and every input channel of W at its own power-of-two scale"""
    rng = np.random.default_rng(seed)
    probe = GGrad(ishape, kshape, padding, strides, groups)
    oshape = probe.oshape
    dy = rng.uniform(-1, 1, oshape) * 2.0 ** rng.integers(-6, 7, oshape[0])[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, oshape[1])[None, :, None, None]
    w = rng.uniform(-1, 1, kshape) * 2.0 ** rng.integers(-6, 7, kshape[1])[None, :, None, None]
    return GGrad(ishape, kshape, padding, strides, groups, w=w.astype(np.float32), dy=dy.astype(np.float32))


@pytest.mark.parametrize("geom", list(WIDE)[:2])
@pytest.mark.parametrize("path", TC)
def test_tensor_core_paths_within_the_bound(path, geom):
    c = scaled_case(*WIDE[geom], seed=11)
    got, _ = c.grouped(PATHS[path])
    n = c.ishape[0]
    A, B = c.operands(c.dy)
    ks, _ = plan(path, c.Cg, c.HW, c.Kp, batch=n * c.groups)
    bound_and_check("grouped input gradient", path, "conv_grouped_input_grad", got.reshape(n, c.groups, c.Cg, c.HW), A, B, 1.0,
                    splits=ks)


@pytest.mark.parametrize("path", TC)
def test_split_k_layer_within_the_bound(path):
    """K' = 64 * 25 = 1600 on few tiles: the 3-pass paths split along K, the grouped call within the bound"""
    ishape, kshape = ((1, 4, 6, 6), (128, 2, 5, 5)) if EMU else ((1, 8, 14, 14), (128, 4, 5, 5))
    c = scaled_case(ishape, kshape, (2, 2), (1, 1), 2, seed=13)
    got, _ = c.grouped(PATHS[path], None, 1.0, 0.0)
    n = c.ishape[0]
    A, B = c.operands(c.dy)
    ks, _ = plan(path, c.Cg, c.HW, c.Kp, batch=n * c.groups)
    assert (ks > 1) == (path != "tf32x1")
    bound_and_check("grouped input gradient", path, "conv_grouped_input_grad", got.reshape(n, c.groups, c.Cg, c.HW), A, B, 1.0,
                    splits=ks)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_launches_do_not_grow_with_images_or_groups(path):
    """one filter copy, then filter rows (tf32x1: none, it reads the 16-byte rows in place), window rows and the GEMM, for 1
    or many images, 2 or 16 groups -- the non-grouped entry's count"""
    many = 4 if EMU else 16
    want = {"f16x3": 4, "tf32x3": 4, "tf32x1": 3}[path]
    for ishape, kshape, groups in [((1, 128, 8, 8), (16, 64, 3, 3), 2), ((many, 128, 8, 8), (16, 64, 3, 3), 2),
                                   ((1, 1024, 6, 6), (64, 64, 3, 3), 16), ((many, 1024, 6, 6), (64, 64, 3, 3), 16)]:
        c = GGrad(ishape, kshape, (1, 1), (1, 1), groups)
        _, n = c.grouped(PATHS[path], "relu_grad")
        ks, _ = plan(path, c.Cg, c.HW, c.Kp, batch=ishape[0] * groups)
        assert n - (1 if ks > 1 else 0) == want, (ishape, groups, n)
        assert L.last_path() == PATHS[path]


_SUB = """
import hashlib, sys, numpy as np, laser_b200 as L, test_gpu_conv_grouped_input_grad as T
c = T.GGrad(%r, %r, (1, 1), (1, 1), %d, seed=23)
dx, n = c.grouped(int(sys.argv[1]), "tanh_grad", 0.5, 1.25)
print("RESULT", n, hashlib.sha256(dx.tobytes()).hexdigest())
"""


def _subprocess(code, *args, env=None):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), **(env or {}))
    out = subprocess.run([sys.executable, "-c", code] + list(args), cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return [line for line in out.stdout.splitlines() if line.startswith("RESULT")][0].split()


@pytest.mark.parametrize("path", ["f16x3", "tf32x1"])
def test_chunks_of_whole_images_give_the_bits_of_one(path):
    """a 1 MB workspace cap holds one image's G problems at a time: the filter copy once, 3 launches per image, the same dX"""
    ishape, kshape, groups = (3, 256, 24, 24), (32, 64, 3, 3), 4
    code = _SUB % (ishape, kshape, groups)
    one = _subprocess(code, str(PATHS[path]))
    many = _subprocess(code, str(PATHS[path]), env={"LASER_B200_BATCH_WS_MB": "1"})
    per_chunk = 3 if path == "f16x3" else 2
    assert int(many[1]) == 1 + 3 * per_chunk and int(one[1]) == 1 + per_chunk, (one, many)
    assert many[2] == one[2]


# ---- reference checks ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", ["3x3", "1x1"])
@pytest.mark.parametrize("path", list(PATHS))
def test_one_group_is_conv2d_input_grad_fused(path, geom):
    if geom == "3x3":
        ishape, kshape, padding = (((2, 8, 6, 6), (16, 8, 3, 3)) if EMU else ((3, 96, 20, 20), (64, 96, 3, 3))) + ((1, 1),)
    else:
        ishape, kshape, padding = (((2, 8, 6, 6), (16, 8, 1, 1)) if EMU else ((3, 96, 14, 14), (64, 96, 1, 1))) + ((0, 0),)
    c = GGrad(ishape, kshape, padding, (1, 1), 1)
    got, got_n = c.grouped(PATHS[path], "relu_grad", -0.5, 1.25)
    got_path = L.last_path()
    dx = c.dx0(1.25)

    def plain():
        L.conv2d_input_grad_fused(dx, ishape, c.tdy, c.tw, kshape, padding, (1, 1), -0.5, 1.25, op="relu_grad",
                                  aux=c.taux["relu_grad"], path=PATHS[path])
    want_n = launches(plain)
    assert (got_n, got_path) == (want_n, L.last_path())
    assert_bits(got, dx.cpu().numpy().reshape(ishape))


@pytest.mark.parametrize("geom", list(NARROW)[:4] + list(WIDE))
def test_auto_path(geom):
    """PATH_AUTO: the exact path when Cg < 64 or K' < 64 (n * G > 1 images), else the path conv2d_input_grad_fused takes for one
    group (the emulated wide groups are small enough for the exact path there too), with the bits of the per-group calls"""
    c = GGrad(*(WIDE[geom] if geom in WIDE else NARROW[geom]))
    got, _ = c.grouped(L.PATH_AUTO, "relu_grad", 1.0, 0.0)
    path = L.last_path()
    if c.Cg < 64 or c.Kp < 64:
        assert path == L.PATH_SIMT
    else:
        c.per_group_calls(L.PATH_AUTO, "relu_grad")
        assert path == L.last_path()
    assert_bits(got, c.per_group_calls(path, "relu_grad"))


def input_grad_f64(c, z):
    import torch
    return torch.nn.grad.conv2d_input(c.ishape, torch.from_numpy(c.w.astype(np.float64)), torch.from_numpy(z.astype(np.float64)),
                                      stride=c.strides, padding=c.padding, groups=c.groups).numpy()


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("geom", ["depthwise", "depthwise_stride2", "cg4"] + list(WIDE)[:1])
def test_accuracy_against_float64(path, geom):
    pytest.importorskip("torch")
    c = GGrad(*(WIDE[geom] if geom in WIDE else NARROW[geom]))
    got, _ = c.grouped(PATHS[path])
    ref = input_grad_f64(c, c.dy).astype(np.float32)
    if path == "tf32x1" or (path == "auto" and L.last_path() == L.PATH_TF32X1):
        assert O.normwise_relative_error(got, ref) < 2e-3
    else:
        assert O.normwise_relative_error(got, ref) < 2e-6 and O.mean_relative_error(got, ref) <= 1e-5


@pytest.mark.parametrize("path", ["simt"] + TC)
def test_layer_backward_pass_against_torch_autograd(path):
    """conv2d_grouped_fused with bias and relu, then this entry with relu_grad and the forward output as aux: torch autograd of
    the grouped convolution in float64 with the same relu mask is the float64 product of the operands, and dX is within the
    bound (the exact path: the oracle's bits)"""
    torch = pytest.importorskip("torch")
    ishape, kshape, padding, strides, groups = WIDE[list(WIDE)[1]]
    rng = np.random.default_rng(21)
    x = rng.uniform(-1, 1, ishape).astype(np.float32)
    w = rng.uniform(-1, 1, kshape).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, kshape[0]).astype(np.float32)
    c = GGrad(ishape, kshape, padding, strides, groups, w=w)
    dy = rng.uniform(-1, 1, c.oshape).astype(np.float32)
    c = GGrad(ishape, kshape, padding, strides, groups, w=w, dy=dy)
    tz = dev(np.zeros(c.oshape, np.float32))
    L.conv2d_grouped_fused(tz, dev(x), ishape, c.tw, kshape, padding, strides, groups, bias=dev(bias), activation="relu",
                           path=PATHS[path])
    sync()
    z = tz.cpu().numpy().reshape(c.oshape).copy()
    dx = dev(np.full(ishape, np.nan, np.float32))
    L.conv2d_grouped_input_grad_fused(dx, ishape, c.tdy, c.tw, kshape, padding, strides, groups, op="relu_grad", aux=tz,
                                      path=PATHS[path])
    sync()
    got = dx.cpu().numpy().reshape(ishape)
    gz = np.where(z > 0, dy, np.float32(0)).astype(np.float32)
    tx = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    y = torch.nn.functional.conv2d(tx, torch.from_numpy(w.astype(np.float64)), torch.from_numpy(bias.astype(np.float64)),
                                   stride=strides, padding=padding, groups=groups)
    y.backward(torch.from_numpy(gz.astype(np.float64)))
    n = ishape[0]
    A, B = c.operands(gz)
    ab = (A.astype(np.float64) @ B.astype(np.float64)).reshape(ishape)
    np.testing.assert_allclose(ab, tx.grad.numpy(), rtol=0, atol=1e-12 * np.abs(tx.grad.numpy()).max())
    if path == "simt":    # (its bits: test_exact_path_matches_the_oracle)
        assert O.normwise_relative_error(got, tx.grad.numpy().astype(np.float32)) < 2e-6
        return
    ks, _ = plan(path, c.Cg, c.HW, c.Kp, batch=n * groups)
    bound_and_check("grouped input gradient", path, "conv_grouped_input_grad", got.reshape(n, groups, c.Cg, c.HW), A, B, 1.0,
                    splits=ks)


def _raw(ishape=(2, 4, 5, 5), kshape=(6, 2, 3, 3), padding=(1, 1), strides=(1, 1), groups=2, op=None, path=L.PATH_AUTO, null=None):
    dx = dev(np.full(2 * 4 * 25, 3.0, np.float32))
    w, dy = dev(np.ones(6 * 2 * 9, np.float32)), dev(np.ones(2 * 6 * 25, np.float32))
    ptrs = {"dx": dx.data_ptr(), "w": w.data_ptr(), "dy": dy.data_ptr()}
    if null:
        ptrs[null] = None
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_conv2d_grouped_input_grad_f32_fused_dev(ptrs["dx"], i4(*ishape), ptrs["dy"], ptrs["w"], i4(*kshape),
                                                                        i2(*padding), i2(*strides), groups, 1.0, 0.0, op, path,
                                                                        G._current_stream())
    sync()
    assert np.all(dx.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    aux = dev(np.ones(2 * 6 * 25, np.float32))
    relu_grad = lambda rs, cs: ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD, aux=aux.data_ptr(), auxRowStride=rs,
                                                            auxColStride=cs))
    for kw in (dict(groups=0), dict(groups=-2), dict(groups=3), dict(ishape=(2, 5, 5, 5), kshape=(6, 1, 3, 3), groups=5),
               dict(kshape=(6, 1, 3, 3)), dict(kshape=(6, 4, 3, 3)), dict(strides=(0, 1)), dict(padding=(-1, 0)),
               dict(kshape=(6, 2, 8, 3)), dict(path=5), dict(path=-1), dict(op=ctypes.byref(_capi.OperandOp(op=9))),
               dict(op=ctypes.byref(_capi.OperandOp(op=_capi.OP_RELU_GRAD))), dict(op=relu_grad(26, 1)), dict(op=relu_grad(25, 2)),
               dict(op=relu_grad(1, 25)), dict(null="dx"), dict(null="w"), dict(null="dy")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    for path in PATHS.values():
        assert _raw(ishape=(0, 4, 5, 5), path=path) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 4, 5, 5), null="dx") == (_capi.E_OK, 0)
    # K' = c_out / G * kH * kW = 2^29 * 9 past int32 (nothing is read: the check comes first)
    assert _raw(kshape=(2 ** 30, 2, 3, 3)) == (_capi.E_UNSUPPORTED, 0)
    # a kernel window of thousands of taps does not fit the direct kernel's shared-memory tile
    assert _raw(ishape=(2, 4, 120, 120), kshape=(6, 2, 110, 110), padding=(0, 0), path=L.PATH_SIMT) == (_capi.E_UNSUPPORTED, 0)


@pytest.mark.skipif(EMU, reason="sizes of the depthwise layers of a real network")
def test_depthwise_network_layer():
    """MobileNet-size depthwise 3 x 3 (32 x 144 x 56 x 56) on PATH_AUTO: the direct kernel, one launch, the bits of the per-group
    calls on the exact path"""
    c = GGrad((32, 144, 56, 56), (144, 1, 3, 3), (1, 1), (1, 1), 144)
    got, n = c.grouped(L.PATH_AUTO, "relu_grad", 1.0, 0.0)
    assert L.last_path() == L.PATH_SIMT and n == 1
    assert_bits(got, c.per_group_calls(L.PATH_SIMT, "relu_grad"))


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode of this file's bound checks (the last test of the file)"""
    from test_gpu_error_bounds import RATIOS
    mine = {k: r for k, r in RATIOS.items() if k[1] == "conv_grouped_input_grad"}
    if not mine:
        pytest.skip("no case ran")
    with capsys.disabled():
        print("\nlargest err / bound of the grouped input gradient:\n" +
              "\n".join("  %-7s %.3g" % (m, r) for (m, _), r in sorted(mine.items())))
