"""GPU: the grouped fused convolution laser_b200_conv2d_grouped_f32_fused_dev (torch.nn.Conv2d(groups=G)).  The exact path is
a direct CUDA-core kernel that must give, bit for bit, the oracle's conv2d_im2col of each group's slice, in one launch.  The
tensor-core paths are one batched GEMM whose filters repeat with period G; they must give the bits of G conv2d_fused calls on
contiguous per-group copies, meet the per-element float64 bound, and take 3 launches whatever n and G.  groups == 1 is
conv2d_fused itself."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, sync

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402
from test_gpu_error_bounds import bound_and_check  # noqa: E402

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
TC = ["f16x3", "tf32x3", "tf32x1"]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# (ishape, kshape = (c_out, c_in / G, kH, kW), padding, strides, groups)
NARROW = {
    "depthwise": ((2, 8, 9, 9), (8, 1, 3, 3), (1, 1), (1, 1), 8),
    "multiplier2": ((2, 4, 7, 7), (8, 1, 3, 3), (1, 1), (1, 1), 4),
    "stride2_non_square": ((2, 6, 9, 7), (6, 1, 3, 2), (1, 0), (2, 1), 6),
    "depthwise_7x7_pad3": ((2, 4, 10, 10), (4, 1, 7, 7), (3, 3), (1, 1), 4),
    "cg4": ((2, 16, 8, 8), (16, 4, 3, 3), (1, 1), (1, 1), 4),
    "cg64_kc_flush": ((1, 128, 5, 5), (8, 64, 3, 3), (1, 1), (1, 1), 2),    # Kg = 576 > 512
    "grouped_1x1": ((2, 8, 6, 6), (12, 2, 1, 1), (0, 0), (1, 1), 4),
    "odd_out_w": ((2, 6, 6, 13), (6, 2, 3, 3), (1, 1), (1, 2), 3),           # outW = 7
    "wide_out_w": ((1, 2, 4, 150), (2, 1, 3, 3), (1, 1), (1, 1), 2),         # two column tiles
}
# groups wide enough for the tensor cores on PATH_AUTO (Mg >= 64, Kg >= 64), Kg <= 768 (split-K off on both sides)
WIDE = {
    "g2": ((2, 16, 8, 8), (128, 8, 3, 3), (1, 1), (1, 1), 2),
    "g4_stride2": ((2, 32, 9, 9), (256, 8, 3, 3), (1, 1), (2, 2), 4),
} if EMU else {
    "g4": ((4, 64, 14, 14), (256, 16, 3, 3), (1, 1), (1, 1), 4),
    "g8_stride2": ((3, 128, 15, 15), (512, 16, 3, 3), (1, 1), (2, 2), 8),
    "g2_1x1": ((2, 128, 14, 14), (128, 64, 1, 1), (0, 0), (1, 1), 2),
}
ACTS = {"relu": lambda v: np.maximum(v, 0), "tanh": np.tanh, "sigmoid": lambda v: 1 / (1 + np.exp(-v))}


class GConv:
    def __init__(self, ishape, kshape, padding, strides, groups, seed=1, lo=-1.0, hi=1.0):
        self.ishape, self.kshape, self.padding, self.strides, self.groups = ishape, kshape, padding, strides, groups
        self.x = O.fill_uniform_f32(int(np.prod(ishape)), seed, lo, hi).reshape(ishape)
        self.k = O.fill_uniform_f32(int(np.prod(kshape)), seed + 1, lo, hi).reshape(kshape)
        self.bias = O.fill_uniform_f32(kshape[0], seed + 2, -0.5, 0.5)
        n, c, h, w = ishape
        self.Cg, self.Mg = c // groups, kshape[0] // groups
        o = O.conv2d_out_shape((n, self.Cg, h, w), (self.Mg,) + tuple(kshape[1:]), padding, strides)
        self.oshape = (n, kshape[0], o[2], o[3])
        self.tx, self.tk, self.tb = dev(self.x), dev(self.k), dev(self.bias)

    def grouped(self, path, bias=False, activation="none", groups=None):
        out = dev(np.full(self.oshape, np.nan, np.float32))
        L.conv2d_grouped_fused(out, self.tx, self.ishape, self.tk, self.kshape, self.padding, self.strides,
                               self.groups if groups is None else groups, bias=self.tb if bias else None, activation=activation,
                               path=path)
        sync()
        return out.cpu().numpy().copy()

    def slices(self, g):
        xs = np.ascontiguousarray(self.x[:, g * self.Cg:(g + 1) * self.Cg])
        ks = np.ascontiguousarray(self.k[g * self.Mg:(g + 1) * self.Mg])
        return xs, ks, (self.ishape[0], self.Cg) + tuple(self.ishape[2:]), (self.Mg,) + tuple(self.kshape[1:])

    def per_group_calls(self, path, bias=False, activation="none"):
        """G conv2d_fused calls on contiguous per-group copies"""
        out = np.empty(self.oshape, np.float32)
        for g in range(self.groups):
            xs, ks, ish, ksh = self.slices(g)
            o = dev(np.full((ish[0], self.Mg) + self.oshape[2:], np.nan, np.float32))
            b = dev(self.bias[g * self.Mg:(g + 1) * self.Mg]) if bias else None
            L.conv2d_fused(o, dev(xs), ish, dev(ks), ksh, self.padding, self.strides, bias=b, activation=activation, path=path)
            sync()
            out[:, g * self.Mg:(g + 1) * self.Mg] = o.cpu().numpy()
        return out

    def oracle(self):
        """the oracle's conv2d_im2col of each group's slice (exact, fp32)"""
        out = np.empty(self.oshape, np.float32)
        for g in range(self.groups):
            xs, ks, ish, ksh = self.slices(g)
            out[:, g * self.Mg:(g + 1) * self.Mg] = O.conv2d_im2col(xs, ish, ks, ksh, self.padding, self.strides)
        return out

    def operands(self):
        """A [n][G][Mg][Kg] and B [n][G][Kg][P] as multiplied: the filters and each group's im2col matrix"""
        n = self.ishape[0]
        A = np.broadcast_to(self.k.reshape(self.groups, self.Mg, -1), (n, self.groups, self.Mg, self.k[0].size))
        Bs = []
        for i in range(n):
            for g in range(self.groups):
                xs, ks, ish, ksh = self.slices(g)
                Bs.append(O.im2col(np.ascontiguousarray(xs[i]), ish, ksh, self.padding, self.strides))
        return A, np.stack(Bs).reshape((n, self.groups) + Bs[0].shape)


def assert_bits(got, want):
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def launches(fn):
    sync()
    n0 = L.launch_count()
    fn()
    return L.launch_count() - n0


# ---- exact path: the direct kernel ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi", ["none", "bias", "bias_relu"])
@pytest.mark.parametrize("geom", list(NARROW))
def test_exact_path_equals_the_oracle_per_group(geom, epi):
    c = GConv(*NARROW[geom])
    got = c.grouped(L.PATH_SIMT, epi != "none", "relu" if epi == "bias_relu" else "none")
    want = c.oracle()
    if epi != "none":
        want = want + c.bias[None, :, None, None]
    if epi == "bias_relu":
        want = np.maximum(want, np.float32(0))
    assert_bits(got, want.astype(np.float32))


@pytest.mark.parametrize("activation", ["tanh", "sigmoid"])
@pytest.mark.parametrize("geom", ["depthwise", "cg4", "cg64_kc_flush"])
def test_exact_path_activations_are_the_exact_kernels(geom, activation):
    """tanh and sigmoid through the exact kernel's epilogue: the bits of conv2d_fused's exact path on each group's slice"""
    c = GConv(*NARROW[geom])
    assert_bits(c.grouped(L.PATH_SIMT, True, activation), c.per_group_calls(L.PATH_SIMT, True, activation))


def test_inf_filter_tap_at_the_border_gives_nan_where_the_oracle_does():
    c = GConv(*NARROW["cg4"])
    c.k[5, 2, 0, 0] = np.inf          # output channel 5 (group 1), top-left tap: in the padding for the first row and column
    c.tk = dev(c.k)
    got, want = c.grouped(L.PATH_SIMT), c.oracle()
    nan = np.isnan(want)
    assert nan.any()
    assert np.array_equal(np.isnan(got), nan)
    assert_bits(got[~nan], want[~nan])   # (the NaN's encoding is the processor's: the GPU's and the CPU oracle's differ)


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("geom", ["depthwise", "cg4", "cg64_kc_flush"])
def test_exact_path_is_one_launch(geom, n):
    ishape, kshape, padding, strides, groups = NARROW[geom]
    c = GConv((n,) + ishape[1:], kshape, padding, strides, groups)
    assert launches(lambda: c.grouped(L.PATH_SIMT, True, "relu")) == 1
    assert L.last_path() == L.PATH_SIMT


# ---- tensor-core paths: one batched GEMM with the filters repeating every G problems -------------------------------------
@pytest.mark.parametrize("epi", [(False, "none"), (True, "relu"), (True, "tanh")])
@pytest.mark.parametrize("geom", list(WIDE) + ["cg4", "multiplier2", "grouped_1x1"])
@pytest.mark.parametrize("path", TC)
def test_tensor_core_paths_equal_per_group_calls(path, geom, epi):
    c = GConv(*(WIDE[geom] if geom in WIDE else NARROW[geom]))
    assert_bits(c.grouped(PATHS[path], *epi), c.per_group_calls(PATHS[path], *epi))


@pytest.mark.parametrize("activation", ["none", "sigmoid"])
@pytest.mark.parametrize("path", TC)
def test_tensor_core_paths_meet_the_per_element_bound(path, activation):
    c = GConv(*list(WIDE.values())[0], lo=-0.5, hi=0.5)
    got = c.grouped(PATHS[path], True, activation)
    A, B = c.operands()
    n, co, oh, ow = c.oshape
    bias = np.broadcast_to(c.bias.reshape(c.groups, c.Mg)[None, :, :, None].astype(np.float64), (n, c.groups, c.Mg, oh * ow))
    bound_and_check("grouped", path, "conv2d_grouped", got.reshape(n, c.groups, c.Mg, oh * ow), A, B, 1.0, bias=bias,
                    act=activation)


@pytest.mark.parametrize("path", ["f16x3", "tf32x3"])
def test_tensor_core_launches_do_not_grow_with_images_or_groups(path):
    """filter rows, window rows, GEMM: 3 launches for 1 or many images, 2 or 32 groups (filter rows 16-byte aligned; tf32x1
    reads such filters in place: one launch fewer)"""
    many = 4 if EMU else 16
    cases = [((1, 16, 8, 8), (64, 8, 3, 3), 2), ((many, 16, 8, 8), (64, 8, 3, 3), 2),
             ((1, 128, 6, 6), (64, 4, 3, 3), 32), ((many, 128, 6, 6), (64, 4, 3, 3), 32)]
    for ishape, kshape, groups in cases:
        c = GConv(ishape, kshape, (1, 1), (1, 1), groups)
        assert launches(lambda: c.grouped(PATHS[path], True, "relu")) == 3, (ishape, groups)
        assert L.last_path() == PATHS[path]


_SUB = """
import numpy as np, laser_b200 as L, test_gpu_conv_grouped as T
c = T.GConv(%r, %r, (1, 1), (1, 1), %d)
n0 = L.launch_count()
got = c.grouped(L.PATH_F16X3, True, "tanh")
print("LAUNCHES", L.launch_count() - n0)
np.save(%r, got)
"""


def test_chunks_of_whole_images_are_bit_identical(tmp_path):
    """a 1 MB workspace cap holds one image's G problems at a time: 3 launches per image, the bits of one chunk"""
    ishape, kshape, groups = ((3, 16, 32, 32), (128, 4, 3, 3), 4) if EMU else ((3, 32, 32, 32), (128, 8, 3, 3), 4)
    whole = GConv(ishape, kshape, (1, 1), (1, 1), groups).grouped(L.PATH_F16X3, True, "tanh")
    f = str(tmp_path / "c.npy")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), LASER_B200_BATCH_WS_MB="1")
    out = subprocess.run([sys.executable, "-c", _SUB % (ishape, kshape, groups, f)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert int(out.stdout.split("LAUNCHES")[1].split()[0]) == 3 * 3
    assert_bits(np.load(f), whole)


# ---- reference checks ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(PATHS))
def test_one_group_is_conv2d_fused(path):
    ishape, kshape = ((2, 8, 6, 6), (64, 8, 3, 3)) if EMU else ((3, 16, 20, 20), (96, 16, 3, 3))
    c = GConv(ishape, kshape, (1, 1), (1, 1), 1)
    got_n = launches(lambda: c.grouped(PATHS[path], True, "relu"))
    got, got_path = c.grouped(PATHS[path], True, "relu"), L.last_path()
    out = dev(np.full(c.oshape, np.nan, np.float32))

    def fused():
        L.conv2d_fused(out, c.tx, ishape, c.tk, kshape, (1, 1), (1, 1), bias=c.tb, activation="relu", path=PATHS[path])
        sync()
    want_n = launches(fused)
    assert (got_n, got_path) == (want_n, L.last_path())
    assert_bits(got, out.cpu().numpy())


@pytest.mark.parametrize("geom", list(NARROW) + list(WIDE))
def test_auto_path(geom):
    """PATH_AUTO: the direct kernel on narrow groups, the path conv2d_fused takes for one group on wide ones, with its bits (these
    wide groups are small enough for the exact path there too; tools/conv_grouped_probe.py shows the tensor-core side)"""
    c = GConv(*(WIDE[geom] if geom in WIDE else NARROW[geom]))
    got = c.grouped(L.PATH_AUTO, True, "relu")
    path = L.last_path()
    if geom in NARROW:
        assert path == L.PATH_SIMT
        return
    want = c.per_group_calls(L.PATH_AUTO, True, "relu")
    assert path == L.last_path()
    assert_bits(got, want)


def grouped_conv_f64(x, k, padding, strides, groups):
    """float64 torch.nn.functional.conv2d(groups=...) semantics, in numpy"""
    n, C, H, W = x.shape
    co, cg, kH, kW = k.shape
    mg = co // groups
    xp = np.zeros((n, C, H + 2 * padding[0], W + 2 * padding[1]))
    xp[:, :, padding[0]:padding[0] + H, padding[1]:padding[1] + W] = x
    oh, ow = 1 + (H + 2 * padding[0] - kH) // strides[0], 1 + (W + 2 * padding[1] - kW) // strides[1]
    out = np.zeros((n, co, oh, ow))
    for g in range(groups):
        xg = xp[:, g * cg:(g + 1) * cg]
        for i in range(kH):
            for j in range(kW):
                win = xg[:, :, i:i + strides[0] * oh:strides[0], j:j + strides[1] * ow:strides[1]]
                out[:, g * mg:(g + 1) * mg] += np.einsum("ncij,mc->nmij", win, k[g * mg:(g + 1) * mg, :, i, j].astype(np.float64))
    return out


@pytest.mark.parametrize("path", ["simt", "f16x3", "tf32x3", "tf32x1", "auto"])
@pytest.mark.parametrize("geom", ["depthwise", "cg4", "odd_out_w"] + list(WIDE)[:1])
def test_accuracy_against_float64(path, geom):
    c = GConv(*(WIDE[geom] if geom in WIDE else NARROW[geom]), lo=-0.1, hi=0.1)
    got = c.grouped(PATHS[path], True, "sigmoid")
    if EMU:
        pre = grouped_conv_f64(c.x, c.k, c.padding, c.strides, c.groups)
    else:
        import torch
        pre = torch.nn.functional.conv2d(torch.from_numpy(c.x).double(), torch.from_numpy(c.k).double(), stride=c.strides,
                                         padding=c.padding, groups=c.groups).numpy()
    ref = ACTS["sigmoid"](pre + c.bias[None, :, None, None]).astype(np.float32)
    if path == "tf32x1":
        assert O.normwise_relative_error(got, ref) < 2e-3
    else:
        assert O.normwise_relative_error(got, ref) < 2e-6 and O.mean_relative_error(got, ref) <= 1e-5


def _raw(ishape=(2, 4, 5, 5), kshape=(6, 2, 3, 3), padding=(1, 1), strides=(1, 1), groups=2, epi=None, path=L.PATH_AUTO,
         null=None):
    out = dev(np.full(2 * 6 * 25, 3.0, np.float32))
    x, k = dev(np.ones(2 * 4 * 25, np.float32)), dev(np.ones(6 * 2 * 9, np.float32))
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    ptrs = [out.data_ptr(), x.data_ptr(), k.data_ptr()]
    if null is not None:
        ptrs[null] = None
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_conv2d_grouped_f32_fused_dev(ptrs[0], ptrs[1], i4(*ishape), ptrs[2], i4(*kshape), i2(*padding),
                                                              i2(*strides), groups, epi, path, G._current_stream())
    sync()
    return rc, L.launch_count() - n0, out.cpu().numpy().copy()


def test_argument_errors_launch_nothing():
    bias = dev(np.zeros(6, np.float32))
    for kw in (dict(groups=0), dict(groups=-2), dict(groups=3), dict(ishape=(2, 5, 5, 5), kshape=(6, 1, 3, 3), groups=5),
               dict(kshape=(6, 1, 3, 3)), dict(kshape=(6, 4, 3, 3)), dict(strides=(0, 1)), dict(kshape=(6, 2, 8, 3)),
               dict(padding=(-1, 0)), dict(path=5), dict(path=-1), dict(epi=ctypes.byref(_capi.Epilogue(None, 1, 7))),
               dict(epi=ctypes.byref(_capi.Epilogue(bias.data_ptr(), 0, 0))), dict(null=0), dict(null=1), dict(null=2)):
        rc, n, out = _raw(**kw)
        assert (rc, n) == (_capi.E_INVAL, 0), kw
        assert np.all(out == 3.0)
    rc, n, out = _raw(ishape=(0, 4, 5, 5))
    assert (rc, n) == (_capi.E_OK, 0) and np.all(out == 3.0)


@pytest.mark.skipif(EMU, reason="sizes of the depthwise layers of a real network")
def test_depthwise_network_layer():
    """MobileNet-size depthwise 3 x 3 (32 x 144 x 56 x 56) on PATH_AUTO: the direct kernel, the oracle's bits"""
    c = GConv((32, 144, 56, 56), (144, 1, 3, 3), (1, 1), (1, 1), 144)
    got = c.grouped(L.PATH_AUTO)
    assert L.last_path() == L.PATH_SIMT
    assert_bits(got, c.oracle())
