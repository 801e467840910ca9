"""GPU: the channels-last fused convolution laser_b200_conv2d_nhwc_f32_fused_dev -- NHWC images and output, the filter matrix
[kH * kW * c_in][c_out] read with its strides, ONE product output[n * P + p][co] = sum_k rows[n * P + p][k] * Wmat[k][co] whose A
(the windows, one row per output pixel) is prepared straight from the images.  On every path the output must equal, bit for
bit, the fused GEMM over the NHWC im2col rows materialised in numpy with the same filter view and epilogue; the exact path
equals the CPU oracle; the reference's known answers hold; the tensor-core paths meet the per-element bound of
tests/test_gpu_error_bounds.py (as the NCHW entry does on the same data); chunks give the bits of one chunk; the launch count
does not grow with the images; argument errors launch nothing."""
import ctypes
import json
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
# (ishape (n, c, h, w), kshape (c_out, c_in, kH, kW), padding, strides)
GEOMS = {
    "pad1": ((2, 8, 8, 8), (16, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 64, 20, 20), (64, 64, 3, 3), (1, 1), (1, 1)),
    "stride2": ((2, 4, 9, 9), (12, 4, 3, 3), (0, 0), (2, 2)) if EMU else ((5, 32, 17, 17), (48, 32, 3, 3), (0, 0), (2, 2)),
    "non_square": ((2, 4, 7, 9), (8, 4, 3, 5), (1, 2), (1, 2)) if EMU else ((3, 16, 16, 19), (32, 16, 3, 5), (1, 2), (2, 1)),
    # c = 3: the scalar path (K = 27)
    "rgb_c3": ((2, 3, 10, 10), (16, 3, 3, 3), (1, 1), (2, 2)) if EMU else ((4, 3, 32, 32), (64, 3, 3, 3), (1, 1), (2, 2)),
    # c = 5 (scalar path), c_out not a multiple of 4
    "c5_cout_odd": ((2, 5, 7, 6), (10, 5, 3, 2), (1, 0), (1, 1)) if EMU else ((3, 5, 15, 14), (30, 5, 3, 2), (1, 0), (1, 1)),
    "one_by_one_stride2": ((2, 8, 7, 7), (12, 8, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 32, 15, 15), (64, 32, 1, 1), (0, 0), (2, 2)),
    # K = 1152: a CTA per row
    "long_k": ((1, 128, 4, 4), (8, 128, 3, 3), (1, 1), (1, 1)) if EMU else ((2, 128, 12, 12), (64, 128, 3, 3), (1, 1), (1, 1)),
}
# (bias, activation), one per geometry in turn
EPIS = [(False, "none"), (True, "none"), (True, "relu"), (True, "tanh"), (True, "sigmoid")]


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def up(x, m):
    return -(-x // m) * m


def nhwc_rows(x, ishape, kshape, padding, strides):
    """[n * outH * outW][kH * kW * c] im2col rows of the NHWC images x: output pixel (oh, ow)'s window in (kh, kw, c) order"""
    n, C, H, W = ishape
    kH, kW = kshape[2:]
    (pH, pW), (sH, sW) = padding, strides
    oh, ow = 1 + (H + 2 * pH - kH) // sH, 1 + (W + 2 * pW - kW) // sW
    xp = np.zeros((n, H + 2 * pH, W + 2 * pW, C), x.dtype)
    xp[:, pH:pH + H, pW:pW + W] = x
    hi = (np.arange(oh) * sH)[:, None] + np.arange(kH)[None, :]
    wi = (np.arange(ow) * sW)[:, None] + np.arange(kW)[None, :]
    return np.ascontiguousarray(xp[:, hi[:, None, :, None], wi[None, :, None, :], :].reshape(n * oh * ow, kH * kW * C))


class Conv:
    """one convolution's data: NHWC images x, the filter matrix wmat [K][c_out] ((kh, kw, ci) rows), a bias per output channel"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, x=None, wmat=None):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        n, C, H, W = ishape
        co, _, kH, kW = kshape
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        self.P, self.K, self.co = self.oshape[2] * self.oshape[3], kH * kW * C, co
        self.x = O.fill_uniform_f32(n * H * W * C, seed, -1, 1).reshape(n, H, W, C) if x is None else x
        self.wmat = O.fill_uniform_f32(self.K * co, seed + 1, -1, 1).reshape(self.K, co) if wmat is None else wmat
        self.bias = O.fill_uniform_f32(co, seed + 2, -0.5, 0.5)
        self.tx, self.tb = dev(self.x), dev(self.bias)
        self.views = {"hwio": (dev(self.wmat), (co, 1)), "ohwi": (dev(np.ascontiguousarray(self.wmat.T)), (1, self.K))}

    def out0(self):
        return dev(np.full((self.ishape[0] * self.P, self.co), np.nan, np.float32))

    def fused(self, path, layout="hwio", bias=False, activation="none"):
        """-> (output [n * P][c_out], launches)"""
        w, st = self.views[layout]
        kernel = w
        if not EMU and layout == "ohwi":
            kernel = w.t()   # torch's channels_last weight seen as [K][c_out]: strides (1, K) read from the view
        out = self.out0()
        sync()
        n0 = L.launch_count()
        L.conv2d_nhwc_fused(out, self.tx, self.ishape, kernel, self.kshape, self.padding, self.strides,
                            bias=self.tb if bias else None, activation=activation, path=path,
                            kernel_strides=st if EMU else None)
        sync()
        return out.cpu().numpy().copy(), L.launch_count() - n0

    def rows(self):
        return nhwc_rows(self.x, self.ishape, self.kshape, self.padding, self.strides)

    def gemm(self, path, layout="hwio", bias=False, activation="none"):
        """the fused GEMM over the materialised rows [n * P][round_up(K, 4)] and the same filter view"""
        K, ld = self.K, up(self.K, 4)
        a = np.zeros((self.ishape[0] * self.P, ld), np.float32)
        a[:, :K] = self.rows()
        w, (rs, cs) = self.views[layout]
        out = self.out0()
        G.gemm_strided_fused(a.shape[0], self.co, K, 1.0, dev(a), ld, 1, w, rs, cs, 0.0, out, self.co, 1,
                             bias=self.tb if bias else None, bias_per_row=False, activation=activation, path=path)
        sync()
        return out.cpu().numpy().copy()

    def nchw(self, path):
        """the NCHW fused entry on the same data -> its output as [n][P][c_out]"""
        n, C, H, W = self.ishape
        co, _, kH, kW = self.kshape
        k = np.ascontiguousarray(self.wmat.reshape(kH, kW, C, co).transpose(3, 2, 0, 1))
        out = dev(np.full(self.oshape, np.nan, np.float32))
        L.conv2d_fused(out, dev(np.ascontiguousarray(self.x.transpose(0, 3, 1, 2))), self.ishape, dev(k), self.kshape, self.padding,
                       self.strides, path=path)
        sync()
        return out.cpu().numpy().reshape(n, co, self.P).transpose(0, 2, 1)


@pytest.mark.parametrize("layout", ["hwio", "ohwi"])
@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_gemm_over_the_rows(path, geom, layout):
    """each geometry with one epilogue (they take turns); PATH_AUTO: the GEMM on the path the entry resolved"""
    bias, act = EPIS[list(GEOMS).index(geom) % len(EPIS)]
    c = Conv(*GEOMS[geom])
    got, _ = c.fused(PATHS[path], layout, bias, act)
    resolved = L.last_path()
    if path != "auto":
        assert resolved == PATHS[path]
    assert not np.isnan(got).any()
    assert_bits(got, c.gemm(resolved, layout, bias, act))


@pytest.mark.parametrize("geom", list(GEOMS))
def test_auto_takes_the_path_of_the_nchw_entry(geom):
    c = Conv(*GEOMS[geom], seed=3)
    c.fused(L.PATH_AUTO)
    nhwc = L.last_path()
    c.nchw(L.PATH_AUTO)
    assert nhwc == L.last_path()


@pytest.mark.parametrize("layout", ["hwio", "ohwi"])
@pytest.mark.parametrize("geom", ["stride2", "rgb_c3"])
def test_exact_path_matches_the_oracle(geom, layout):
    c = Conv(*GEOMS[geom], seed=5)
    got, _ = c.fused(L.PATH_SIMT, layout)
    rows = c.rows()
    want = np.zeros((rows.shape[0], c.co), np.float32)
    O.gemm_strided(rows.shape[0], c.co, c.K, 1.0, rows, c.K, 1, np.ascontiguousarray(c.wmat), c.co, 1, 0.0, want, c.co, 1)
    assert_bits(got, want)


def conv_cases():
    with open(os.path.join(HERE, "golden", "conv2d_known_answer.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("case", conv_cases(), ids=lambda c: c["src"])
def test_known_answer(case, path):
    """the reference's vectors with the input through nchw2nhwc and the filters through kernel_to_hwcc ([kH][kW][C_in][C_out])"""
    ishape, kshape = tuple(case["ishape"]), tuple(case["kshape"])
    inp = np.array(case["input"], np.float32).reshape(ishape)
    ker = np.array(case["kernel"], np.float32).reshape(kshape)
    tgt = np.array(case["target"], np.float32)
    oshape = tuple(O.conv2d_out_shape(ishape, kshape, case["padding"], case["strides"]))
    co, ci, kH, kW = kshape
    wmat = np.ascontiguousarray(ker.transpose(2, 3, 1, 0).reshape(kH * kW * ci, co))
    out = dev(np.full((oshape[0], oshape[2], oshape[3], co), 99.0, np.float32))
    L.conv2d_nhwc_fused(out, dev(np.ascontiguousarray(inp.transpose(0, 2, 3, 1))), ishape, dev(wmat), kshape, case["padding"],
                        case["strides"], path=PATHS[path], kernel_strides=(co, 1))
    sync()
    assert np.array_equal(out.cpu().numpy().transpose(0, 3, 1, 2).reshape(tgt.shape), tgt)


def scaled_case(geom, seed):
    """signed data: every image, pixel and channel of x and every output channel of the filters at its own power of two"""
    ishape, kshape, padding, strides = GEOMS[geom]
    n, C, H, W = ishape
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, H, W, C)) * 2.0 ** rng.integers(-6, 7, n)[:, None, None, None] * \
        2.0 ** rng.integers(-6, 7, (1, H, W, 1)) * 2.0 ** rng.integers(-6, 7, C)[None, None, None, :]
    K, co = kshape[2] * kshape[3] * C, kshape[0]
    w = rng.uniform(-1, 1, (K, co)) * 2.0 ** rng.integers(-6, 7, co)[None, :]
    return Conv(ishape, kshape, padding, strides, x=x.astype(np.float32), wmat=w.astype(np.float32))


@pytest.mark.parametrize("layout", ["hwio", "ohwi"])
@pytest.mark.parametrize("geom", ["pad1", "rgb_c3", "c5_cout_odd"])
@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_tensor_core_paths_within_the_bound(path, geom, layout):
    """the NHWC result within the per-element bound against float64, and the NCHW entry's result on the same data, transposed,
    within the same bound (the two sum K in different orders: not compared bit for bit)"""
    c = scaled_case(geom, 11)
    got, _ = c.fused(PATHS[path], layout)
    n = c.ishape[0]
    A, B = c.rows(), c.wmat
    if not EMU:
        torch = pytest.importorskip("torch")
        co, C, kH, kW = c.kshape
        ref = torch.nn.functional.conv2d(torch.from_numpy(c.x.astype(np.float64)).permute(0, 3, 1, 2),
                                         torch.from_numpy(B.astype(np.float64).reshape(kH, kW, C, co)).permute(3, 2, 0, 1),
                                         stride=c.strides, padding=c.padding).permute(0, 2, 3, 1).reshape(-1, co).numpy()
        np.testing.assert_allclose(A.astype(np.float64) @ B.astype(np.float64), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    bound_and_check("conv nhwc", path, "conv_nhwc", got, A, B, 1.0, splits=plan(path, n * c.P, c.co, c.K)[0])
    theirs = c.nchw(PATHS[path])
    bound_and_check("conv nchw on the same data", path, "conv_nhwc", np.ascontiguousarray(theirs),
                    np.ascontiguousarray(A.reshape(n, c.P, c.K)), np.broadcast_to(B, (n, c.K, c.co)), 1.0,
                    splits=plan(path, c.co, c.P, c.K, batch=n)[0])


@pytest.mark.parametrize("path", list(PATHS))
def test_one_by_one_reads_the_images_in_place(path):
    """1 x 1, unit strides, no padding: the fused product over the images as [n * h * w][c] -- same bits, same launches (no
    window pass)"""
    ishape, kshape = ((2, 8, 6, 6), (12, 8, 1, 1)) if EMU else ((4, 64, 14, 14), (128, 64, 1, 1))
    c = Conv(ishape, kshape, (0, 0), (1, 1), seed=17)
    got, n_fused = c.fused(PATHS[path], "hwio", True, "relu")
    resolved = L.last_path()
    out = c.out0()
    sync()
    n0 = L.launch_count()
    G.gemm_strided_fused(ishape[0] * c.P, c.co, c.K, 1.0, c.tx, c.K, 1, c.views["hwio"][0], c.co, 1, 0.0, out, c.co, 1,
                         bias=c.tb, bias_per_row=False, activation="relu", path=resolved)
    sync()
    assert n_fused == L.launch_count() - n0
    assert_bits(got, out.cpu().numpy())


@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1", "simt"])
def test_launch_count_does_not_grow_with_the_images(path):
    ishape, kshape, padding, strides = GEOMS["pad1"]
    counts = []
    for imgs in (1, 3 if EMU else 16):
        c = Conv((imgs,) + ishape[1:], kshape, padding, strides)
        _, n = c.fused(PATHS[path])
        ks = plan(path, imgs * c.P, c.co, c.K)[0] if path != "simt" else 1
        counts.append(n - (1 if ks > 1 else 0))   # (a split adds the reduce kernel)
    assert counts[0] == counts[1] <= 4, counts


# the small workspace cap runs in processes of its own: LASER_B200_BATCH_WS_MB and LASER_B200_SPLITK are read once per process
_CHUNKS = """
import hashlib, sys, test_gpu_conv_nhwc as T, laser_b200 as L
c = T.Conv((3, 64, 16, 16), (16, 64, 3, 3), (1, 1), (1, 1), seed=23)
out, n = c.fused(int(sys.argv[1]), "ohwi", True, "tanh")
print("RESULT", n, hashlib.sha256(out.tobytes()).hexdigest())
"""


def _subprocess(code, *args, env=None):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), **(env or {}))
    out = subprocess.run([sys.executable, "-c", code] + list(args), cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout.splitlines()


@pytest.mark.parametrize("path", ["f16x3", "tf32x1", "simt"])
def test_chunks_give_the_bits_of_one_chunk(path):
    """LASER_B200_BATCH_WS_MB=1 holds one image per chunk (K = 576, P = 256): three chunks, each the launches of the one-chunk
    call (split-K off), the same output"""
    one = [line for line in _subprocess(_CHUNKS, str(PATHS[path]), env={"LASER_B200_SPLITK": "0"})
           if line.startswith("RESULT")][0].split()
    many = [line for line in _subprocess(_CHUNKS, str(PATHS[path]), env={"LASER_B200_SPLITK": "0", "LASER_B200_BATCH_WS_MB": "1"})
            if line.startswith("RESULT")][0].split()
    assert int(many[1]) == 3 * int(one[1]), (one, many)
    assert many[2] == one[2]


def _raw(ishape=(2, 4, 5, 5), kshape=(3, 4, 3, 3), padding=(1, 1), strides=(1, 1), kstrides=(3, 1), bias=False, per_row=1,
         act=0, path=L.PATH_AUTO, null=None):
    out = dev(np.full(2 * 25 * 3, 3.0, np.float32))
    x, w, b = dev(np.ones(2 * 25 * 4, np.float32)), dev(np.ones(36 * 3, np.float32)), dev(np.ones(3, np.float32))
    ptrs = {"out": out.data_ptr(), "x": x.data_ptr(), "w": w.data_ptr()}
    if null:
        ptrs[null] = None
    epi = _capi.Epilogue(bias=b.data_ptr() if bias else None, bias_per_row=per_row, activation=act)
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    fn = _capi.lib().laser_b200_conv2d_nhwc_f32_fused_dev
    if kstrides is None:   # a NULL kernelStrides: the same symbol through a handle whose argtypes take a plain pointer there
        fn = ctypes.CDLL(_capi.lib()._name).laser_b200_conv2d_nhwc_f32_fused_dev
        fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, i4, ctypes.c_void_p, i4, ctypes.c_void_p, i2, i2, ctypes.POINTER(_capi.Epilogue),
                       ctypes.c_int, ctypes.c_void_p]
    rc = fn(ptrs["out"], ptrs["x"], i4(*ishape), ptrs["w"], i4(*kshape), i2(*kstrides) if kstrides else None, i2(*padding),
            i2(*strides), ctypes.byref(epi), path, G._current_stream())
    sync()
    assert np.all(out.cpu().numpy() == 3.0)
    return rc, L.launch_count() - n0


def test_argument_errors_launch_nothing():
    for kw in (dict(path=5), dict(path=-1), dict(act=4), dict(bias=True, per_row=0), dict(kstrides=None), dict(kshape=(3, 2, 3, 3)),
               dict(strides=(0, 1)), dict(padding=(-1, 0)), dict(kshape=(3, 4, 8, 3)), dict(null="out"), dict(null="x"),
               dict(null="w")):
        assert _raw(**kw) == (_capi.E_INVAL, 0), kw
    assert _raw(ishape=(0, 4, 5, 5)) == (_capi.E_OK, 0)
    assert _raw(ishape=(0, 4, 5, 5), null="out") == (_capi.E_OK, 0)
    # n * outH * outW = 2^20 * 4096 past int32 on a tensor-core path (nothing is read: the check comes first)
    assert _raw(ishape=(2 ** 20, 4, 64, 64), path=L.PATH_F16X3) == (_capi.E_UNSUPPORTED, 0)


def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode of this file's bound checks (the last test of the file)"""
    from test_gpu_error_bounds import RATIOS
    mine = {k: r for k, r in RATIOS.items() if k[1] == "conv_nhwc"}
    if not mine:
        pytest.skip("no case ran")
    with capsys.disabled():
        print("\nlargest err / bound of the NHWC convolution:\n" + "\n".join("  %-7s %.3g" % (m, r) for (m, _), r in sorted(mine.items())))
