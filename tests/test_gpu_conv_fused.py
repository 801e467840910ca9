"""GPU: the fused convolution laser_b200_conv2d_f32_fused_dev -- im2col folded into the preparation of the GEMM's B operand,
every image of a chunk in one GEMM launch, bias and activation in the epilogue.  On every path the output must equal, bit for
bit, the batched fused product over the materialised im2col matrix in the layout the preparation kernel writes; it must meet
the fp32 accuracy gates against the direct convolution; and the launch count must not grow with the number of images."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from backend import EMU, dev, emu_budget, sync

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402
from laser_b200 import _capi  # noqa: E402
from laser_b200 import gemm as G  # noqa: E402

PATHS = {"simt": L.PATH_SIMT, "f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "auto": L.PATH_AUTO}
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# M = c_out >= 64 and K >= 64: PATH_AUTO decides as the batched product does; K <= 768 keeps split-K off
GEOMS = {
    "pad1": ((2, 8, 6, 6), (64, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((3, 16, 20, 20), (96, 16, 3, 3), (1, 1), (1, 1)),
    "stride2_non_square": ((2, 12, 7, 6), (64, 12, 3, 2), (1, 0), (2, 1)) if EMU else ((2, 12, 17, 15), (80, 12, 3, 2), (1, 0), (2, 1)),
    "one_by_one_stride2": ((2, 72, 5, 5), (64, 72, 1, 1), (0, 0), (2, 2)) if EMU else ((3, 72, 15, 15), (64, 72, 1, 1), (0, 0), (2, 2)),
    "one_by_one": ((2, 72, 4, 4), (64, 72, 1, 1), (0, 0), (1, 1)) if EMU else ((3, 72, 14, 14), (64, 72, 1, 1), (0, 0), (1, 1)),
}


class Conv:
    """one convolution's data: images U(lo, hi), filters U(lo, hi), a bias per output channel (host and device copies)"""

    def __init__(self, ishape, kshape, padding, strides, seed=1, lo=-1.0, hi=1.0):
        self.ishape, self.kshape, self.padding, self.strides = ishape, kshape, padding, strides
        self.x = O.fill_uniform_f32(int(np.prod(ishape)), seed, lo, hi).reshape(ishape)
        self.k = O.fill_uniform_f32(int(np.prod(kshape)), seed + 1, lo, hi).reshape(kshape)
        self.bias = O.fill_uniform_f32(kshape[0], seed + 2, -0.5, 0.5)
        self.oshape = tuple(O.conv2d_out_shape(ishape, kshape, padding, strides))
        self.tx, self.tk, self.tb = dev(self.x), dev(self.k), dev(self.bias)

    def fused(self, path, bias=False, activation="none"):
        out = dev(np.full(self.oshape, np.nan, np.float32))
        L.conv2d_fused(out, self.tx, self.ishape, self.tk, self.kshape, self.padding, self.strides,
                       bias=self.tb if bias else None, activation=activation, path=path)
        sync()
        return out.cpu().numpy().copy()

    def unfused(self, path, bias=False, activation="none"):
        """the batched fused product, B = the im2col matrices transposed: rows [image][pixel][ld], ld = round_up(K, 4) -- or,
        for a 1 x 1 kernel with unit strides and no padding, the images themselves ([C][H*W] each)"""
        n, M = self.ishape[0], self.kshape[0]
        K, N = int(np.prod(self.kshape[1:])), self.oshape[2] * self.oshape[3]
        if self.kshape[2:] == (1, 1) and tuple(self.padding) == (0, 0) and tuple(self.strides) == (1, 1):
            B, rsB, csB, bsB = self.tx, N, 1, K * N
        else:
            ld = -(-K // 4) * 4
            rows = np.zeros((n, N, ld), np.float32)
            for b in range(n):
                rows[b, :, :K] = O.im2col(np.ascontiguousarray(self.x[b]), self.ishape, self.kshape, self.padding, self.strides).T
            B, rsB, csB, bsB = dev(rows), 1, ld, N * ld
        out = dev(np.full(self.oshape, np.nan, np.float32))
        kw = dict(bias=self.tb, bias_per_row=True) if bias else {}
        L.gemm_strided_batched_fused(n, M, N, K, 1.0, self.tk, K, 1, 0, B, rsB, csB, bsB, 0.0, out, N, 1, M * N,
                                     activation=activation, path=path, **kw)
        sync()
        return out.cpu().numpy().copy()


def assert_bits(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nanmax(np.abs(got - want))


def conv_cases():
    with open(os.path.join(HERE, "golden", "conv2d_known_answer.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("case", conv_cases(), ids=lambda c: c["src"])
def test_known_answer(case, path):
    inp = np.array(case["input"], np.float32); ker = np.array(case["kernel"], np.float32)
    tgt = np.array(case["target"], np.float32)
    out = dev(np.full(tgt.shape, 99.0, np.float32))
    L.conv2d_fused(out, dev(inp), case["ishape"], dev(ker), case["kshape"], case["padding"], case["strides"], path=PATHS[path])
    sync()
    assert np.array_equal(out.cpu().numpy(), tgt)


@pytest.mark.parametrize("epi", [(False, "none"), (True, "relu"), (True, "sigmoid")])
@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("path", list(PATHS))
def test_bit_identical_to_the_unfused_batched_product(path, geom, epi):
    c = Conv(*GEOMS[geom])
    assert_bits(c.fused(PATHS[path], *epi), c.unfused(PATHS[path], *epi))


ACC_GEOM = ((2, 8, 8, 8), (64, 8, 3, 3), (1, 1), (1, 1)) if EMU else ((4, 32, 24, 24), (64, 32, 3, 3), (1, 1), (1, 1))


@pytest.mark.parametrize("activation", ["relu", "tanh", "sigmoid"])
@pytest.mark.parametrize("path", ["f16x3", "tf32x3", "tf32x1"])
def test_accuracy_against_the_direct_convolution(path, activation):
    c = Conv(*ACC_GEOM, lo=-0.1, hi=0.1)
    got = c.fused(PATHS[path], True, activation)
    pre = O.conv2d_direct(c.x, c.ishape, c.k, c.kshape, c.padding, c.strides).astype(np.float64) + c.bias[None, :, None, None]
    ref = {"relu": lambda v: np.maximum(v, 0), "tanh": np.tanh, "sigmoid": lambda v: 1 / (1 + np.exp(-v))}[activation](pre)
    ref = ref.astype(np.float32)
    if path == "tf32x1":
        assert O.normwise_relative_error(got, ref) < 2e-3
    else:
        assert O.normwise_relative_error(got, ref) < 2e-6 and O.mean_relative_error(got, ref) <= 1e-5


def launches(c, path, bias=False):
    sync()
    n0 = L.launch_count()
    c.fused(path, bias, "relu" if bias else "none")
    return L.launch_count() - n0


@pytest.mark.parametrize("geom", ["pad1", "stride2_non_square"])
def test_launch_count_does_not_grow_with_the_images(geom):
    ishape, kshape, padding, strides = GEOMS[geom]
    one = launches(Conv((1,) + ishape[1:], kshape, padding, strides), L.PATH_F16X3)
    many = launches(Conv((4 if EMU else 16,) + ishape[1:], kshape, padding, strides), L.PATH_F16X3, bias=True)
    # the filters' row pass, the images' im2col-row pass, the GEMM: no im2col_kernel, no per-image preparation
    assert one == many == 3


@pytest.mark.skipif(EMU, reason="torch.profiler needs the GPU")
def test_no_im2col_kernel_is_launched():
    import torch
    c = Conv(*GEOMS["pad1"])
    c.fused(L.PATH_F16X3)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        c.fused(L.PATH_F16X3)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("im2col_rows_kernel" in n for n in names), names
    assert not any("im2col_kernel" in n for n in names), names


_SUB = """
import numpy as np, test_gpu_conv_fused as T, laser_b200 as L
c = T.Conv(%r, %r, (1, 1), (1, 1))
n0 = L.launch_count()
got = c.fused(L.PATH_F16X3, True, "tanh")
print("LAUNCHES", L.launch_count() - n0)
np.save(%r, got)
"""


def test_chunks_of_whole_images_are_bit_identical(tmp_path):
    """a 1 MB workspace cap holds one image at a time: one launch sequence per image, the same output as one chunk"""
    ishape, kshape = ((3, 8, 32, 32), (64, 8, 3, 3)) if EMU else ((3, 16, 32, 32), (64, 16, 3, 3))
    whole = Conv(ishape, kshape, (1, 1), (1, 1)).fused(L.PATH_F16X3, True, "tanh")
    f = str(tmp_path / "c.npy")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), LASER_B200_BATCH_WS_MB="1")
    out = subprocess.run([sys.executable, "-c", _SUB % (ishape, kshape, f)], cwd=ROOT, env=env, capture_output=True, text=True,
                         timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert int(out.stdout.split("LAUNCHES")[1].split()[0]) == 3 * 3
    assert_bits(np.load(f), whole)


def test_reference_bench_geometry_stays_on_the_exact_kernel():
    """2 of the reference bench's 16 images, 20 filters of 3 x 3 (conv2d_im2col.nim:150-166): PATH_AUTO takes the exact
    kernel and equals conv2d_im2col_f32_dev bit for bit"""
    ishape, kshape = (2, 3, 224, 224), (20, 3, 3, 3)
    emu_budget(2 * 20 * 27 * 222 * 222)
    c = Conv(ishape, kshape, (0, 0), (1, 1))
    got = c.fused(L.PATH_AUTO)
    assert L.last_path() == L.PATH_SIMT
    out = dev(np.full(c.oshape, np.nan, np.float32))
    ws = dev(np.zeros(2 * L.im2col_workspace_size(ishape, kshape, (0, 0), (1, 1)), np.float32))
    L.conv2d_im2col(out, c.tx, ishape, c.tk, kshape, (0, 0), (1, 1), workspace=ws, workspace_images=2)
    sync()
    assert_bits(got, out.cpu().numpy())


def _raw(ishape=(2, 2, 5, 5), kshape=(3, 2, 3, 3), padding=(1, 1), strides=(1, 1), epi=None, path=L.PATH_AUTO):
    out = dev(np.full(2 * 3 * 25, 3.0, np.float32))
    x, k = dev(np.ones(2 * 2 * 25, np.float32)), dev(np.ones(3 * 2 * 9, np.float32))
    i4, i2 = ctypes.c_int64 * 4, ctypes.c_int64 * 2
    sync()
    n0 = L.launch_count()
    rc = _capi.lib().laser_b200_conv2d_f32_fused_dev(out.data_ptr(), x.data_ptr(), i4(*ishape), k.data_ptr(), i4(*kshape),
                                                      i2(*padding), i2(*strides), epi, path, G._current_stream())
    sync()
    return rc, L.launch_count() - n0, out.cpu().numpy().copy()


def test_argument_errors_launch_nothing():
    for kw in (dict(path=5), dict(path=-1), dict(epi=ctypes.byref(_capi.Epilogue(None, 1, 7))), dict(kshape=(3, 1, 3, 3)),
               dict(strides=(0, 1)), dict(strides=(5, 1)), dict(kshape=(3, 2, 8, 3)), dict(padding=(-1, 0))):
        rc, n, out = _raw(**kw)
        assert (rc, n) == (_capi.E_INVAL, 0), kw
        assert np.all(out == 3.0)
    rc, n, out = _raw(ishape=(0, 2, 5, 5))
    assert (rc, n) == (_capi.E_OK, 0) and np.all(out == 3.0)
    rc, n, out = _raw(ishape=(0, 2, 5, 5), path=5)
    assert (rc, n) == (_capi.E_INVAL, 0)


@pytest.mark.parametrize("path", list(PATHS))
def test_null_epilogue_is_no_bias_no_activation(path):
    rc, n, got = _raw(path=PATHS[path])
    assert rc == _capi.E_OK and n >= 1
    rc, _, want = _raw(path=PATHS[path], epi=ctypes.byref(_capi.Epilogue(None, 1, 0)))
    assert rc == _capi.E_OK
    assert_bits(got, want)
    assert np.array_equal(got.reshape(2, 3, 5, 5), O.conv2d_direct(np.ones((2, 2, 5, 5), np.float32), (2, 2, 5, 5),
                                                                     np.ones((3, 2, 3, 3), np.float32), (3, 2, 3, 3), (1, 1), (1, 1)))
