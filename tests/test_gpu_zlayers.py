"""GPU: the steps either side of the GEMM (SURVEY.md 8f rank 4) through the C ABI against the
oracle: transposes / NCHW<->NHWC (swapaxes.nim:16-112), im2col convolution
(conv2d_im2col.nim:44-166, the reference's conv known-answer vectors conv2d_common.nim:128-283),
batched GEMM, copyFrom and forEach on strided views (initialization.nim:80-112, foreach.nim:229-251).

Besides this file, the kernels are checked as far as a machine without a GPU allows: the kernel source runs on CPU threads against the
oracle (tests/test_emulated_kernels.py), the host side of the entry points too
(tests/test_emulated_layers_host.py), and this very file runs on the CPU against a stand-in library
(LASER_B200_EMU=1, tests/test_emulated_python_mirror.py), which checks the Python mirror and the
expectations below."""
import json
import os

import numpy as np
import pytest

import oracle as O

EMU = os.environ.get("LASER_B200_EMU", "0") == "1"       # CPU stand-in library: "device" memory is host memory
pytestmark = pytest.mark.gpu
if not EMU:
    torch = pytest.importorskip("torch")
import laser_b200 as L  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
NP_OF = {2: np.int16, 4: np.float32, 8: np.float64}   # int16: torch has no full uint16 support
NAME_OF = {np.dtype(np.int16): "bf16", np.dtype(np.uint16): "bf16", np.dtype(np.float32): "f32", np.dtype(np.float64): "f64",
           np.dtype(np.int32): "i32", np.dtype(np.int64): "i64"}


class HostDev(L.DevPtr):  # (same idea as backend.HostTensor)
    """EMU backend: a numpy array posing as device memory."""

    def __init__(self, arr):
        self.arr = np.ascontiguousarray(arr)
        super().__init__(self.arr.ctypes.data, NAME_OF[self.arr.dtype])


def dev(a):
    """host array -> device array"""
    a = np.ascontiguousarray(a)
    return HostDev(a.copy()) if EMU else torch.from_numpy(a).cuda()


def full(shape, value, dt=np.float32):
    return dev(np.full(shape, value, dt))


def to_np(t):
    if EMU:
        return t.arr
    torch.cuda.synchronize()
    return t.cpu().numpy()


def addr(t):
    return t.ptr if EMU else t.data_ptr()


def raw(t, esz):
    """DevPtr of the right element width for byte-level transposes."""
    return L.DevPtr(addr(t), {2: "bf16", 4: "f32", 8: "f64"}[esz])


def cpu_budget(elements):
    if EMU and elements > 400_000:
        pytest.skip("too large for the CPU stand-in")


def conv_ref(inp, ishape, ker, kshape, padding, strides):
    """Oracle convolution.  For 1x1 kernels with a stride or padding the reference's im2col shortcut
    (conv2d_im2col.nim:121,145-149) reads the image in place and is wrong; the product deliberately
    goes through im2col there (include/laser_b200.h), so the expectation is im2col + the GEMM oracle."""
    if kshape[2] * kshape[3] != 1 or (tuple(strides) == (1, 1) and tuple(padding) == (0, 0)):
        return O.conv2d_im2col(inp, ishape, ker, kshape, padding, strides)
    o = O.conv2d_out_shape(ishape, kshape, padding, strides)
    M, K, N = kshape[0], ishape[1], o[2] * o[3]
    out = np.zeros((ishape[0], M, N), np.float32)
    kmat = np.ascontiguousarray(ker, np.float32).reshape(M, K)
    for n in range(ishape[0]):
        ws = np.ascontiguousarray(O.im2col(np.ascontiguousarray(inp[n]), ishape, kshape, padding, strides))
        O.gemm_strided(M, N, K, 1.0, kmat, K, 1, ws, N, 1, 0.0, out[n], N, 1)
    return out.reshape(o)


# ---- transposes ------------------------------------------------------------------------------
@pytest.mark.parametrize("esz", [2, 4, 8])
@pytest.mark.parametrize("N,NR,NC", [(1, 1, 1), (1, 64, 64), (1, 4000, 2000), (3, 33, 70), (2, 68, 132),
                                     (1, 5, 4099), (16, 3, 224 * 224), (1, 8192, 8192)])
def test_transpose_dev(esz, N, NR, NC):
    cpu_budget(N * NR * NC)
    dt = NP_OF[esz]
    src = (np.arange(N * NR * NC, dtype=np.int64) * 2654435761 % 65521).astype(dt)
    tsrc = dev(src); tdst = full(src.shape, 0, dt)
    L.transpose2D_batched(raw(tdst, esz), raw(tsrc, esz), N, NR, NC)
    assert np.array_equal(to_np(tdst).reshape(N, NC, NR), src.reshape(N, NR, NC).transpose(0, 2, 1))


def test_transpose_matches_oracle_and_round_trips():
    NR, NC = (400, 200) if EMU else (4000, 2000)   # the reference transpose bench shape (transpose_bench.nim:54-55)
    src = O.fill_uniform_f32(NR * NC, 7, 0, 1)
    tsrc = dev(src); t1 = full(src.shape, 0); t2 = full(src.shape, 0)
    L.transpose2D_copy(t1, tsrc, NR, NC)
    L.transpose2D_copy(t2, t1, NC, NR)
    assert np.array_equal(to_np(t1).reshape(NC, NR), O.transpose2D_copy(src, NR, NC))
    assert np.array_equal(to_np(t2), src)


def test_misaligned_pointers_take_the_scalar_kernel():
    NR, NC = 128, 256
    buf = dev(np.arange(NR * NC + 1, dtype=np.float32))
    out = full((NR * NC + 1,), 0)
    L.transpose2D_copy(L.DevPtr(addr(out) + 4, "f32"), L.DevPtr(addr(buf) + 4, "f32"), NR, NC)
    assert np.array_equal(to_np(out)[1:].reshape(NC, NR), to_np(buf)[1:].reshape(NR, NC).T)
    assert to_np(out)[0] == 0.0


def test_nchw_nhwc_device_and_host():
    N, C, H, W = 4, 3, 17, 20
    x = O.fill_uniform_f32(N * C * H * W, 3, -1, 1).reshape(N, C, H, W)
    tx = dev(x); ty = full((N * H * W * C,), 0); tz = full(x.shape, 0)
    L.nchw2nhwc(ty, tx, N, C, H, W)
    L.nhwc2nchw(tz, ty, N, C, H, W)
    assert np.array_equal(to_np(ty).reshape(N, H, W, C), x.transpose(0, 2, 3, 1))
    assert np.array_equal(to_np(tz), x)
    hy = np.empty(N * H * W * C, np.float32)
    L.nchw2nhwc(hy, x.reshape(-1).copy(), N, C, H, W)          # host-pointer entry, synchronous
    assert np.array_equal(hy.reshape(N, H, W, C), x.transpose(0, 2, 3, 1))


def test_transpose_rejects_bad_arguments():
    a = full((16,), 0)
    with pytest.raises(L.LaserB200Error):
        L.transpose2D_copy(a, a, 4, 4)                          # aliasing
    with pytest.raises(L.LaserB200Error):
        L.transpose2D_copy(a, full((16,), 0), -1, 4)


# ---- convolution ------------------------------------------------------------------------------
def conv_cases():
    with open(os.path.join(HERE, "golden", "conv2d_known_answer.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", conv_cases(), ids=lambda c: c["src"])
def test_conv2d_known_answer(case):
    inp = np.array(case["input"], np.float32); ker = np.array(case["kernel"], np.float32)
    tgt = np.array(case["target"], np.float32)
    ish, ksh, pad, st = case["ishape"], case["kshape"], case["padding"], case["strides"]
    assert L.conv2d_out_shape(ish, ksh, pad, st) == tgt.shape
    out = np.full(tgt.shape, 99.0, np.float32)
    L.conv2d_im2col(out, inp, ish, ker, ksh, pad, st)           # host entry
    assert np.array_equal(out, tgt)
    tout = full(tgt.shape, 99.0)
    ws = full((L.im2col_workspace_size(ish, ksh, pad, st),), 0)
    L.conv2d_im2col(tout, dev(inp), ish, dev(ker), ksh, pad, st, workspace=ws)
    assert np.array_equal(to_np(tout), tgt)


IM2COL_CASES = [
    ((2, 3, 9, 11), (4, 3, 3, 3), (0, 0), (1, 1)),
    ((3, 2, 8, 8), (5, 2, 3, 3), (1, 1), (2, 2)),
    ((2, 1, 12, 6), (2, 1, 5, 2), (2, 1), (3, 3)),
    ((1, 2, 40, 36), (1, 2, 3, 3), (1, 1), (1, 1)),
    ((4, 16, 28, 28), (32, 16, 3, 3), (1, 1), (1, 1)),
    ((2, 3, 224, 224), (20, 3, 3, 3), (0, 0), (1, 1)),          # the reference conv bench geometry, 2 of 16 images
]


@pytest.mark.parametrize("ishape,kshape,padding,strides", IM2COL_CASES)
def test_im2col_matches_oracle(ishape, kshape, padding, strides):
    B = ishape[0]
    per = L.im2col_workspace_size(ishape, kshape, padding, strides)
    cpu_budget(B * per)
    inp = O.fill_uniform_f32(int(np.prod(ishape)), 21, 1, 2).reshape(ishape)
    assert per == O.im2col_workspace_size(ishape, kshape, padding, strides)
    ws = full((B * per + 8,), -5.0)
    L.im2col(ws, dev(inp), ishape, kshape, padding, strides, images=B)
    got = to_np(ws)
    for b in range(B):
        assert np.array_equal(got[b * per:(b + 1) * per], O.im2col(inp[b], ishape, kshape, padding, strides).reshape(-1))
    assert np.all(got[B * per:] == -5.0)


@pytest.mark.parametrize("ishape,kshape,padding,strides,ws_images", [
    ((2, 3, 9, 11), (4, 3, 3, 3), (0, 0), (1, 1), 1),
    ((5, 2, 8, 8), (5, 2, 3, 3), (1, 1), (2, 2), 2),            # batch not a multiple of the workspace
    ((3, 4, 7, 10), (3, 4, 1, 1), (0, 0), (1, 1), 1),           # 1x1: no im2col
    ((2, 4, 9, 9), (3, 4, 1, 1), (1, 1), (2, 2), 2),            # strided/padded 1x1 goes through im2col
    ((4, 16, 28, 28), (32, 16, 3, 3), (1, 1), (1, 1), 4),
    ((2, 3, 224, 224), (20, 3, 3, 3), (0, 0), (1, 1), 2),
])
def test_conv2d_matches_oracle(ishape, kshape, padding, strides, ws_images):
    per = L.im2col_workspace_size(ishape, kshape, padding, strides)
    cpu_budget(ishape[0] * per)
    inp = O.fill_uniform_f32(int(np.prod(ishape)), 31, 0, 1).reshape(ishape)
    ker = O.fill_uniform_f32(int(np.prod(kshape)), 32, 0, 1).reshape(kshape)
    ref = conv_ref(inp, ishape, ker, kshape, padding, strides)
    oshape = L.conv2d_out_shape(ishape, kshape, padding, strides)
    tout = full(oshape, np.nan)                                 # beta = 0: NaN must not survive
    ws = full((max(1, ws_images * per),), 0)
    L.conv2d_im2col(tout, dev(inp), ishape, dev(ker), kshape, padding, strides, workspace=ws, workspace_images=ws_images)
    got = to_np(tout)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4   # BASELINE gate for fp32 (positive data)
    exact = full(oshape, 0)
    L.conv2d_im2col(exact, dev(inp), ishape, dev(ker), kshape, padding, strides, workspace=ws,
                    workspace_images=ws_images, path=L.PATH_SIMT)
    assert np.array_equal(to_np(exact), ref)                    # exact kernel: bit-identical to the CPU order
    hout = np.empty(oshape, np.float32)
    L.conv2d_im2col(hout, inp, ishape, ker, kshape, padding, strides)
    assert np.abs(hout - ref).max() / np.abs(ref).max() < 1e-4


def test_conv2d_rejects_bad_shapes():
    x = full((16,), 0)
    with pytest.raises(L.LaserB200Error):
        L.conv2d_out_shape((1, 1, 4, 4), (1, 1, 3, 3), (0, 0), (4, 1))
    with pytest.raises(L.LaserB200Error):   # c_in mismatch (conv2d_direct_convolution.nim:20)
        L.conv2d_im2col(x, x, (1, 1, 4, 4), x, (1, 2, 3, 3), (1, 1), (1, 1), workspace=x)


# ---- batched GEMM -----------------------------------------------------------------------------
@pytest.mark.parametrize("path", [L.PATH_AUTO, L.PATH_SIMT])
def test_batched_gemm(path):
    batch, M, N, K = 5, 70, 200, 150
    A = O.fill_uniform_f32(batch * M * K, 41, 0, 1); B = O.fill_uniform_f32(K * N, 42, 0, 1)
    C0 = O.fill_uniform_f32(batch * M * N, 43, 0, 1)
    ref = C0.copy()
    O.gemm_strided_batched(batch, M, N, K, 0.5, A, K, 1, M * K, B, N, 1, 0, -1.25, ref, N, 1, M * N)
    tC = dev(C0)
    L.gemm_strided_batched(batch, M, N, K, 0.5, dev(A), K, 1, M * K, dev(B), N, 1, 0, -1.25, tC, N, 1, M * N, path=path)
    got = to_np(tC)
    if path == L.PATH_SIMT:
        assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()   # alpha != 1: contraction may differ by 1 ulp
    else:
        assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4


def test_batched_small_problems_single_launch_is_bit_exact():
    batch, M, N, K = 64, 32, 48, 40          # below the 128^3 threshold: exact kernel, one launch
    A = O.fill_uniform_f32(batch * M * K, 51, -1, 1); B = O.fill_uniform_f32(batch * K * N, 52, -1, 1)
    ref = np.zeros(batch * M * N, np.float32)
    O.gemm_strided_batched(batch, M, N, K, 1.0, A, K, 1, M * K, B, N, 1, K * N, 0.0, ref, N, 1, M * N)
    tC = full((batch * M * N,), np.nan)
    before = L.launch_count()
    L.gemm_strided_batched(batch, M, N, K, 1.0, dev(A), K, 1, M * K, dev(B), N, 1, K * N, 0.0, tC, N, 1, M * N)
    assert L.launch_count() - before == 1
    assert np.array_equal(to_np(tC), ref)


def test_batched_f64_and_i64():
    batch, M, N, K = 6, 40, 50, 300
    rng = np.random.default_rng(4)
    A = rng.random(batch * M * K); B = rng.random(batch * K * N); C0 = rng.random(batch * M * N); ref = C0.copy()
    for b in range(batch):
        O.gemm_strided(M, N, K, 1.0, A[b * M * K:], K, 1, B[b * K * N:], N, 1, 1.0, ref[b * M * N:(b + 1) * M * N], N, 1)
    tC = dev(C0)
    L.gemm_strided_batched(batch, M, N, K, 1.0, dev(A), K, 1, M * K, dev(B), N, 1, K * N, 1.0, tC, N, 1, M * N)
    assert np.array_equal(to_np(tC), ref)
    Ai = rng.integers(-2**62, 2**62, size=batch * M * K, dtype=np.int64); Bi = rng.integers(-2**62, 2**62, size=K * N, dtype=np.int64)
    refi = np.zeros(batch * M * N, np.int64)
    for b in range(batch):
        O.gemm_strided(M, N, K, 1, Ai[b * M * K:], K, 1, Bi, N, 1, 0, refi[b * M * N:(b + 1) * M * N], N, 1)
    tCi = full((batch * M * N,), 0, np.int64)
    L.gemm_strided_batched(batch, M, N, K, 1, dev(Ai), K, 1, M * K, dev(Bi), N, 1, 0, 0, tCi, N, 1, M * N)
    assert np.array_equal(to_np(tCi), refi)


# ---- copyFrom on strided views ------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["f32", "f64", "i32", "i64", "bf16"])
def test_copyFrom_views(dtype):
    npdt = {"f32": np.float32, "f64": np.float64, "i32": np.int32, "i64": np.int64, "bf16": np.uint16}[dtype]
    src_host = (np.arange(40 * 60) % 30000).astype(npdt).reshape(40, 60)
    src = L.toTensor(src_host, dtype)
    dst = L.newTensor([60, 40], dtype)
    L.copyFrom(dst, src.transpose())                              # materialise a transposed view
    assert np.array_equal(dst.to_numpy(), src_host.T)
    dst2 = L.newTensor([40, 60], dtype)
    L.copyFrom(dst2.slice2d(slice(0, 40, 2), slice(1, 60, 3)), src.slice2d(slice(1, 40, 2), slice(0, 60, 3)))
    exp = np.zeros((40, 60), npdt); exp[0:40:2, 1:60:3] = src_host[1:40:2, 0:60:3]
    assert np.array_equal(dst2.to_numpy(), exp)                   # only the exposed elements are written
    dst3 = L.newTensor([40, 60], dtype)
    L.copyFrom(dst3, src)                                         # contiguous pair: plain device copy
    assert np.array_equal(dst3.to_numpy(), src_host)
    with pytest.raises(L.LaserB200Error):
        L.copyFrom(L.newTensor([40, 61], dtype), src)             # shape mismatch (initialization.nim:96)


# ---- forEach opcodes on strided device views (foreach.nim:229-251) ---------------------------------
FOREACH = {"copy": lambda x, y, z, a: x, "fill": lambda x, y, z, a: np.full_like(x, a), "scale": lambda x, y, z, a: a * x,
           "add": lambda x, y, z, a: x + y, "sub": lambda x, y, z, a: x - y, "mul": lambda x, y, z, a: x * y,
           "fma": lambda x, y, z, a: x + y * z, "axpy": lambda x, y, z, a: a * x + y,
           "bench": lambda x, y, z, a: x + y - np.sin(z)}


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("op", sorted(FOREACH))
def test_forEach_ops(dtype, op):
    npdt = np.float32 if dtype == "f32" else np.float64
    rng = np.random.default_rng(3)
    R, Cc = (100, 1000) if EMU else (100, 10000)                           # the reference's non-contiguous bench shapes
    hx, hy, hz = (rng.standard_normal((R, Cc)).astype(npdt), rng.standard_normal((Cc, R)).astype(npdt),
                  rng.standard_normal((Cc, R)).astype(npdt))
    x, y, z = L.toTensor(hx, dtype), L.toTensor(hy, dtype).transpose(), L.toTensor(hz, dtype).transpose()
    out = L.newTensor([R, Cc], dtype)
    L.forEach(op, out, x, y, z, alpha=0.75)
    want = FOREACH[op](hx, hy.T, hz.T, npdt(0.75))
    tol = 4e-6 if dtype == "f32" else 1e-14                               # mul+add may be contracted to an FMA
    assert np.abs(out.to_numpy() - want).max() <= tol * max(1.0, np.abs(want).max())


def test_forEach_in_place_and_errors():
    hx, hy, hz = (np.arange(12, dtype=np.float32).reshape(3, 4), np.ones((3, 4), np.float32) * 2, np.ones((3, 4), np.float32) * 3)
    x, y, z = L.toTensor(hx), L.toTensor(hy), L.toTensor(hz)
    L.forEach("fma", x, x, y, z)                                          # x += y * z
    assert np.array_equal(x.to_numpy(), hx + 6)
    with pytest.raises(L.LaserB200Error):
        L.forEach("add", x, y)                                            # missing operand
    with pytest.raises(L.LaserB200Error):
        L.forEach("add", x, y, L.newTensor([4, 3]))                       # shape mismatch
    with pytest.raises(L.LaserB200Error):
        L.forEach("add", L.newTensor([3, 4], "i32"), L.newTensor([3, 4], "i32"), L.newTensor([3, 4], "i32"))
