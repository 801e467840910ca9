"""Host-side mirror of the reference's operator for the hot path.

    gemm_strided(M, N, K, alpha, A, rowStrideA, colStrideA, B, rowStrideB, colStrideB,
                 beta, C, rowStrideC, colStrideC)

has the reference's name, argument order and meaning
(laser/primitives/matrix_multiplication/gemm.nim:184-193).  A, B, C are "pointers":
  * numpy arrays          -> HOST pointers (address of element [0]); the call goes through
                             the drop-in C entry laser_b200_gemm_strided_<T>, which stages
                             H2D, runs on the GPU, copies C back and returns synchronously;
  * torch CUDA tensors, laser_b200.Tensor, or DevPtr(int, dtype)
                          -> DEVICE pointers; the call goes through ..._dev, asynchronous
                             on the given (default: torch current) stream.
All arithmetic happens in liblaser_b200.so (CUDA).  Nothing here computes.
"""
import ctypes

import numpy as np

from . import _capi
from ._capi import (PATH_AUTO, PATH_BF16, PATH_F16X3, PATH_SIMT, PATH_TF32X1, PATH_TF32X3,
                    LaserB200Error, check, lib)

__all__ = ["gemm_strided", "gemm_strided_fused", "gemm_strided_batched_fused", "DevPtr", "last_path", "launch_count", "set_f32_mode", "get_f32_mode",
           "fill_uniform_f32", "init", "shutdown", "synchronize", "profile_begin", "profile_end"]

_NP_DTYPES = {np.dtype(np.float32): "f32", np.dtype(np.float64): "f64", np.dtype(np.int32): "i32",
              np.dtype(np.int64): "i64", np.dtype(np.uint16): "bf16"}


class DevPtr:
    """A raw device address plus element type ('f32', 'f64', 'i32', 'i64', 'bf16')."""

    def __init__(self, ptr, dtype):
        self.ptr = int(ptr)
        self.dtype = dtype


_torch = None          # the torch module, once a torch tensor has been seen
_TORCH_DTYPES = None   # torch dtype -> element-type name (built once: this sits on the call path)


def _torch_dtype_name(t):
    global _torch, _TORCH_DTYPES
    if _TORCH_DTYPES is None:
        import torch
        _torch = torch
        _TORCH_DTYPES = {torch.float32: "f32", torch.float64: "f64", torch.int32: "i32", torch.int64: "i64",
                         torch.bfloat16: "bf16"}
    return _TORCH_DTYPES.get(t.dtype)


_Tensor = None


def _resolve(x):
    """-> (address, dtype name, is_device)"""
    global _Tensor
    if _Tensor is None:
        from .tensor import Tensor as _T
        _Tensor = _T
    Tensor = _Tensor
    if isinstance(x, np.ndarray):
        name = _NP_DTYPES.get(x.dtype)
        if name is None:
            raise TypeError("unsupported numpy dtype %s" % x.dtype)
        return x.ctypes.data, name, False
    if isinstance(x, DevPtr):
        return x.ptr, x.dtype, True
    if isinstance(x, Tensor):
        return x.unsafe_raw_data(), x.dtype, True
    if type(x).__module__.startswith("torch"):
        name = _torch_dtype_name(x)
        if name is None:
            raise TypeError("unsupported torch dtype %s" % x.dtype)
        if not x.is_cuda:
            raise TypeError("torch CPU tensors are not accepted: pass t.numpy() for the host-pointer "
                            "entry or a CUDA tensor for the device entry")
        return x.data_ptr(), name, True
    raise TypeError("A, B, C must be numpy arrays (host), torch CUDA tensors, laser_b200.Tensor or DevPtr")


def _current_stream():
    """torch's current CUDA stream if torch is in use in this process, else 0 (library stream)."""
    global _torch
    if _torch is None:
        import sys
        _torch = sys.modules.get("torch")
        if _torch is None:
            return 0
    try:
        h = int(_torch.cuda.current_stream().cuda_stream)
    except Exception:  # no CUDA in this torch build / no device: the library reports the error
        return 0
    # torch reports its default stream as handle 0, which the C ABI reserves for "the library's
    # own stream, synchronous".  The legacy default stream has the explicit handle
    # cudaStreamLegacy == (cudaStream_t)0x1: work is then ordered with everything torch queued.
    return h if h != 0 else 1


def _scalar(name, v):
    if name in ("f32", "bf16"):
        return ctypes.c_float(float(v))
    if name == "f64":
        return ctypes.c_double(float(v))
    if name == "i32":
        return ctypes.c_int32(int(v))
    return ctypes.c_int64(int(v))


def gemm_strided(M, N, K, alpha, A, rowStrideA, colStrideA, B, rowStrideB, colStrideB, beta, C,
                 rowStrideC, colStrideC, path=PATH_AUTO, stream=None):
    """C <- alpha * A(MxK) * B(KxN) + beta * C; strides in elements (see module docstring)."""
    pa, ta, da = _resolve(A)
    pb, tb, db = _resolve(B)
    pc, tc, dc = _resolve(C)
    if not (ta == tb == tc):
        raise TypeError("A, B, C element types differ: %s, %s, %s" % (ta, tb, tc))
    if not (da == db == dc):
        raise TypeError("A, B, C must all be host pointers or all be device pointers")
    L = lib()
    args = [M, N, K, _scalar(ta, alpha), pa, rowStrideA, colStrideA, pb, rowStrideB, colStrideB,
            _scalar(ta, beta), pc, rowStrideC, colStrideC]
    if not da:
        if path != PATH_AUTO:
            raise ValueError("the host-pointer entry has the reference's exact signature (no path "
                             "argument); use set_f32_mode() or device pointers")
        check(getattr(L, "laser_b200_gemm_strided_" + ta)(*args))
        return
    if stream is None:
        stream = _current_stream()
    if ta == "f32":
        check(L.laser_b200_gemm_strided_f32_dev(*args, path, stream))
    else:
        if path not in (PATH_AUTO, PATH_SIMT if ta != "bf16" else PATH_BF16):
            raise ValueError("path %d is not available for %s" % (path, ta))
        check(getattr(L, "laser_b200_gemm_strided_%s_dev" % ta)(*args, stream))


def _operand_op(spec, batched=False):
    """op_a / op_b of gemm_strided_fused -> (an OperandOp or None, aux batch stride).  batched: the aux tensor also takes its
    batch stride, (name, aux, auxRowStride, auxColStride, auxBatchStride)."""
    if spec is None:
        return None, 0
    if isinstance(spec, str):
        spec = (spec,)
    name, rest = spec[0], tuple(spec[1:])
    op = _capi.OperandOp()
    op.op = _capi.OP_NAMES[name]
    aux_bs = 0
    if rest:
        if len(rest) != (4 if batched else 3):
            raise ValueError("an operand op is a name or (name, aux, auxRowStride, auxColStride%s)" %
                             (", auxBatchStride" if batched else ""))
        paux, taux, daux = _resolve(rest[0])
        if not daux or taux != "f32":
            raise TypeError("aux must be a float32 device buffer")
        op.aux = paux
        op.auxRowStride, op.auxColStride = int(rest[1]), int(rest[2])
        if batched:
            aux_bs = int(rest[3])
    return op, aux_bs


def gemm_strided_fused(M, N, K, alpha, A, rowStrideA, colStrideA, B, rowStrideB, colStrideB, beta, C,
                       rowStrideC, colStrideC, bias=None, bias_per_row=False, activation="none",
                       path=PATH_AUTO, stream=None, *, op_a=None, op_b=None):
    """C <- act(alpha*opA(A)*opB(B) + beta*C + bias) on float32 DEVICE buffers: the epilogue fusion the
    reference lists as its next step (gemm.nim:196).  activation: none | relu | tanh | sigmoid.
    op_a / op_b (the prologue fusion): an elementwise op applied to the operand while it is prepared --
    "relu", "tanh", "sigmoid", or a derivative with its aux tensor and that tensor's element strides,
    e.g. op_a=("relu_grad", Z, rowStrideZ, colStrideZ) for dY * relu'(Z); also "tanh_grad" (aux: the
    tanh output) and "sigmoid_grad" (aux: the sigmoid output)."""
    pa, pb, pc, epi = _fused_args("gemm_strided_fused", A, B, C, bias, bias_per_row, activation)
    (oa, _), (ob, _) = _operand_op(op_a), _operand_op(op_b)
    if stream is None:
        stream = _current_stream()
    if oa is None and ob is None:
        check(lib().laser_b200_gemm_strided_f32_epi_dev(M, N, K, float(alpha), pa, rowStrideA, colStrideA, pb, rowStrideB,
                                                        colStrideB, float(beta), pc, rowStrideC, colStrideC,
                                                        ctypes.byref(epi), path, stream))
        return
    check(lib().laser_b200_gemm_strided_f32_fused_dev(M, N, K, float(alpha), pa, rowStrideA, colStrideA, pb, rowStrideB,
                                                      colStrideB, float(beta), pc, rowStrideC, colStrideC,
                                                      ctypes.byref(oa) if oa is not None else None,
                                                      ctypes.byref(ob) if ob is not None else None,
                                                      ctypes.byref(epi), path, stream))


def _fused_args(fn, A, B, C, bias, bias_per_row, activation):
    """-> (A, B, C addresses, Epilogue) of a fused entry"""
    pa, ta, da = _resolve(A); pb, tb, db = _resolve(B); pc, tc, dc = _resolve(C)
    if not (ta == tb == tc == "f32") or not (da and db and dc):
        raise TypeError("%s takes float32 device buffers" % fn)
    epi = _capi.Epilogue()
    if bias is not None:
        pbias, tbias, dbias = _resolve(bias)
        if not dbias or tbias != "f32":
            raise TypeError("bias must be a float32 device vector")
        epi.bias = pbias
    epi.bias_per_row = 1 if bias_per_row else 0
    epi.activation = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}[activation]
    return pa, pb, pc, epi


def gemm_strided_batched_fused(batch, M, N, K, alpha, A, rowStrideA, colStrideA, batchStrideA, B, rowStrideB, colStrideB,
                               batchStrideB, beta, C, rowStrideC, colStrideC, batchStrideC, bias=None, bias_per_row=False,
                               activation="none", path=PATH_AUTO, stream=None, *, op_a=None, op_b=None):
    """gemm_strided_fused over a batch on float32 DEVICE buffers: problem b reads A + b * batchStrideA, B + b * batchStrideB
    and writes C + b * batchStrideC (a batch stride of 0 shares A or B; the bias is shared).  Every problem's operands are
    prepared together and one GEMM launch runs the tiles of all of them.  op_a / op_b as in gemm_strided_fused, with the aux
    tensor's batch stride last: e.g. op_a=("relu_grad", Z, rowStrideZ, colStrideZ, batchStrideZ)."""
    pa, pb, pc, epi = _fused_args("gemm_strided_batched_fused", A, B, C, bias, bias_per_row, activation)
    (oa, aux_a), (ob, aux_b) = _operand_op(op_a, batched=True), _operand_op(op_b, batched=True)
    strides = _capi.BatchStrides(int(batchStrideA), int(batchStrideB), int(batchStrideC), aux_a, aux_b)
    if stream is None:
        stream = _current_stream()
    check(lib().laser_b200_gemm_strided_batched_f32_fused_dev(
        int(batch), M, N, K, float(alpha), pa, rowStrideA, colStrideA, pb, rowStrideB, colStrideB, float(beta), pc, rowStrideC,
        colStrideC, ctypes.byref(strides), ctypes.byref(oa) if oa is not None else None,
        ctypes.byref(ob) if ob is not None else None, ctypes.byref(epi), path, stream))


def gemm_strided_batch_reduce_fused(batch, M, N, K, alpha, A, rowStrideA, colStrideA, batchStrideA, B, rowStrideB, colStrideB,
                                    batchStrideB, beta, C, rowStrideC, colStrideC, bias=None, bias_per_row=False,
                                    activation="none", path=PATH_AUTO, stream=None, *, op_a=None, op_b=None):
    """C <- act(alpha * sum_b opA(A_b) * opB(B_b) + beta*C + bias) on float32 DEVICE buffers (torch.addbmm): the sum of a
    batch's products into one C, computed as one fused product over the operands concatenated along K.  A_b = A +
    b * batchStrideA, B_b = B + b * batchStrideB; op_a / op_b as in gemm_strided_batched_fused, with the aux tensor's batch
    stride last."""
    pa, pb, pc, epi = _fused_args("gemm_strided_batch_reduce_fused", A, B, C, bias, bias_per_row, activation)
    (oa, aux_a), (ob, aux_b) = _operand_op(op_a, batched=True), _operand_op(op_b, batched=True)
    strides = _capi.BatchStrides(int(batchStrideA), int(batchStrideB), 0, aux_a, aux_b)
    if stream is None:
        stream = _current_stream()
    check(lib().laser_b200_gemm_strided_batch_reduce_f32_fused_dev(
        int(batch), M, N, K, float(alpha), pa, rowStrideA, colStrideA, pb, rowStrideB, colStrideB, float(beta), pc, rowStrideC,
        colStrideC, ctypes.byref(strides), ctypes.byref(oa) if oa is not None else None,
        ctypes.byref(ob) if ob is not None else None, ctypes.byref(epi), path, stream))


def last_path():
    return lib().laser_b200_last_path()


def launch_count():
    return int(lib().laser_b200_launch_count())


def set_f32_mode(path):
    check(lib().laser_b200_set_f32_mode(path))


def get_f32_mode():
    return lib().laser_b200_get_f32_mode()


def profile_begin():
    check(lib().laser_b200_profile_begin())


def profile_end():
    """-> dict(gemm_ms, gemm_launches, prep_ms, prep_launches): device time of the library's
    own kernels since profile_begin(), from CUDA events on the launching stream."""
    g, p = ctypes.c_double(), ctypes.c_double()
    ng, npr = ctypes.c_int64(), ctypes.c_int64()
    check(lib().laser_b200_profile_end(ctypes.byref(g), ctypes.byref(ng), ctypes.byref(p), ctypes.byref(npr)))
    return dict(gemm_ms=g.value, gemm_launches=ng.value, prep_ms=p.value, prep_launches=npr.value)


def init():
    check(lib().laser_b200_init())


def shutdown():
    lib().laser_b200_shutdown()


def synchronize():
    check(lib().laser_b200_synchronize())


def fill_uniform_f32(dst, n, seed, lo, hi, stream=None):
    """Counter-based U[lo,hi) fill of a device buffer (bit-identical to the CPU oracle's)."""
    p, t, d = _resolve(dst)
    if not d or t != "f32":
        raise TypeError("fill_uniform_f32 needs a float32 device buffer")
    if stream is None:
        stream = _current_stream()
    check(lib().laser_b200_fill_uniform_f32_dev(p, int(n), int(seed), float(lo), float(hi), stream))
