"""Host mirror of the steps either side of the GEMM in the reference's intended use
(SURVEY.md section 8f, rank 4), on top of the C ABI:

    transpose2D_copy(dst, src, NR, NC)            laser/primitives/swapaxes.nim:16-54
    transpose2D_batched(dst, src, N, NR, NC)      swapaxes.nim:56-81
    nchw2nhwc / nhwc2nchw(dst, src, N, C, H, W)   swapaxes.nim:83-112
    conv2d_out_shape, im2col_workspace_size       benchmarks/convolution/conv2d_common.nim:15-45,
                                                  conv2d_im2col.nim:8-18
    im2col, conv2d_im2col                         conv2d_im2col.nim:44-166
    conv2d_fused                                  conv2d_im2col.nim:95-166 + bias + activation, im2col folded into the
                                                  GEMM's operand preparation (README.md:251)
    conv2d_grouped_fused                          conv2d_fused with groups > 1 (torch.nn.Conv2d(groups=G)): depthwise and
                                                  grouped layers in one call
    conv2d_filter_grad_fused                      its filter gradient, derivative op on grad_output and the window gather
                                                  folded into the operand preparation (README.md:244-245, :251)
    conv2d_nhwc_filter_grad_fused                 the filter gradient of conv2d_nhwc_fused: NHWC images and gradients, the
                                                  tap rows transposed out of the images in the operand preparation
    conv2d_input_grad_fused                       its input gradient, the transposed window gather over grad_output folded
                                                  into the operand preparation
    conv2d_grouped_input_grad_fused               the input gradient of conv2d_grouped_fused: every group in one call
    conv2d_nhwc_input_grad_fused                  the input gradient of conv2d_nhwc_fused: NHWC gradients, the transposed
                                                  windows gathered along the channels in the operand preparation
    gemm_strided_batched                          (roadmap item of the reference, README.md:253-263)
    copyFrom(dst, src)                            laser/tensor/initialization.nim:80-112

Same argument order and meaning as the reference; numpy arrays go through the host-pointer
entries (synchronous), torch CUDA tensors / laser_b200.Tensor / DevPtr through the `_dev`
entries on the current stream.  Shapes are (n, c, h, w) / (c_out, c_in, kH, kW) tuples."""
import ctypes

import numpy as np

from ._capi import OP_NAMES, PATH_AUTO, Epilogue, OperandOp, check, lib
from .gemm import _current_stream, _resolve, _scalar
from .tensor import _ITEMSIZE, Tensor

FOREACH_OPS = {"copy": 0, "fill": 1, "scale": 2, "add": 3, "sub": 4, "mul": 5, "fma": 6, "axpy": 7, "bench": 8}

__all__ = ["forEach", "FOREACH_OPS", "transpose2D_copy", "transpose2D_batched", "nchw2nhwc", "nhwc2nchw", "conv2d_out_shape",
           "im2col_workspace_size", "im2col", "conv2d_im2col", "conv2d_fused", "conv2d_grouped_fused", "conv2d_filter_grad_fused", "conv2d_input_grad_fused",
           "conv2d_grouped_input_grad_fused",
           "gemm_strided_batched", "copyFrom"]

_i64 = ctypes.c_int64


def _i4(t):
    if len(t) != 4:
        raise ValueError("expected a 4-tuple, got %r" % (t,))
    return (_i64 * 4)(*[int(v) for v in t])


def _i2(t):
    if len(t) != 2:
        raise ValueError("expected a 2-tuple, got %r" % (t,))
    return (_i64 * 2)(*[int(v) for v in t])


def _pair(dst, src):
    pd, td, dd = _resolve(dst)
    ps, ts, ds = _resolve(src)
    if td != ts:
        raise TypeError("dst and src element types differ: %s, %s" % (td, ts))
    if dd != ds:
        raise TypeError("dst and src must both be host pointers or both be device pointers")
    return pd, ps, _ITEMSIZE[td], dd


def _transpose(name, dst, src, dims, stream):
    pd, ps, esz, dev = _pair(dst, src)
    if dev:
        stream = _current_stream() if stream is None else stream
        check(getattr(lib(), "laser_b200_%s_dev" % name)(pd, ps, *dims, esz, stream))
    else:
        check(getattr(lib(), "laser_b200_" + name)(pd, ps, *dims, esz))


def transpose2D_copy(dst, src, NR, NC, stream=None):
    """dst[NC, NR] <- transpose of the contiguous src[NR, NC]."""
    _transpose("transpose2D_copy", dst, src, (NR, NC), stream)


def transpose2D_batched(dst, src, N, NR, NC, stream=None):
    _transpose("transpose2D_batched", dst, src, (N, NR, NC), stream)


def nchw2nhwc(dst_nhwc, src_nchw, N, C, H, W, stream=None):
    _transpose("nchw2nhwc", dst_nhwc, src_nchw, (N, C, H, W), stream)


def nhwc2nchw(dst_nchw, src_nhwc, N, C, H, W, stream=None):
    _transpose("nhwc2nchw", dst_nchw, src_nhwc, (N, C, H, W), stream)


def conv2d_out_shape(ishape, kshape, padding, strides):
    out = (_i64 * 4)()
    check(lib().laser_b200_conv2d_out_shape(_i4(ishape), _i4(kshape), _i2(padding), _i2(strides), out))
    return tuple(out)


def im2col_workspace_size(ishape, kshape, padding, strides):
    """ELEMENTS of workspace for one image: c * kH * kW * outH * outW (conv2d_im2col.nim:8-18)."""
    n = int(lib().laser_b200_im2col_workspace_size(_i4(ishape), _i4(kshape), _i2(padding), _i2(strides)))
    if n < 0:
        check(lib().laser_b200_conv2d_out_shape(_i4(ishape), _i4(kshape), _i2(padding), _i2(strides), (_i64 * 4)()))
    return n


def _dev_f32(x):
    p, t, d = _resolve(x)
    if not d or t != "f32":
        raise TypeError("expected a float32 device pointer")
    return p


def im2col(workspace, input, ishape, kshape, padding, strides, images=1, stream=None):
    """`images` images [c, h, w] starting at `input` -> `images` matrices [c*kH*kW, outH*outW]."""
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_im2col_f32_dev(_dev_f32(workspace), _dev_f32(input), images, _i4(ishape), _i4(kshape),
                                          _i2(padding), _i2(strides), stream))


def conv2d_im2col(output, input, ishape, kernel, kshape, padding, strides, workspace=None, workspace_images=1,
                  path=PATH_AUTO, stream=None):
    """NCHW convolution through im2col + GEMM.  numpy arrays: host entry (library-owned
    workspace); device pointers: `workspace` must hold workspace_images * im2col_workspace_size
    float32 elements (may be None for 1x1 / stride 1 / no padding)."""
    po, to, do = _resolve(output)
    pi, ti, di = _resolve(input)
    pk, tk, dk = _resolve(kernel)
    if not (to == ti == tk == "f32"):
        raise TypeError("conv2d_im2col is float32 only")
    if not (do == di == dk):
        raise TypeError("output, input, kernel must all be host pointers or all be device pointers")
    if not do:
        if workspace is not None or path != PATH_AUTO:
            raise ValueError("the host-pointer entry owns its workspace and has no path argument")
        check(lib().laser_b200_conv2d_im2col_f32(po, pi, _i4(ishape), pk, _i4(kshape), _i2(padding), _i2(strides)))
        return
    stream = _current_stream() if stream is None else stream
    pw = _dev_f32(workspace) if workspace is not None else 0
    check(lib().laser_b200_conv2d_im2col_f32_dev(po, pi, _i4(ishape), pk, _i4(kshape), _i2(padding), _i2(strides), pw,
                                                 int(workspace_images), int(path), stream))


def conv2d_fused(output, input, ishape, kernel, kshape, padding, strides, bias=None, bias_per_row=True, activation="none",
                 path=PATH_AUTO, stream=None):
    """output_n <- act(conv(input_n, kernel) + bias) for every image n, on float32 DEVICE buffers (NCHW in and out, kernel
    [c_out, c_in, kH, kW]).  bias_per_row=True: one bias per output channel.  activation: none | relu | tanh | sigmoid.
    The im2col step is folded into the preparation of the GEMM operand: no workspace, one GEMM launch for the images."""
    po, pi, pk = _dev_f32(output), _dev_f32(input), _dev_f32(kernel)
    epi = Epilogue()
    if bias is not None:
        epi.bias = _dev_f32(bias)
    epi.bias_per_row = 1 if bias_per_row else 0
    epi.activation = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}[activation]
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_f32_fused_dev(po, pi, _i4(ishape), pk, _i4(kshape), _i2(padding), _i2(strides),
                                                ctypes.byref(epi), int(path), stream))


def conv2d_grouped_fused(output, input, ishape, kernel, kshape, padding, strides, groups, bias=None, activation="none",
                         path=PATH_AUTO, stream=None):
    """conv2d_fused with `groups` groups, as torch.nn.functional.conv2d(groups=groups), on float32 DEVICE buffers: NCHW in and
    out, kernel [c_out, c_in / groups, kH, kW] (kshape in that order).  Output channel co of group g = co // (c_out / groups)
    sees input channels g * c_in / groups .. (g + 1) * c_in / groups - 1.  bias: one per output channel.  activation: none |
    relu | tanh | sigmoid.  One call for every group: a direct CUDA-core kernel on the exact path (depthwise and narrow
    groups), one batched tensor-core GEMM launch on the others.  groups=1 is conv2d_fused."""
    po, pi, pk = _dev_f32(output), _dev_f32(input), _dev_f32(kernel)
    epi = Epilogue()
    if bias is not None:
        epi.bias = _dev_f32(bias)
    epi.bias_per_row = 1
    epi.activation = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}[activation]
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_grouped_f32_fused_dev(po, pi, _i4(ishape), pk, _i4(kshape), _i2(padding), _i2(strides), int(groups),
                                                        ctypes.byref(epi), int(path), stream))


def conv2d_nhwc_fused(output, input, ishape, kernel, kshape, padding, strides, bias=None, activation="none", path=PATH_AUTO,
                      stream=None, kernel_strides=None):
    """output_n <- act(conv(input_n, kernel) + bias) for every image n, on float32 DEVICE buffers in channels-last layout:
    input dense NHWC [n, h, w, c], output dense NHWC [n, outH, outW, c_out]; ishape = (n, c, h, w) and kshape = (c_out, c_in,
    kH, kW) as for conv2d_fused.  kernel: a 2-D device view [kH * kW * c_in, c_out] of the filter matrix, rows in (kh, kw, ci)
    order -- e.g. a [kH, kW, c_in, c_out] tensor viewed as 2-D, or torch's channels_last weight viewed as [c_out, K] and
    transposed; its element strides are read from the view (kernel_strides: for a pointer without strides).  bias: one per
    output channel.  activation: none | relu | tanh | sigmoid.  One GEMM for the images, its A operand (the windows) prepared
    straight from the images: no workspace."""
    po, pi, pk = _dev_f32(output), _dev_f32(input), _dev_f32(kernel)
    if kernel_strides is None:
        kernel_strides = tuple(kernel.stride())
    if len(kernel_strides) != 2:
        raise ValueError("kernel must be a 2-D view [kH * kW * c_in, c_out]")
    epi = Epilogue()
    if bias is not None:
        epi.bias = _dev_f32(bias)
    epi.bias_per_row = 1
    epi.activation = {"none": 0, "relu": 1, "tanh": 2, "sigmoid": 3}[activation]
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_nhwc_f32_fused_dev(po, pi, _i4(ishape), pk, _i4(kshape), _i2(kernel_strides), _i2(padding),
                                                     _i2(strides), ctypes.byref(epi), int(path), stream))


def conv2d_filter_grad_fused(grad_kernel, input, ishape, grad_output, kshape, padding, strides, alpha=1.0, beta=0.0, op=None,
                             aux=None, path=PATH_AUTO, stream=None):
    """grad_kernel <- alpha * sum_n op(grad_output_n) * im2col(input_n)^T + beta * grad_kernel on float32 DEVICE buffers: the
    filter gradient of conv2d_fused (input and grad_output dense NCHW, grad_kernel dense [c_out, c_in, kH, kW]).  op: None or
    relu | tanh | sigmoid | relu_grad | tanh_grad | sigmoid_grad, applied to grad_output; a derivative takes `aux`, a dense
    NCHW tensor of grad_output's shape (the forward output).  beta=1 accumulates across micro-batches.  One batch-reduced
    product whose B operand is prepared straight from the images: no im2col matrix, no workspace."""
    pw, pi, pg = _dev_f32(grad_kernel), _dev_f32(input), _dev_f32(grad_output)
    o = None
    if op is not None:
        o = OperandOp()
        o.op = OP_NAMES[op]
        if aux is not None:
            _, _, oh, ow = conv2d_out_shape(ishape, kshape, padding, strides)
            o.aux = _dev_f32(aux)
            o.auxRowStride, o.auxColStride = oh * ow, 1
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_filter_grad_f32_fused_dev(pw, pi, _i4(ishape), pg, _i4(kshape), _i2(padding), _i2(strides),
                                                            float(alpha), float(beta), ctypes.byref(o) if o is not None else None,
                                                            int(path), stream))


def conv2d_nhwc_filter_grad_fused(grad_kernel, input, ishape, grad_output, kshape, padding, strides, alpha=1.0, beta=0.0, op=None,
                                  aux=None, path=PATH_AUTO, stream=None, kernel_strides=None):
    """grad_kernel <- alpha * sum_{n,p} rows[n * P + p]^T * op(grad_output)[n * P + p] + beta * grad_kernel on float32 DEVICE
    buffers: the filter gradient of conv2d_nhwc_fused (input dense NHWC [n, h, w, c], grad_output dense NHWC [n, outH, outW,
    c_out]).  grad_kernel: a 2-D device view [kH * kW * c_in, c_out] of the filter matrix, rows in (kh, kw, ci) order, whose
    element strides are read as conv2d_nhwc_fused reads them (kernel_strides: for a pointer without strides).  op: None or
    relu | tanh | sigmoid | relu_grad | tanh_grad | sigmoid_grad, applied to grad_output; a derivative takes `aux`, a dense NHWC
    tensor of grad_output's shape (the forward output).  beta=1 accumulates across micro-batches.  One product whose B operand
    (the tap rows) is prepared straight from the images: no conversion to NCHW, no workspace."""
    pw, pi, pg = _dev_f32(grad_kernel), _dev_f32(input), _dev_f32(grad_output)
    if kernel_strides is None:
        kernel_strides = tuple(grad_kernel.stride())
    if len(kernel_strides) != 2:
        raise ValueError("grad_kernel must be a 2-D view [kH * kW * c_in, c_out]")
    o = None
    if op is not None:
        o = OperandOp()
        o.op = OP_NAMES[op]
        if aux is not None:
            o.aux = _dev_f32(aux)
            o.auxRowStride, o.auxColStride = 1, kshape[0]
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_nhwc_filter_grad_f32_fused_dev(pw, pi, _i4(ishape), pg, _i4(kshape), _i2(kernel_strides),
                                                                 _i2(padding), _i2(strides), float(alpha), float(beta),
                                                                 ctypes.byref(o) if o is not None else None, int(path), stream))


def conv2d_input_grad_fused(grad_input, ishape, grad_output, kernel, kshape, padding, strides, alpha=1.0, beta=0.0, op=None,
                            aux=None, path=PATH_AUTO, stream=None):
    """grad_input <- alpha * conv_transpose(op(grad_output), kernel) + beta * grad_input on float32 DEVICE buffers: the input
    gradient of conv2d_fused (grad_input dense NCHW of shape ishape, grad_output dense NCHW, kernel dense [c_out, c_in, kH,
    kW]).  op and aux as for conv2d_filter_grad_fused, applied to grad_output.  beta=1 accumulates into an existing gradient.
    The forward call's product over the filters rotated by 180 degrees and a B operand prepared straight from grad_output
    (zero-dilated by the strides): no col2im, no workspace argument."""
    pg, po, pk = _dev_f32(grad_input), _dev_f32(grad_output), _dev_f32(kernel)
    o = None
    if op is not None:
        o = OperandOp()
        o.op = OP_NAMES[op]
        if aux is not None:
            _, _, oh, ow = conv2d_out_shape(ishape, kshape, padding, strides)
            o.aux = _dev_f32(aux)
            o.auxRowStride, o.auxColStride = oh * ow, 1
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_input_grad_f32_fused_dev(pg, _i4(ishape), po, pk, _i4(kshape), _i2(padding), _i2(strides),
                                                           float(alpha), float(beta), ctypes.byref(o) if o is not None else None,
                                                           int(path), stream))


def conv2d_grouped_input_grad_fused(grad_input, ishape, grad_output, kernel, kshape, padding, strides, groups, alpha=1.0, beta=0.0,
                                    op=None, aux=None, path=PATH_AUTO, stream=None):
    """conv2d_input_grad_fused with `groups` groups, as torch.nn.grad.conv2d_input(groups=groups), on float32 DEVICE buffers:
    the input gradient of conv2d_grouped_fused (grad_input dense NCHW of shape ishape, grad_output dense NCHW, kernel
    [c_out, c_in / groups, kH, kW]).  op and aux as for conv2d_input_grad_fused.  One call for every group: the direct
    CUDA-core kernel over the transposed geometry on the exact path (depthwise and narrow groups), one batched tensor-core
    GEMM launch per chunk on the others.  groups=1 is conv2d_input_grad_fused."""
    pg, po, pk = _dev_f32(grad_input), _dev_f32(grad_output), _dev_f32(kernel)
    o = None
    if op is not None:
        o = OperandOp()
        o.op = OP_NAMES[op]
        if aux is not None:
            _, _, oh, ow = conv2d_out_shape(ishape, kshape, padding, strides)
            o.aux = _dev_f32(aux)
            o.auxRowStride, o.auxColStride = oh * ow, 1
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_grouped_input_grad_f32_fused_dev(pg, _i4(ishape), po, pk, _i4(kshape), _i2(padding), _i2(strides),
                                                                   int(groups), float(alpha), float(beta),
                                                                   ctypes.byref(o) if o is not None else None, int(path), stream))


def conv2d_nhwc_input_grad_fused(grad_input, ishape, grad_output, kernel, kshape, padding, strides, alpha=1.0, beta=0.0, op=None,
                                 aux=None, path=PATH_AUTO, stream=None, kernel_strides=None):
    """grad_input <- alpha * conv_transpose(op(grad_output), kernel) + beta * grad_input on float32 DEVICE buffers: the input
    gradient of conv2d_nhwc_fused (grad_input dense NHWC [n, h, w, c_in], grad_output dense NHWC [n, outH, outW, c_out]).
    kernel: the 2-D device view [kH * kW * c_in, c_out] of the filter matrix conv2d_nhwc_fused takes, its element strides read
    from the view (kernel_strides: for a pointer without strides).  op and aux as for conv2d_nhwc_filter_grad_fused, applied
    to grad_output.  beta=1 accumulates into an existing gradient.  One product for the images, its A operand (the windows
    over grad_output, zero-dilated by the strides) prepared straight from grad_output: no conversion to NCHW."""
    pg, po, pk = _dev_f32(grad_input), _dev_f32(grad_output), _dev_f32(kernel)
    if kernel_strides is None:
        kernel_strides = tuple(kernel.stride())
    if len(kernel_strides) != 2:
        raise ValueError("kernel must be a 2-D view [kH * kW * c_in, c_out]")
    o = None
    if op is not None:
        o = OperandOp()
        o.op = OP_NAMES[op]
        if aux is not None:
            o.aux = _dev_f32(aux)
            o.auxRowStride, o.auxColStride = kshape[0], 1
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_conv2d_nhwc_input_grad_f32_fused_dev(pg, _i4(ishape), po, pk, _i4(kshape), _i2(kernel_strides),
                                                                _i2(padding), _i2(strides), float(alpha), float(beta),
                                                                ctypes.byref(o) if o is not None else None, int(path), stream))


def gemm_strided_batched(batch, M, N, K, alpha, A, rowStrideA, colStrideA, batchStrideA, B, rowStrideB, colStrideB,
                         batchStrideB, beta, C, rowStrideC, colStrideC, batchStrideC, path=PATH_AUTO, stream=None):
    """`batch` problems C_b <- alpha * A_b * B_b + beta * C_b on device pointers (f32, f64, i32,
    i64); a batch stride of 0 shares that operand; outputs must not overlap."""
    pa, ta, da = _resolve(A)
    pb, tb, db = _resolve(B)
    pc, tc, dc = _resolve(C)
    if not (ta == tb == tc) or ta == "bf16":
        raise TypeError("batched GEMM needs A, B, C of one type among f32, f64, i32, i64 (got %s, %s, %s)" % (ta, tb, tc))
    if not (da and db and dc):
        raise TypeError("batched GEMM takes device pointers")
    stream = _current_stream() if stream is None else stream
    args = [batch, M, N, K, _scalar(ta, alpha), pa, rowStrideA, colStrideA, batchStrideA, pb, rowStrideB, colStrideB,
            batchStrideB, _scalar(ta, beta), pc, rowStrideC, colStrideC, batchStrideC]
    if ta == "f32":
        check(lib().laser_b200_gemm_strided_batched_f32_dev(*args, int(path), stream))
    else:
        if path not in (PATH_AUTO, 1):
            raise ValueError("path %d is not available for %s" % (path, ta))
        check(getattr(lib(), "laser_b200_gemm_strided_batched_%s_dev" % ta)(*args, stream))


def copyFrom(dst, src, stream=None):
    """dst <- src for two device Tensors of the same shape and dtype, any strides; only the
    elements the dst view exposes are written (initialization.nim:80-112)."""
    if not isinstance(dst, Tensor) or not isinstance(src, Tensor):
        raise TypeError("copyFrom takes laser_b200.Tensor views (use Tensor.from_torch for torch tensors)")
    vd, vs = dst.view_struct(), src.view_struct()
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_copy_views(ctypes.byref(vd), ctypes.byref(vs), stream))
    return dst


def forEach(op, out, x=None, y=None, z=None, alpha=0.0, stream=None):
    """forEach o in out, x in a, y in b, z in c: <body> on device Tensors of one shape, any strides
    (laser/strided_iteration/foreach.nim:229-251).  `op` names the body:
      copy o = x | fill o = alpha | scale o = alpha*x | add o = x+y | sub o = x-y | mul o = x*y |
      fma o = x + y*z | axpy o = alpha*x + y | bench o = x + y - sin(z) (the reference's iteration benchmark)"""
    code = FOREACH_OPS[op] if isinstance(op, str) else int(op)
    views = [t.view_struct() if t is not None else None for t in (out, x, y, z)]
    refs = [ctypes.byref(v) if v is not None else None for v in views]
    stream = _current_stream() if stream is None else stream
    check(lib().laser_b200_foreach_views(code, refs[0], refs[1], refs[2], refs[3], float(alpha), stream))
    return out
