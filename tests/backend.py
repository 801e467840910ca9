"""Backend of the `-m gpu` test files: an H100 through torch CUDA tensors, or -- LASER_B200_EMU=1, set by
tests/test_emulated_python_mirror.py together with LASER_B200_LIB -- the host-emulated build of the
library, where "device" memory is host memory held by numpy arrays."""
import os

import numpy as np
import pytest

EMU = os.environ.get("LASER_B200_EMU", "0") == "1"
if not EMU:
    torch = pytest.importorskip("torch")

needs_gpu = pytest.mark.skipif(EMU, reason="uses torch CUDA tensors directly / too large for the CPU build")


import laser_b200 as L  # noqa: E402

_NAME = {np.dtype(np.int16): "bf16", np.dtype(np.uint16): "bf16", np.dtype(np.float32): "f32", np.dtype(np.float64): "f64",
         np.dtype(np.int32): "i32", np.dtype(np.int64): "i64"}


class HostTensor(L.DevPtr):
    """EMU backend: a numpy array posing as device memory.  It is a DevPtr, so it can be handed to the
    Python mirror like a torch CUDA tensor, and it has the few torch.Tensor methods the tests use."""

    def __init__(self, arr):
        self.arr = np.ascontiguousarray(arr)
        super().__init__(self.arr.ctypes.data, _NAME.get(self.arr.dtype, "f32"))

    def data_ptr(self):
        return self.arr.ctypes.data

    def element_size(self):
        return self.arr.itemsize

    def cpu(self):
        return self

    def numpy(self):
        return self.arr


def dev(buf):
    """host array -> device array (a copy)"""
    buf = np.ascontiguousarray(buf)
    return HostTensor(buf.copy()) if EMU else torch.from_numpy(buf).cuda()


def sync():
    if not EMU:
        torch.cuda.synchronize()


def emu_budget(work):
    """skip problems whose M*N*K would take too long on host threads"""
    if EMU and work > 1.2e8:
        pytest.skip("too large for the CPU build")
