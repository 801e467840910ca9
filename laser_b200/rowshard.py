"""Row-panel sharding of a large GEMM across the GPUs of one box: the Python mirror of
laser_b200_gemm_rowsharded_f32_dev / laser_b200_gemm_rowsharded_f32 (include/laser_b200.h).

The reference parallelises exactly this way on a CPU: its `ic` loop hands each worker a row block of A
and C while all workers share one packed panel of B (gemm.nim:160-176).  Here a worker is a GPU:
  * rank r owns rows [start_r, stop_r) of A and C (never moved);
  * B lives on `src` and is broadcast ONCE per product over NCCL / NVLink by the library itself (ncclBroadcast on
    a communication stream of the communicator) -- no collective inside the MMA loop, no reduction;
  * the scale + split of the rank's rows of A is queued before the wait for B, so it overlaps the transfer.
Everything on the data path happens behind the C ABI; torch.distributed is used only to hand the 128-byte NCCL
unique id from rank 0 to the other ranks when the communicator is created (any backend: gloo, nccl).
"""
import ctypes

from ._capi import check, lib
from .gemm import _current_stream, _resolve

__all__ = ["partition_rows", "Comm", "comm_init_all", "comm_init_rank", "comm_from_torch_distributed", "gemm_rowsharded",
           "gemm_rowsharded_dev", "gemm_rowsharded_host"]


def partition_rows(M, world_size, align=256):
    """[(start, stop)] per rank: ceil(M / world) rounded up to a multiple of 256 rows (the partition the library has always
    used); the last ranks take what is left (possibly nothing).  Same rule as laser_b200_rowshard_partition (align = 256)."""
    per = -(-M // world_size)
    per = -(-per // align) * align
    out = []
    for r in range(world_size):
        lo = min(M, r * per)
        out.append((lo, min(M, lo + per)))
    return out


def partition_rows_c(M, world_size, rank):
    """(start, stop) of `rank` as the library computes it."""
    a, n = ctypes.c_int64(), ctypes.c_int64()
    lib().laser_b200_rowshard_partition(int(M), int(world_size), int(rank), ctypes.byref(a), ctypes.byref(n))
    return a.value, a.value + n.value


class Comm:
    """Owner of a laser_b200_comm handle (one rank of a row-sharded product on one device)."""

    def __init__(self, handle):
        self.handle = ctypes.c_void_p(handle)

    @property
    def rank(self):
        return lib().laser_b200_comm_rank(self.handle)

    @property
    def size(self):
        return lib().laser_b200_comm_size(self.handle)

    def destroy(self):
        if self.handle:
            check(lib().laser_b200_comm_destroy(self.handle))
            self.handle = ctypes.c_void_p(None)


def comm_get_unique_id():
    buf = ctypes.create_string_buffer(128)
    check(lib().laser_b200_comm_get_unique_id(buf))
    return buf.raw


def comm_init_rank(nranks, rank, unique_id):
    """The calling thread's current CUDA device joins a communicator of `nranks` (one process or thread per GPU)."""
    h = ctypes.c_void_p()
    buf = ctypes.create_string_buffer(bytes(unique_id), 128) if unique_id is not None else None
    check(lib().laser_b200_comm_init_rank(ctypes.byref(h), int(nranks), int(rank), buf))
    return Comm(h.value)


def comm_init_all(ngpus):
    """One process driving devices 0 .. ngpus-1: a list of `ngpus` communicators (rank d on device d)."""
    arr = (ctypes.c_void_p * ngpus)()
    check(lib().laser_b200_comm_init_all(arr, int(ngpus)))
    return [Comm(arr[d]) for d in range(ngpus)]


_dist_comms = {}


def comm_from_torch_distributed(group=None):
    """The communicator of this rank of a torch.distributed job (created once per group): rank 0 draws the NCCL unique
    id, torch.distributed carries the 128 bytes to the other ranks, every rank joins with its current device."""
    import torch.distributed as dist
    key = id(group)
    if key not in _dist_comms:
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        box = [comm_get_unique_id() if rank == 0 and world > 1 else None]
        if world > 1:
            dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        _dist_comms[key] = comm_init_rank(world, rank, box[0])
    return _dist_comms[key]


def gemm_rowsharded(M_local, N, K, alpha, A_local, B, beta, C_local, src=0, comm=None, group=None, stream=None, gemm_fn=None):
    """C_local <- alpha * A_local @ B + beta * C_local on every rank (device buffers on this rank's GPU).

    A_local: (M_local, K) view (any strides), C_local: (M_local, N) view, B: (K, N) dense tensor on every rank, an INPUT
    that needs to be valid on `src` only.  On the other ranks the buffer is scratch: the library may fill it with B (raw
    broadcast) or leave it alone (default fp32 mode, row- or column-major B: B travels prepared, in column panels).  gemm_fn (tests of the host logic only): a
    gemm_strided-like callable that stands in for the library, with torch.distributed doing the broadcast."""
    rsA, csA = (A_local.stride(0), A_local.stride(1)) if M_local > 0 else (K, 1)
    rsC, csC = (C_local.stride(0), C_local.stride(1)) if M_local > 0 else (N, 1)
    rsB, csB = B.stride(0), B.stride(1)
    if gemm_fn is not None:
        import torch.distributed as dist
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.broadcast(B, src=src, group=group)
        if M_local > 0:
            gemm_fn(M_local, N, K, alpha, A_local, rsA, csA, B, rsB, csB, beta, C_local, rsC, csC)
        return C_local
    if comm is None:
        comm = comm_from_torch_distributed(group)
    return gemm_rowsharded_dev(comm, M_local, N, K, alpha, A_local, rsA, csA, B, rsB, csB, src, beta, C_local, rsC, csC, stream)


def gemm_rowsharded_dev(comm, M_local, N, K, alpha, A_local, rsA, csA, B, rsB, csB, root, beta, C_local, rsC, csC, stream=None):
    """laser_b200_gemm_rowsharded_f32_dev with explicit element strides (device buffers: torch CUDA tensors, Tensor, DevPtr)."""
    pb, tb, db = _resolve(B)
    if not db or tb != "f32":
        raise TypeError("gemm_rowsharded takes float32 device buffers")
    pa = pc = 0
    if M_local > 0:
        pa, ta, da = _resolve(A_local); pc, tc, dc = _resolve(C_local)
        if not (da and dc and ta == tc == "f32"):
            raise TypeError("gemm_rowsharded takes float32 device buffers")
    if stream is None:
        stream = _current_stream()
    check(lib().laser_b200_gemm_rowsharded_f32_dev(comm.handle, int(M_local), int(N), int(K), float(alpha), pa, rsA, csA, pb, rsB,
                                                   csB, int(root), float(beta), pc, rsC, csC, stream))
    return C_local


def gemm_rowsharded_host(ngpus, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC):
    """The reference signature with HOST (numpy) buffers, row panels spread over `ngpus` devices of this process."""
    pa, ta, da = _resolve(A); pb, tb, db = _resolve(B); pc, tc, dc = _resolve(C)
    if da or db or dc or not (ta == tb == tc == "f32"):
        raise TypeError("gemm_rowsharded_host takes float32 numpy arrays")
    check(lib().laser_b200_gemm_rowsharded_f32(int(ngpus), int(M), int(N), int(K), float(alpha), pa, rsA, csA, pb, rsB, csB,
                                               float(beta), pc, rsC, csC))
