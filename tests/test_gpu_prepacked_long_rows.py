"""GPU: the pre-pack prepares long K-major rows as the unpacked default-mode product does, bit for bit -- rows the
shared-memory ring kernel takes (1024 < K <= 8192 floats, 16-byte aligned) and rows just past that range."""
import numpy as np
import pytest

import oracle as O
from backend import dev, emu_budget, sync

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402


@pytest.mark.parametrize("K", [2048, 8200])
def test_packed_long_rows_match_unpacked(K):
    """row-major A and column-major B: both are K-major, so both pre-packs run the row kernel on the caller's memory"""
    M, N = 96, 72
    emu_budget(M * N * K)
    A = O.fill_uniform_f32(M * K, 41, 0, 1).reshape(M, K)
    B = O.fill_uniform_f32(K * N, 42, 0, 1).reshape(K, N)
    tA, tB = dev(A), dev(np.ascontiguousarray(B.T))     # B column-major: element (k, n) at n * K + k
    pa = L.alloc_packed(L.gemm_prepackA_mem_required(M, N, K)); pb = L.alloc_packed(L.gemm_prepackB_mem_required(M, N, K))
    L.gemm_prepackA(pa, M, N, K, tA, K, 1)
    L.gemm_prepackB(pb, M, N, K, tB, 1, K)
    C0 = np.zeros((M, N), np.float32)
    tC, tC2, tC3 = dev(C0), dev(C0), dev(C0)
    L.gemm_packed(M, N, K, 1.0, pa, pb, 0.0, tC, N, 1)
    L.gemm_packedB(M, N, K, 1.0, tA, K, 1, pb, 0.0, tC2, N, 1)
    L.gemm_strided(M, N, K, 1.0, tA, K, 1, tB, 1, K, 0.0, tC3, N, 1, path=L.PATH_F16X3)
    sync()
    want = C0.copy(); O.gemm_strided(M, N, K, 1.0, A, K, 1, B, N, 1, 0.0, want, N, 1)
    got = tC3.cpu().numpy()
    assert O.max_relative_error(got, want) < 1e-4
    assert np.array_equal(tC.cpu().numpy(), got) and np.array_equal(tC2.cpu().numpy(), got)
