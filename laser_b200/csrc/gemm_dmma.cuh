// gemm_dmma.cuh -- fp64 strided GEMM on the FP64 tensor cores (mma.sync.m8n8k4.f64, "DMMA").
//
// Same contract as the exact CUDA-core kernel (gemm_simt.cuh), same parameter block (SimtParams<double>), same numerics:
// every C[i,j] is the k-sequential FMA chain from 0 inside blocks of kc = 2048 / sizeof(double) = 256 (gemm_tiling.nim:
// 309-310), followed per block by the reference epilogue on C itself with beta' = beta on the first block and 1 afterwards
// (gemm.nim:150-158, gemm_ukernel_generic.nim:53-76).  One DMMA computes, per output element, four steps of exactly that
// chain (d = fma(a_k, b_k, d) for k = 0..3 in order -- checked bit for bit against the oracle by
// tests/test_gpu_parity.py::test_f64_dmma_bit_exact), so the tensor core only changes who executes the chain.  wgmma has
// no fp64 type; mma.sync is the one tensor path the part offers for doubles (gemm.nim:234-246 dispatches float64 to the
// same loop nest as float32: this is that row of the dispatch).
//
// Tiling: 128 x 128 x 16 block tile, 256 threads = 8 warps in a 4 (m) x 2 (n) grid, warp tile 32 x 64 = 4 x 8 DMMA tiles
// (64 accumulator doubles per thread).  Operands of any strides travel global -> shared as 8-byte cp.async copies (no
// register staging; elements outside the matrix or past K arrive as zeros), three k-tiles deep; the thread -> element
// mapping follows the smaller stride, as in the SIMT kernel.  Tiles are stored k-major with a row pitch of 132 doubles: the
// fragment reads (lane -> k = lane % 4, m or n = lane / 4) then hit 16 different 8-byte banks per half-warp.
#pragma once

#include "gemm_simt.cuh"
#include "ptx.cuh"

namespace lb200 {

constexpr int DMMA_BM = 128, DMMA_BN = 128, DMMA_BK = 16, DMMA_LD = 132, DMMA_STAGES = 3;

#ifndef LB200_HOST_EMULATION
__device__ __forceinline__ void dmma_m8n8k4(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
#endif

inline int64_t dmma_plan(SimtParams<double> &p, int64_t M, int64_t N, int64_t K, double alpha, const double *A, int64_t rsA,
                         int64_t csA, const double *B, int64_t rsB, int64_t csB, double beta, double *C, int64_t rsC,
                         int64_t csC) {
  simt_plan<double, 8, 8>(p, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);   // 16 * 8 = 128-wide tiles
  return static_cast<int64_t>(p.num_m_blocks) * p.num_n_blocks;
}

__global__ void __launch_bounds__(256, 1)
gemm_dmma_kernel(const SimtParams<double> p) {
  constexpr int BM = DMMA_BM, BN = DMMA_BN, BK = DMMA_BK, LD = DMMA_LD, ST = DMMA_STAGES;
  constexpr int PER_T = BM * BK / 256;   // 8 elements of A and of B per thread and k-tile
  constexpr int64_t KC = 2048 / static_cast<int64_t>(sizeof(double));
  static_assert(KC % BK == 0, "k-tiles never straddle a kc block");
  LB200_DYN_SMEM(double, smem);          // ST stages of { As[BK][LD], Bs[BK][LD] }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 64;
  const int fk = lane & 3, fr = lane >> 2;     // fragment coordinates: k inside the group of four, row (of A) / column (of B)
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int64_t total_tiles = static_cast<int64_t>(num_tiles) * p.batch;
  const int64_t num_kt = (p.K + BK - 1) / BK;

  for (int64_t t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int64_t bi = t / num_tiles;
    const int tile = static_cast<int>(t - bi * num_tiles);
    const double *Ab = p.A + bi * p.bsA;
    const double *Bb = p.B + bi * p.bsB;
    double *Cb = p.C + bi * p.bsC;
    const int mb = tile % p.num_m_blocks, nb = tile / p.num_m_blocks;
    const int64_t m0 = static_cast<int64_t>(mb) * BM, n0 = static_cast<int64_t>(nb) * BN;

    // k-tile kt of this output tile -> stage kt % ST (always one commit group per call, possibly empty)
    auto issue_tile = [&](int64_t kt) {
      if (kt < num_kt) {
        double *As = smem + (kt % ST) * (2 * BK * LD), *Bs = As + BK * LD;
        const int64_t k0 = kt * BK;
#pragma unroll
        for (int i = 0; i < PER_T; ++i) {
          const int idx = tid + i * 256;
          const int m = p.a_along_m ? (idx % BM) : (idx / BK);
          const int k = p.a_along_m ? (idx / BM) : (idx % BK);
          const int64_t gm = m0 + m, gk = k0 + k;
          const bool ok = gm < p.M && gk < p.K;
          ptx::cp_async_8(&As[k * LD + m], ok ? Ab + gm * p.rsA + gk * p.csA : Ab, ok);
        }
#pragma unroll
        for (int i = 0; i < PER_T; ++i) {
          const int idx = tid + i * 256;
          const int n = p.b_along_k ? (idx / BK) : (idx % BN);
          const int k = p.b_along_k ? (idx % BK) : (idx / BN);
          const int64_t gn = n0 + n, gk = k0 + k;
          const bool ok = gn < p.N && gk < p.K;
          ptx::cp_async_8(&Bs[k * LD + n], ok ? Bb + gk * p.rsB + gn * p.csB : Bb, ok);
        }
      }
      ptx::cp_async_commit();
    };
#pragma unroll
    for (int s = 0; s < ST - 1; ++s) issue_tile(s);

    double acc[4][8][2];
    for (int64_t kt = 0; kt < num_kt; ++kt) {
      const int64_t k0 = kt * BK;
      if (k0 % KC == 0) {   // a kc block of the reference's loop 2 starts (gemm.nim:150): its FMA chains start from 0
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
      }
      ptx::cp_async_wait<ST - 2>();   // this thread's copies of tile kt have landed ...
      __syncthreads();                // ... everybody's have, and tile kt - 1 is fully consumed: its stage may be refilled
      issue_tile(kt + ST - 1);
      const double *As = smem + (kt % ST) * (2 * BK * LD), *Bs = As + BK * LD;
      // groups of four k; a group past K holds zeros only and is skipped (it would turn a -0 sum into +0)
      const int groups = static_cast<int>(((p.K - k0 < BK ? p.K - k0 : BK) + 3) / 4);
#pragma unroll
      for (int g = 0; g < BK / 4; ++g) {
        if (g < groups) {
          double a[4], b[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = As[(4 * g + fk) * LD + wm + 8 * i + fr];
#pragma unroll
          for (int j = 0; j < 8; ++j) b[j] = Bs[(4 * g + fk) * LD + wn + 8 * j + fr];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
        }
      }
      if ((k0 + BK) % KC == 0 || kt + 1 == num_kt) {
        // reference epilogue for this kc block (gemm_ukernel_generic.nim:53-76): beta on the first block, 1 afterwards
        const double beta1 = (k0 < KC) ? p.beta : 1.0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int64_t gm = m0 + wm + 8 * i + fr;
          if (gm >= p.M) continue;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int64_t gn = n0 + wn + 8 * j + 2 * fk + e;
              if (gn >= p.N) continue;
              double *c = Cb + gm * p.rsC + gn * p.csC;
              double v;
              if (beta1 == 0.0) v = 0.0;
              else if (beta1 != 1.0) v = __dmul_rn(*c, beta1);
              else v = *c;
              if (p.alpha == 1.0) v = __dadd_rn(v, acc[i][j][e]);
              else v = __dadd_rn(v, __dmul_rn(p.alpha, acc[i][j][e]));
              *c = v;
            }
          }
        }
      }
    }
    ptx::cp_async_wait<0>();
    __syncthreads();   // the stages are free again before the next tile's prologue refills them
  }
}
constexpr size_t DMMA_SMEM_BYTES = static_cast<size_t>(DMMA_STAGES) * 2 * DMMA_BK * DMMA_LD * sizeof(double);   // 101 KB

}  // namespace lb200
