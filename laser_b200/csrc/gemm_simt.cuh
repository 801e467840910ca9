// gemm_simt.cuh -- exact CUDA-core strided GEMM (fp32 FFMA; also f64 / i32 / i64).
//
// The non-tensor-core path: any strides, any alignment, any size.  For float
// types every C[i,j] is produced by the SAME sequence of operations as the
// reference CPU path, so results are bit-identical to it (and to oracle/):
//   - k-sequential FMA chain from 0 inside blocks of kc = min(2048/sizeof(T), K)
//       (gemm_tiling.nim:309-310, gemm_ukernel_generator.nim:196-250)
//   - after every kc block the reference epilogue runs on C itself, with
//       beta' = beta on the first block and 1 afterwards   (gemm.nim:150-158,
//       gemm_ukernel_generic.nim:53-76): beta'==0 -> C not read.
// Integer types wrap (the reference uses mullo + add).
//
// Tiling: (16*TM) x (16*TN) x BK block tile, 256 threads, TM x TN outputs per thread
// in two strided halves so that shared-memory reads are 16-byte broadcasts and the
// C accesses of a warp are contiguous along N.  Global loads of the next k-tile are
// issued into registers before the FMAs of the current one (software pipelining);
// the thread -> element mapping of the loads follows whichever stride of the operand
// is smaller so that HBM accesses coalesce for row-major, transposed and sliced views.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "layers.cuh"
#include "ptx.cuh"
#include "split.cuh"

namespace lb200 {

template <typename T> struct SimtOps;
template <> struct SimtOps<float> {
  static __device__ __forceinline__ float fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
};
template <> struct SimtOps<double> {
  static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
};
template <> struct SimtOps<int32_t> {
  static __device__ __forceinline__ int32_t fma(int32_t a, int32_t b, int32_t c) {
    return static_cast<int32_t>(static_cast<uint32_t>(a) * static_cast<uint32_t>(b) + static_cast<uint32_t>(c));
  }
  static __device__ __forceinline__ int32_t mul(int32_t a, int32_t b) {
    return static_cast<int32_t>(static_cast<uint32_t>(a) * static_cast<uint32_t>(b));
  }
  static __device__ __forceinline__ int32_t add(int32_t a, int32_t b) {
    return static_cast<int32_t>(static_cast<uint32_t>(a) + static_cast<uint32_t>(b));
  }
};
template <> struct SimtOps<int64_t> {
  static __device__ __forceinline__ int64_t fma(int64_t a, int64_t b, int64_t c) {
    return static_cast<int64_t>(static_cast<uint64_t>(a) * static_cast<uint64_t>(b) + static_cast<uint64_t>(c));
  }
  static __device__ __forceinline__ int64_t mul(int64_t a, int64_t b) {
    return static_cast<int64_t>(static_cast<uint64_t>(a) * static_cast<uint64_t>(b));
  }
  static __device__ __forceinline__ int64_t add(int64_t a, int64_t b) {
    return static_cast<int64_t>(static_cast<uint64_t>(a) + static_cast<uint64_t>(b));
  }
};

template <typename T>
struct SimtParams {
  int64_t M, N, K;
  T alpha, beta;
  const T *A; int64_t rsA, csA;
  const T *B; int64_t rsB, csB;
  T *C; int64_t rsC, csC;
  int a_along_m;  // 1: consecutive loader threads walk m (|rsA| < |csA|), 0: walk k
  int b_along_k;  // 1: consecutive loader threads walk k (|rsB| < |csB|), 0: walk n
  int num_m_blocks, num_n_blocks;
  // fused epilogue (float only), applied after the LAST kc block: v -> act(v + bias)
  const float *bias = nullptr;
  int bias_per_row = 0;
  int act = 0;
  // batch of independent problems in one launch: problem b reads A + b*bsA, B + b*bsB and
  // writes C + b*bsC (a stride of 0 shares the operand; outputs must not overlap)
  int64_t batch = 1, bsA = 0, bsB = 0, bsC = 0;
};

// host side: everything but the fused epilogue; returns the number of output tiles
template <typename T, int TM, int TN>
inline int64_t simt_plan(SimtParams<T> &p, int64_t M, int64_t N, int64_t K, T alpha, const T *A, int64_t rsA,
                         int64_t csA, const T *B, int64_t rsB, int64_t csB, T beta, T *C, int64_t rsC,
                         int64_t csC) {
  p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.beta = beta;
  p.A = A; p.rsA = rsA; p.csA = csA;
  p.B = B; p.rsB = rsB; p.csB = csB;
  p.C = C; p.rsC = rsC; p.csC = csC;
  p.a_along_m = ((rsA < 0 ? -rsA : rsA) < (csA < 0 ? -csA : csA)) ? 1 : 0;
  p.b_along_k = ((rsB < 0 ? -rsB : rsB) < (csB < 0 ? -csB : csB)) ? 1 : 0;
  constexpr int BM = 16 * TM, BN = 16 * TN;
  const int64_t mblocks = (M + BM - 1) / BM, nblocks = (N + BN - 1) / BN;
  p.num_m_blocks = static_cast<int>(mblocks);
  p.num_n_blocks = static_cast<int>(nblocks);
  return mblocks * nblocks;
}

// bias + activation of the fused epilogue, out of line: inlined into the unrolled MT x NC store loops the tanhf / expf bodies
// made the kernels several times larger than the instruction cache (ncu: 58 % of the stall samples "no instruction")
#ifndef LB200_HOST_EMULATION
static __device__ __noinline__
#else
inline
#endif
float simt_bias_act(float x, const float *bias, int bias_per_row, int act, int64_t row, int64_t col) {
  if (bias) x += bias_per_row ? bias[row] : bias[col];
  if (act == 1) x = fmaxf(x, 0.0f);
  else if (act == 2) x = tanhf(x);
  else if (act == 3) x = 1.0f / (1.0f + expf(-x));
  return x;
}
#ifndef LB200_SIMT_MINB
#define LB200_SIMT_MINB 1
#endif
#define LB200_SIMT_KERNEL_NAME gemm_simt_kernel
#define LB200_SIMT_BATCHED 0
#include "gemm_simt_kernel.inc"
#undef LB200_SIMT_KERNEL_NAME
#undef LB200_SIMT_BATCHED
#define LB200_SIMT_KERNEL_NAME gemm_simt_batched_kernel
#define LB200_SIMT_BATCHED 1
#include "gemm_simt_kernel.inc"
#undef LB200_SIMT_KERNEL_NAME
#undef LB200_SIMT_BATCHED

// dynamic shared memory (tests/emu runs this header on host threads, where it is a plain buffer)
#ifndef LB200_DYN_SMEM
#ifdef LB200_HOST_EMULATION
#define LB200_DYN_SMEM(T, name) T *name = reinterpret_cast<T *>(emu::dyn_smem_ptr())
#else
#define LB200_DYN_SMEM(T, name) extern __shared__ T name[]
#endif
#endif

// ---------------------------------------------------------------------------
// Skinny GEMM: N <= 4 (matrix x few vectors).  One warp per output row: lanes stride
// over K with coalesced loads of A's row, partial dot products are combined with
// warp shuffles.  Not bit-identical to the reference's k-sequential chain (the
// reduction tree differs) - used only when the caller asks for PATH_AUTO on a
// skinny problem; PATH_SIMT always takes the exact kernel above.
// ---------------------------------------------------------------------------
template <int NV, bool VEC>
__global__ void __launch_bounds__(256)
gemv_warp_kernel(int64_t M, int64_t K, float alpha, const float *__restrict__ A, int64_t rsA,
                 int64_t csA, const float *__restrict__ B, int64_t rsB, int64_t csB, float beta,
                 float *__restrict__ C, int64_t rsC, int64_t csC) {
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < M;
       row += warps_total) {
    float acc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) acc[j] = 0.0f;
    const float *a = A + row * rsA;
    if constexpr (VEC) {
      // A rows contiguous and 16-byte aligned, K % 4 == 0: each lane streams float4s, four
      // independent 16-byte loads in flight per lane (the kernel is pure HBM streaming of A)
      const float4 *a4 = reinterpret_cast<const float4 *>(a);
      const int64_t K4 = K >> 2;
#pragma unroll 4
      for (int64_t q = lane; q < K4; q += 32) {
        const float4 av = __ldg(a4 + q);
        const int64_t k = q << 2;
#pragma unroll
        for (int j = 0; j < NV; ++j) {
          acc[j] = fmaf(av.x, __ldg(B + (k + 0) * rsB + j * csB), acc[j]);
          acc[j] = fmaf(av.y, __ldg(B + (k + 1) * rsB + j * csB), acc[j]);
          acc[j] = fmaf(av.z, __ldg(B + (k + 2) * rsB + j * csB), acc[j]);
          acc[j] = fmaf(av.w, __ldg(B + (k + 3) * rsB + j * csB), acc[j]);
        }
      }
    } else {
#pragma unroll 4
      for (int64_t k = lane; k < K; k += 32) {
        const float av = a[k * csA];
#pragma unroll
        for (int j = 0; j < NV; ++j) acc[j] = fmaf(av, B[k * rsB + j * csB], acc[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], off);
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        float *c = C + row * rsC + j * csC;
        const float v = alpha * acc[j];
        *c = (beta == 0.0f) ? v : fmaf(beta, *c, v);
      }
    }
  }
}

// Same contract, B (K x NV) staged once per CTA in shared memory, transposed to Bs[j][k] so
// that each 16-byte load of A is matched by NV 16-byte shared loads instead of 4*NV global
// ones.  Needs A rows contiguous + 16-byte aligned, K % 4 == 0 and NV*K*4 bytes of smem.
template <int NV>
__global__ void __launch_bounds__(256)
gemv_warp_smem_kernel(int64_t M, int64_t K, float alpha, const float *__restrict__ A, int64_t rsA,
                      const float *__restrict__ B, int64_t rsB, int64_t csB, float beta,
                      float *__restrict__ C, int64_t rsC, int64_t csC) {
  LB200_DYN_SMEM(float4, gemv_smem4);
  float *Bs = reinterpret_cast<float *>(gemv_smem4);
  for (int64_t i = threadIdx.x; i < K * NV; i += blockDim.x) {
    const int64_t k = i / NV;
    const int j = static_cast<int>(i - k * NV);
    Bs[j * K + k] = B[k * rsB + j * csB];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warps_total = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int64_t K4 = K >> 2;
  for (int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < M;
       row += warps_total) {
    float acc[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) acc[j] = 0.0f;
    const float4 *a4 = reinterpret_cast<const float4 *>(A + row * rsA);
#pragma unroll 8
    for (int64_t q = lane; q < K4; q += 32) {
      const float4 av = __ldg(a4 + q);
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const float4 bv = *reinterpret_cast<const float4 *>(Bs + j * K + (q << 2));
        acc[j] = fmaf(av.x, bv.x, acc[j]);
        acc[j] = fmaf(av.y, bv.y, acc[j]);
        acc[j] = fmaf(av.z, bv.z, acc[j]);
        acc[j] = fmaf(av.w, bv.w, acc[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], off);
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        float *c = C + row * rsC + j * csC;
        const float v = alpha * acc[j];
        *c = (beta == 0.0f) ? v : fmaf(beta, *c, v);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Few output ROWS, very wide N: the GEMM of the im2col convolution (conv2d_im2col.nim:150-166: M = filters = 20,
// K = C * kH * kW = 27, N = outH * outW = 49284 per image).  A 128 x 128 tile of the general kernel would compute 84 %
// padding; here a thread owns 4 consecutive columns of ALL rows: per k one 16-byte load of B (coalesced along n), MT / 4
// 16-byte broadcast reads of A's k-th column from shared memory and 4 * MT FMAs -- the kernel streams B and C once.
// Exact: every C[i,j] is the reference's k-sequential FMA chain inside kc = 512 blocks with the reference epilogue per
// block (same statements as gemm_simt_kernel), so results are bit-identical to the general kernel's.  Batched like it.
// MT: rows held in registers (M <= MT, a multiple of 4).
// ---------------------------------------------------------------------------
constexpr int SKINNY_KCHUNK = 64;   // k-columns of A staged in shared memory at a time
// NC: columns per thread (4 for MT <= 16, 2 above: MT * NC running sums per thread must leave room for two CTAs per SM)
template <int MT, int NC>
__global__ void __launch_bounds__(256, 2)
gemm_skinny_m_kernel(const SimtParams<float> p) {
  static_assert(MT % 4 == 0 && MT <= 32 && (NC == 2 || NC == 4), "rows in registers");
  constexpr int64_t KC = 2048 / 4;   // gemm_tiling.nim:310
  constexpr int COLS = 256 * NC;     // columns per CTA and iteration
  __shared__ float4 As4[SKINNY_KCHUNK][MT / 4];   // As[k][m]: the m of one k are contiguous (16-byte broadcast reads)
  float *As = reinterpret_cast<float *>(As4);
  const int tid = threadIdx.x;
  const int64_t nblocks = (p.N + COLS - 1) / COLS;
  const int64_t total = nblocks * p.batch;
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int64_t bi = t / nblocks;
    const int64_t n0 = (t - bi * nblocks) * COLS + NC * tid;
    const float *Ab = p.A + bi * p.bsA;
    const float *Bb = p.B + bi * p.bsB;
    float *Cb = p.C + bi * p.bsC;
    const bool vec_b = p.csB == 1 && n0 + NC <= p.N &&
                       ((reinterpret_cast<uintptr_t>(Bb + n0) | (static_cast<uint64_t>(p.rsB) * 4)) & (4 * NC - 1)) == 0;
    for (int64_t pc = 0; pc < p.K; pc += KC) {  // reference loop 2 (gemm.nim:150)
      const int64_t kend = (pc + KC < p.K) ? pc + KC : p.K;
      float acc[MT][NC];
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NC; ++j) acc[i][j] = 0.0f;
      for (int64_t k0 = pc; k0 < kend; k0 += SKINNY_KCHUNK) {
        const int kn = static_cast<int>(kend - k0 < SKINNY_KCHUNK ? kend - k0 : SKINNY_KCHUNK);
        __syncthreads();   // the previous chunk of A is consumed
        for (int i = tid; i < SKINNY_KCHUNK * MT; i += 256) {
          const int k = i / MT, m = i - k * MT;
          As[i] = (m < p.M && k < kn) ? Ab[m * p.rsA + (k0 + k) * p.csA] : 0.0f;
        }
        __syncthreads();
        if (n0 < p.N) {
          // (k-steps in flight: as many as the register budget of two CTAs per SM allows next to the MT * NC sums)
#pragma unroll(MT * NC > 48 ? 2 : 4)
          for (int k = 0; k < kn; ++k) {
            float b[NC];
            const float *brow = Bb + (k0 + k) * p.rsB + n0 * p.csB;
            if (vec_b) {
              if constexpr (NC == 4) {
                const float4 v = *reinterpret_cast<const float4 *>(brow);
                b[0] = v.x; b[1] = v.y; b[2] = v.z; b[3] = v.w;
              } else {
                const float2 v = *reinterpret_cast<const float2 *>(brow);
                b[0] = v.x; b[1] = v.y;
              }
            } else {
#pragma unroll
              for (int j = 0; j < NC; ++j) b[j] = (n0 + j < p.N) ? brow[j * p.csB] : 0.0f;
            }
#pragma unroll
            for (int i4 = 0; i4 < MT / 4; ++i4) {
              const float4 a = As4[k][i4];
              const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
              for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int j = 0; j < NC; ++j) acc[4 * i4 + e][j] = __fmaf_rn(av[e], b[j], acc[4 * i4 + e][j]);
            }
          }
        }
      }
      // reference epilogue for this kc block (gemm_ukernel_generic.nim:53-76)
      const float beta1 = (pc == 0) ? p.beta : 1.0f;
      const bool has_epi = kend == p.K && (p.bias != nullptr || p.act != 0);
      if (n0 < p.N) {
#pragma unroll
        for (int i = 0; i < MT; ++i) {
          if (i >= p.M) break;
          float *crow = Cb + i * p.rsC + n0 * p.csC;
          float v[NC];
#pragma unroll
          for (int j = 0; j < NC; ++j) {
            if (n0 + j >= p.N) { v[j] = 0.0f; continue; }
            float x;
            if (beta1 == 0.0f) x = 0.0f;
            else if (beta1 != 1.0f) x = __fmul_rn(crow[j * p.csC], beta1);
            else x = crow[j * p.csC];
            if (p.alpha == 1.0f) x = __fadd_rn(x, acc[i][j]);
            else x = __fadd_rn(x, __fmul_rn(p.alpha, acc[i][j]));
            if (has_epi) x = simt_bias_act(x, p.bias, p.bias_per_row, p.act, i, n0 + j);
            v[j] = x;
          }
          if (p.csC == 1 && n0 + NC <= p.N && (reinterpret_cast<uintptr_t>(crow) & (4 * NC - 1)) == 0) {
            if constexpr (NC == 4) *reinterpret_cast<float4 *>(crow) = make_float4(v[0], v[1], v[2], v[3]);
            else *reinterpret_cast<float2 *>(crow) = make_float2(v[0], v[1]);
          } else {
#pragma unroll
            for (int j = 0; j < NC; ++j)
              if (n0 + j < p.N) crow[j * p.csC] = v[j];
          }
        }
      }
    }
  }
}

// The same product with B streamed through shared memory by cp.async: thread t copies exactly the 16 bytes (its 4 columns) of
// each k-row it will consume into a private FIFO of SKA_STAGES x SKA_K rows -- no registers hold data in flight and no barrier
// guards it, so ~100 KB per SM are on their way from HBM at any time (the register-only kernel above keeps 16 KB in flight and
// runs at 1.1 TB/s).  Needs unit column stride and 16-byte aligned rows of B (the host checks); same FMA chains, same results.
constexpr int SKA_K = 8, SKA_STAGES = 4;
template <int MT>
__global__ void __launch_bounds__(256, 1)
gemm_skinny_m_async_kernel(const SimtParams<float> p) {
  static_assert(MT % 4 == 0 && MT <= 32, "rows in registers");
  static_assert(SKINNY_KCHUNK % SKA_K == 0, "whole FIFO stages per chunk of A");
  constexpr int64_t KC = 2048 / 4;   // gemm_tiling.nim:310 (a multiple of SKA_K: stages never straddle a kc block)
  LB200_DYN_SMEM(float4, ska_smem);  // [SKA_STAGES][SKA_K][256] float4 of B, then As4[SKINNY_KCHUNK][MT / 4]
  float4 *Bf = ska_smem;
  float4 *As4 = ska_smem + SKA_STAGES * SKA_K * 256;
  float *As = reinterpret_cast<float *>(As4);
  const int tid = threadIdx.x;
  const int64_t nblocks = (p.N + 1023) / 1024;
  const int64_t total = nblocks * p.batch;
  // The CTA's tiles (1024 columns of one problem each) form ONE stream of FIFO stages, SKA_K k-rows each: the copies of the
  // next tile are in flight while this one is multiplied and stored (with K = 27 a tile is only four stages long)
  const int64_t st_per_tile = (p.K + SKA_K - 1) / SKA_K;
  const int64_t my_tiles = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int64_t total_stages = my_tiles * st_per_tile;
  auto issue = [&](int64_t g) {   // one commit group per call (possibly empty)
    if (g < total_stages) {
      const int64_t it = g / st_per_tile, s = g - it * st_per_tile;
      const int64_t t = blockIdx.x + it * gridDim.x;
      const int64_t bi = t / nblocks;
      const int64_t n0 = (t - bi * nblocks) * 1024 + 4 * tid;
      if (n0 < p.N) {
        const uint32_t src_bytes = static_cast<uint32_t>((p.N - n0 < 4 ? p.N - n0 : 4) * 4);   // ragged right edge: zero fill
        const float *Bb = p.B + bi * p.bsB + n0;
        float4 *dst = Bf + ((g % SKA_STAGES) * SKA_K) * 256 + tid;
#pragma unroll
        for (int r = 0; r < SKA_K; ++r) {
          const int64_t k = s * SKA_K + r;
          if (k < p.K) ptx::cp_async_16(dst + r * 256, Bb + k * p.rsB, src_bytes);
        }
      }
    }
    ptx::cp_async_commit();
  };
#pragma unroll
  for (int s = 0; s < SKA_STAGES - 1; ++s) issue(s);
  int64_t g = 0;   // stage being consumed
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int64_t bi = t / nblocks;
    const int64_t n0 = (t - bi * nblocks) * 1024 + 4 * tid;
    const float *Ab = p.A + bi * p.bsA;
    float *Cb = p.C + bi * p.bsC;
    const bool live = n0 < p.N;
    for (int64_t pc = 0; pc < p.K; pc += KC) {  // reference loop 2 (gemm.nim:150)
      const int64_t kend = (pc + KC < p.K) ? pc + KC : p.K;
      float acc[MT][4];
#pragma unroll
      for (int i = 0; i < MT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.0f;
      for (int64_t k0 = pc; k0 < kend; k0 += SKINNY_KCHUNK) {
        const int kn = static_cast<int>(kend - k0 < SKINNY_KCHUNK ? kend - k0 : SKINNY_KCHUNK);
        __syncthreads();   // the previous chunk of A is consumed
        for (int i = tid; i < SKINNY_KCHUNK * MT; i += 256) {
          const int k = i / MT, m = i - k * MT;
          As[i] = (m < p.M && k < kn) ? Ab[m * p.rsA + (k0 + k) * p.csA] : 0.0f;
        }
        __syncthreads();
#pragma unroll 1
        for (int kk = 0; kk < kn; kk += SKA_K, ++g) {
          ptx::cp_async_wait<SKA_STAGES - 2>();   // this thread's copies of stage g have landed (nobody else reads them)
          const float4 *bs = Bf + ((g % SKA_STAGES) * SKA_K) * 256 + tid;
          const int kr = kn - kk < SKA_K ? kn - kk : SKA_K;
          if (live) {
#pragma unroll
            for (int r = 0; r < SKA_K; ++r) {
              if (r < kr) {
                const float4 bv = bs[r * 256];
                const float b[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
                for (int i4 = 0; i4 < MT / 4; ++i4) {
                  const float4 a = As4[(kk + r) * (MT / 4) + i4];
                  const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[4 * i4 + e][j] = __fmaf_rn(av[e], b[j], acc[4 * i4 + e][j]);
                }
              }
            }
          }
          issue(g + SKA_STAGES - 1);   // refill the slot consumed one iteration ago (it may belong to the next tile)
        }
      }
      // reference epilogue for this kc block (gemm_ukernel_generic.nim:53-76)
      const float beta1 = (pc == 0) ? p.beta : 1.0f;
      const bool has_epi = kend == p.K && (p.bias != nullptr || p.act != 0);
      // the common case of the convolution (alpha = 1, beta = 0, nothing fused, whole float4 inside C): 0 + sum, one vector
      // store per row -- a few hundred instructions instead of the general store loop below (instruction-cache footprint)
      const bool plain = beta1 == 0.0f && p.alpha == 1.0f && !has_epi && p.csC == 1 && n0 + 4 <= p.N &&
                         ((reinterpret_cast<uintptr_t>(Cb + n0) | (static_cast<uint64_t>(p.rsC) * 4)) & 15) == 0;
      if (live && plain) {
#pragma unroll
        for (int i = 0; i < MT; ++i) {
          if (i < p.M)
            *reinterpret_cast<float4 *>(Cb + i * p.rsC + n0) =
                make_float4(__fadd_rn(0.0f, acc[i][0]), __fadd_rn(0.0f, acc[i][1]), __fadd_rn(0.0f, acc[i][2]), __fadd_rn(0.0f, acc[i][3]));
        }
      } else if (live) {
#pragma unroll
        for (int i = 0; i < MT; ++i) {
          if (i >= p.M) break;
          float *crow = Cb + i * p.rsC + n0 * p.csC;
          float v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (n0 + j >= p.N) { v[j] = 0.0f; continue; }
            float x;
            if (beta1 == 0.0f) x = 0.0f;
            else if (beta1 != 1.0f) x = __fmul_rn(crow[j * p.csC], beta1);
            else x = crow[j * p.csC];
            if (p.alpha == 1.0f) x = __fadd_rn(x, acc[i][j]);
            else x = __fadd_rn(x, __fmul_rn(p.alpha, acc[i][j]));
            if (has_epi) x = simt_bias_act(x, p.bias, p.bias_per_row, p.act, i, n0 + j);
            v[j] = x;
          }
          if (p.csC == 1 && n0 + 4 <= p.N && (reinterpret_cast<uintptr_t>(crow) & 15) == 0) {
            *reinterpret_cast<float4 *>(crow) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (n0 + j < p.N) crow[j * p.csC] = v[j];
          }
        }
      }
    }
  }
  ptx::cp_async_wait<0>();
}
template <int MT> constexpr size_t ska_smem_bytes() { return (static_cast<size_t>(SKA_STAGES) * SKA_K * 256 + SKINNY_KCHUNK * (MT / 4)) * sizeof(float4); }

// ---------------------------------------------------------------------------
// Direct grouped convolution: the exact path of laser_b200_conv2d_grouped_f32_fused_dev, a convolution on the CUDA cores,
// one launch, no preparation pass and no workspace.
//
// NCHW images [n][C][H][W], filters [Cout][Cg][kH][kW] (torch's grouped weight), G groups of Cg = C / G input and
// Mg = Cout / G output channels.  Output channel co = g * Mg + m of image i:
//   out[i][co] = act(sum_{k < Kg} w[co][k] * im2col(in[i][g * Cg : (g + 1) * Cg])[k] + bias[co]),  Kg = Cg * kH * kW
// Each output is the exact GEMM's chain over the im2col matrix of its group (gemm_simt_kernel.inc), so the path is bit for
// bit the oracle's conv2d_im2col of each group's slice:
//   - one fmaf chain from 0 over k = ci * kH * kW + kh * kW + kw, restarted every KC = 512 k-steps, the block sums added in
//     order (v = 0 + acc_0, v = v + acc_1, ...: the alpha = 1, beta' = 0 then 1 epilogue of the exact kernel);
//   - taps in the padding are fmaf(w, 0, acc), not skipped (the staged patch holds the zeros), so an Inf or NaN filter tap
//     gives NaN wherever the GEMM over the im2col matrix does;
//   - bias and activation through simt_bias_act, the exact kernel's function.
//
// A CTA computes a tile of one image and one group: CG * MC output channels x TY output rows x 4 * XT output columns.
// Thread (cg, ty, tx) owns MC consecutive channels and the 4 pixels tx, tx + XT, tx + 2 XT, tx + 3 XT of row ty: the
// lanes of a warp read consecutive patch words (no bank conflict at unit stride) and store consecutive output words.  For
// each input channel ci of the group the CTA stages in shared memory the zero-padded input rows and columns the tile
// reads, [PR][PC], and the tile's filter taps of ci, [kH * kW][CG * MC] (a thread's MC weights of one tap in one 4-, 8- or
// 16-byte load); the FMAs then read only shared memory.  Depthwise layers (Cg = 1) stage one channel per CTA tile.
//
// GRAD = true: the exact path of laser_b200_conv2d_grouped_input_grad_f32_fused_dev, the same tiles and chains over the
// transposed geometry of the input gradient (capi.cu: conv2d_grouped_input_grad_dev).  `in` is dY, its C = c_out channels
// (Cg = c_out / G per group) zero-dilated by (dH, dW) = the forward strides and padded by kH - 1 - pH (negative: cropped),
// stride 1; `out` is dX, Mg = c_in / G channels per group.  The three differences, each under `if constexpr`:
//   - patch word (h, w) of the dilated plane is op(dY[h / dH][w / dW]) (split.cuh: operand_op, the aux read at dY's offset)
//     when h >= 0, h % dH == 0 and h / dH < H (columns likewise), else 0: a hole is 0, never op(0), and its taps are
//     fmaf(w, 0, acc) as the padding's are;
//   - the taps of source channel co for output channel m are the caller's filters rotated and transposed in place,
//     wts[(g * Cg + co) * Mg * T + m * T + T - 1 - t], T = kH * kW: the rows W'_g of the input gradient, no copy;
//   - the exact kernel's alpha / beta epilogue per KC block (beta1 in gemm_simt_kernel.inc): v starts at 0 (beta = 0: dX
//     not read), dX or dX * beta, and every block adds acc or alpha * acc; no bias, no activation.
// So dX is bit for bit the oracle's gemm_strided(W'_g, rows_{n,g}, alpha, beta) per image and group.
// ---------------------------------------------------------------------------
constexpr int CONV_GROUPED_PX = 4;                 // output pixels per thread, XT apart along a row
constexpr int CONV_GROUPED_THREADS = 256;          // most threads of a CTA
constexpr int CONV_GROUPED_SMEM = 48 * 1024;       // most shared memory of a CTA (no opt-in needed)

struct ConvGroupedParams {
  int64_t images;
  int C, H, W, G, Cg, Mg, kH, kW, pH, pW, sH, sW, outH, outW;
  int XT, TY, CG;                    // threads along a row, rows, channel groups of MC per CTA
  int x_tiles, y_tiles, m_tiles;     // CTA tiles per image and group
  int PR, PC;                        // staged patch: rows, columns
  int64_t tiles;                     // images * G * m_tiles * y_tiles * x_tiles
  const float *bias;
  int act;
};
// the input gradient's (GRAD) parameters: the plan's, and what the caller sets after it -- the source's dilation, the scalars
// and the op on the source (aux laid out like it, NULL: none)
struct ConvGroupedGradParams : ConvGroupedParams {
  int dH, dW;
  float alpha, beta;
  int op;
  const float *aux;
};

// Host side: the tile of a geometry (C, Cout, ... of the whole layer; G groups).  *mc = channels per thread (1, 2 or 4:
// the largest that divides Mg).  Returns the threads of a CTA, or 0 when even a one-row, one-quad tile needs more than
// CONV_GROUPED_SMEM bytes (a kernel window of thousands of taps).  *smem_bytes: the CTA's dynamic shared memory.
inline int conv_grouped_plan(const ConvGeom &g, int64_t G, const float *bias, int act, ConvGroupedParams *p, int *mc,
                             size_t *smem_bytes) {
  p->images = g.B;
  p->C = static_cast<int>(g.C); p->H = static_cast<int>(g.H); p->W = static_cast<int>(g.W);
  p->G = static_cast<int>(G); p->Cg = static_cast<int>(g.C / G); p->Mg = static_cast<int>(g.Cout / G);
  p->kH = static_cast<int>(g.kH); p->kW = static_cast<int>(g.kW); p->pH = static_cast<int>(g.pH); p->pW = static_cast<int>(g.pW);
  p->sH = static_cast<int>(g.sH); p->sW = static_cast<int>(g.sW);
  p->outH = static_cast<int>(g.outH); p->outW = static_cast<int>(g.outW);
  p->bias = bias;
  p->act = act;
  *mc = p->Mg % 4 == 0 ? 4 : p->Mg % 2 == 0 ? 2 : 1;
  const int chans = p->Mg / *mc, taps = p->kH * p->kW;
  const int quads = (p->outW + CONV_GROUPED_PX - 1) / CONV_GROUPED_PX;
  int xt = quads < 32 ? quads : 32;
  int ty_max = CONV_GROUPED_THREADS / xt;
  int cg_max = chans;
  for (;;) {
    p->XT = xt;
    p->x_tiles = (p->outW + CONV_GROUPED_PX * xt - 1) / (CONV_GROUPED_PX * xt);
    const int tym = ty_max < p->outH ? ty_max : p->outH;
    p->y_tiles = (p->outH + tym - 1) / tym;
    p->TY = (p->outH + p->y_tiles - 1) / p->y_tiles;   // rows balanced over the tiles
    int cg = CONV_GROUPED_THREADS / (xt * p->TY);
    if (cg < 1) cg = 1;
    if (cg > cg_max) cg = cg_max;
    p->m_tiles = (chans + cg - 1) / cg;
    p->CG = (chans + p->m_tiles - 1) / p->m_tiles;
    p->PR = (p->TY - 1) * p->sH + p->kH;
    p->PC = (CONV_GROUPED_PX * xt - 1) * p->sW + p->kW;
    const int64_t words = static_cast<int64_t>(taps) * p->CG * *mc + static_cast<int64_t>(p->PR) * p->PC;
    if (words * 4 <= CONV_GROUPED_SMEM) {
      *smem_bytes = static_cast<size_t>(words) * 4;
      break;
    }
    if (p->TY > 1) ty_max = (p->TY + 1) / 2;
    else if (xt > 1) xt = (xt + 1) / 2;
    else if (p->CG > 1) cg_max = (p->CG + 1) / 2;
    else return 0;
  }
  p->tiles = g.B * G * p->m_tiles * p->y_tiles * p->x_tiles;
  return p->XT * p->TY * p->CG;
}

template <int MC, bool GRAD = false>
__global__ void __launch_bounds__(CONV_GROUPED_THREADS)
conv_grouped_direct_kernel(float *__restrict__ out, const float *__restrict__ in, const float *__restrict__ wts,
                           const typename std::conditional<GRAD, ConvGroupedGradParams, ConvGroupedParams>::type p) {
  static_assert(MC == 1 || MC == 2 || MC == 4, "channels per thread");
  constexpr int KC = 512;   // gemm_simt_kernel.inc: 2048 / sizeof(float)
  constexpr int PX = CONV_GROUPED_PX;
  LB200_DYN_SMEM(float4, cg_smem4);
  const int MB = p.CG * MC, taps = p.kH * p.kW;
  float *ws = reinterpret_cast<float *>(cg_smem4);   // [taps][MB]
  float *patch = ws + taps * MB;                      // [PR][PC]
  const int nthr = p.XT * p.TY * p.CG;
  const int tid = threadIdx.x;
  const int cg = tid / (p.XT * p.TY), rem = tid - cg * (p.XT * p.TY);
  const int ty = rem / p.XT, tx = rem - ty * p.XT;
  const int patch_words = p.PR * p.PC;
  const int64_t HW = static_cast<int64_t>(p.H) * p.W;
  for (int64_t t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    int64_t r = t;
    const int xt = static_cast<int>(r % p.x_tiles); r /= p.x_tiles;
    const int yt = static_cast<int>(r % p.y_tiles); r /= p.y_tiles;
    const int mt = static_cast<int>(r % p.m_tiles); r /= p.m_tiles;
    const int g = static_cast<int>(r % p.G);
    const int64_t img = r / p.G;
    const int x0 = xt * PX * p.XT, oh0 = yt * p.TY, m0 = mt * MB;
    const int ih0 = oh0 * p.sH - p.pH, iw0 = x0 * p.sW - p.pW;
    const float *src = in + (img * p.C + static_cast<int64_t>(g) * p.Cg) * HW;
    const float *wsrc = GRAD ? wts + static_cast<int64_t>(g) * p.Cg * p.Mg * taps
                             : wts + (static_cast<int64_t>(g) * p.Mg + m0) * p.Cg * taps;
    float acc[MC][PX], v[MC][PX];
#pragma unroll
    for (int c = 0; c < MC; ++c)
#pragma unroll
      for (int j = 0; j < PX; ++j) { acc[c][j] = 0.0f; v[c][j] = 0.0f; }
    if constexpr (GRAD) {   // beta * dX as the exact kernel's first block takes it (beta = 0: dX is not read)
      const int oh = oh0 + ty;
      if (p.beta != 0.0f && oh < p.outH) {
#pragma unroll
        for (int c = 0; c < MC; ++c) {
          const int m = m0 + cg * MC + c;
          if (m >= p.Mg) continue;
          const float *orow = out + ((img * p.G * p.Mg + static_cast<int64_t>(g) * p.Mg + m) * p.outH + oh) * p.outW;
#pragma unroll
          for (int j = 0; j < PX; ++j) {
            const int ow = x0 + tx + j * p.XT;
            if (ow < p.outW) v[c][j] = p.beta == 1.0f ? orow[ow] : __fmul_rn(orow[ow], p.beta);
          }
        }
      }
    }
    int kc = 0;   // k-steps of the current chain
    for (int ci = 0; ci < p.Cg; ++ci) {
      __syncthreads();   // the previous channel's patch and taps are consumed
      for (int i = tid; i < taps * MB; i += nthr) {
        const int tap = i / MB, mm = i - tap * MB;
        if constexpr (GRAD)   // W'_g: source channel ci's filter for output channel m0 + mm, rotated by 180 degrees
          ws[i] = m0 + mm < p.Mg ? wsrc[(static_cast<int64_t>(ci) * p.Mg + m0 + mm) * taps + (taps - 1 - tap)] : 0.0f;
        else
          ws[i] = m0 + mm < p.Mg ? wsrc[(static_cast<int64_t>(mm) * p.Cg + ci) * taps + tap] : 0.0f;
      }
      const float *sc = src + ci * HW;
      if constexpr (GRAD) {
        const float *ac = p.aux ? p.aux + (sc - in) : nullptr;
        for (int i = tid; i < patch_words; i += nthr) {
          const int pr = i / p.PC, pc = i - pr * p.PC;
          const int h = ih0 + pr, w = iw0 + pc;   // in the dilated plane
          const int hq = h / p.dH, wq = w / p.dW;
          float x = 0.0f;
          if (h >= 0 && w >= 0 && hq * p.dH == h && wq * p.dW == w && hq < p.H && wq < p.W) {
            const int64_t off = static_cast<int64_t>(hq) * p.W + wq;
            x = sc[off];
            if (p.op != 0) x = operand_op(p.op, x, ac ? ac[off] : 0.0f);
          }
          patch[i] = x;
        }
      } else {
        for (int i = tid; i < patch_words; i += nthr) {
          const int pr = i / p.PC, pc = i - pr * p.PC;
          const int ih = ih0 + pr, iw = iw0 + pc;
          patch[i] = (static_cast<unsigned>(ih) < static_cast<unsigned>(p.H) && static_cast<unsigned>(iw) < static_cast<unsigned>(p.W))
                         ? sc[static_cast<int64_t>(ih) * p.W + iw] : 0.0f;
        }
      }
      __syncthreads();
      const float *prow = patch + ty * p.sH * p.PC + tx * p.sW;
      for (int kh = 0; kh < p.kH; ++kh) {
        for (int kw = 0; kw < p.kW; ++kw) {
          if (kc == KC) {   // the exact kernel's next kc block: its sum is added to the previous ones
#pragma unroll
            for (int c = 0; c < MC; ++c)
#pragma unroll
              for (int j = 0; j < PX; ++j) {
                if constexpr (GRAD) v[c][j] = __fadd_rn(v[c][j], p.alpha == 1.0f ? acc[c][j] : __fmul_rn(p.alpha, acc[c][j]));
                else v[c][j] = __fadd_rn(v[c][j], acc[c][j]);
                acc[c][j] = 0.0f;
              }
            kc = 0;
          }
          ++kc;
          const float *wt = ws + (kh * p.kW + kw) * MB + cg * MC;
          float w[MC];
          if constexpr (MC == 4) {
            const float4 q = *reinterpret_cast<const float4 *>(wt);
            w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
          } else if constexpr (MC == 2) {
            const float2 q = *reinterpret_cast<const float2 *>(wt);
            w[0] = q.x; w[1] = q.y;
          } else {
            w[0] = wt[0];
          }
          const float *px = prow + kh * p.PC + kw;
          float x[PX];
#pragma unroll
          for (int j = 0; j < PX; ++j) x[j] = px[j * p.XT * p.sW];
#pragma unroll
          for (int c = 0; c < MC; ++c)
#pragma unroll
            for (int j = 0; j < PX; ++j) acc[c][j] = __fmaf_rn(w[c], x[j], acc[c][j]);
        }
      }
    }
    const int oh = oh0 + ty;
    if (oh < p.outH) {
#pragma unroll
      for (int c = 0; c < MC; ++c) {
        const int m = m0 + cg * MC + c;
        if (m >= p.Mg) continue;
        const int64_t co = static_cast<int64_t>(g) * p.Mg + m;
        float *orow = out + ((img * p.G * p.Mg + co) * p.outH + oh) * p.outW;
#pragma unroll
        for (int j = 0; j < PX; ++j) {
          const int ow = x0 + tx + j * p.XT;
          if (ow >= p.outW) continue;
          if constexpr (GRAD) {
            orow[ow] = __fadd_rn(v[c][j], p.alpha == 1.0f ? acc[c][j] : __fmul_rn(p.alpha, acc[c][j]));
          } else {
            float y = __fadd_rn(v[c][j], acc[c][j]);
            if (p.bias != nullptr || p.act != 0) y = simt_bias_act(y, p.bias, 1, p.act, co, 0);
            orow[ow] = y;
          }
        }
      }
    }
  }
}

}  // namespace lb200
