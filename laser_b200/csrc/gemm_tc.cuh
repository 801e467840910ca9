// gemm_tc.cuh -- the wgmma / TMA strided GEMM for sm_90a (ONE kernel template).
//
// What it replaces in the reference (mratsim/laser, paths relative to
// laser/primitives/matrix_multiplication/):
//   pack_A_mc_kc / pack_B_kc_nc (gemm_packing.nim:24-94)  -> TMA tensor maps: the
//       copy engine resolves the operand's strides and lands 128-byte-swizzled
//       tiles in shared memory; no packing buffers exist.
//   gebb_ukernel register micro-kernel (gemm_ukernel_generator.nim:140-250)
//       -> wgmma.mma_async (tf32 / f16 / bf16) issued by two consumer warpgroups per CTA, each
//       owning 64 rows x 128 columns of the 128 x 128 output tile, accumulators in registers.
//   gemm_impl loop pc (gemm.nim:150-158: K is cut in kc blocks, every block's partial
//       product is ADDED to C in fp32) -> K is cut in accumulation blocks of `kb_per_block`
//       k-tiles: the tensor core accumulates one block in the wgmma accumulator registers, which
//       are then added (IEEE round-to-nearest FADD) to running sums held in other registers.
//       This matters numerically: the tensor core's own accumulation does not round to nearest,
//       so long chains must not live in the accumulator.
//   gebp_mkernel loops jr/ir + loop ic (gemm.nim:48-176; `omp for` over ic blocks)
//       -> persistent CTAs (or clusters of two CTAs on neighbouring 128-row blocks of one
//       256 x 128 tile) that DRAW output tiles from an atomic counter in device memory (a scheduler
//       thread per cluster publishes the unit through shared memory / DSMEM): tiles go to whichever
//       CTA is free, so SMs that start late (another kernel -- e.g. the NCCL broadcast of the
//       row-sharded driver -- still holds them) or run slower simply take fewer tiles.
//   epilogues (gemm_ukernel_generic.nim:53-126)
//       -> alpha/beta in fp32 from the running sums; beta == 0 never reads C; optional fused
//       bias + activation (the reference's TODO at gemm.nim:196).
//
// Warp roles (384 threads): warp 0 lane 0 issues the TMA loads into a ring of stages, warp 3 lane 0 of the
// leader CTA runs the tile scheduler, warpgroups 1 and 2 issue the MMAs and store their rows of C.
//
// Template parameters:
//   ESZ     element size of the tiles (4: fp32 containers read as tf32, 2: 16-bit)
//   FMT16   ptx::kFmtBF16 or ptx::kFmtF16 (ESZ == 2)
//   NPASS   1: one MMA pass over (A, B).  3: fp32-faithful product of two-piece operands
//           x = hi + lo: per k-tile the stage holds FOUR tiles (A_hi, A_lo, B_hi, B_lo), each loaded
//           ONCE, and feeds three passes hi*lo', lo*hi', hi*hi'
//   A_MN/B_MN operand major-ness (wgmma reads K-major and MN-major 16-bit tiles natively, so A^T*B,
//           A*B^T ... need no data movement; tf32 tiles must be K-major)
//   OutT    float or uint16_t (bf16 bits)
//   PAIR    clusters of 2 CTAs; CTA rank r owns rows [128r, 128r+128) of the 256-row tile
//   SCALED  F16X3 mode: the operands are fp16 pieces of A's rows / B's columns scaled by powers of
//           two (f16_scale.cuh); the epilogue multiplies output (i, j) by 2^-sA[i] * 2^-sB[j]
// gemm_tc_batched_kernel runs p.batch problems in one launch (tc_params.h), single CTAs only: rank-3 tensor maps {inner, outer,
// problem} with a box depth of 1, so that TMA zero-fills past M, N and K within each problem.  Both kernels share one body
// (gemm_tc_body.inc), compiled with the constant BATCHED false or true.
#pragma once

#include <type_traits>

#include "f16_scale.cuh"
#include "ptx.cuh"
#include "tc_params.h"

namespace lb200 {

// (out of line: inlined into the unrolled stores the tanhf / expf bodies would multiply the kernel's code size, and the
// consumer warps would miss the instruction cache on every tile)
#ifndef LB200_HOST_EMULATION
static __device__ __noinline__ float epi_act(float v, int act) {
#else
inline float epi_act(float v, int act) {
#endif
  if (act == 1) return fmaxf(v, 0.0f);
  if (act == 2) return tanhf(v);
  if (act == 3) return 1.0f / (1.0f + expf(-v));
  return v;
}

__device__ __forceinline__ float bf16_bits_to_f32(uint16_t h) {
  return __uint_as_float(static_cast<uint32_t>(h) << 16);
}
__device__ __forceinline__ uint16_t f32_to_bf16_bits(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}

// Tensor maps of the kernel: piece 0 (hi, or the operand itself) and piece 1 (lo; unused when NPASS == 1)
template <int ESZ, uint32_t FMT16, int NPASS, bool A_MN, bool B_MN, typename OutT, bool PAIR, bool SCALED>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
               const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1,
               const TcParams p) {
  constexpr bool BATCHED = false;
#include "gemm_tc_body.inc"
}
template <int ESZ, uint32_t FMT16, int NPASS, bool A_MN, bool B_MN, typename OutT, bool SCALED>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_batched_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                       const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1,
                       const TcParams p) {
  constexpr bool PAIR = false, BATCHED = true;
#include "gemm_tc_body.inc"
}

}  // namespace lb200
