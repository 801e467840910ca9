// tc_launch.h -- host-side launchers of gemm_tc_kernel, one translation unit per kernel family (tc_*.cu) so that the
// library builds in parallel; capi.cu sees only this header (it never instantiates the kernel).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include "tc_params.h"

namespace lb200 {

struct TcLaunch {
  CUtensorMap a0, a1, b0, b1;   // piece 0 (hi / the operand itself) and piece 1 (lo) of A and B
  TcParams p;
  bool a_mn = false, b_mn = false;   // operand major-ness
  bool pair = false;                 // clusters of two CTAs sharing one tile scheduler
  bool batched = false;              // p.batch problems, rank-3 tensor maps (fp32 families, single CTAs: tc_params.h)
  bool pdl = false;                  // programmatic dependent launch: overlap the prologue with the preceding kernel's tail
  int dev = 0, sm_count = 0;
  cudaStream_t stream = nullptr;
};

// each returns a cudaError_t value (0 = launched)
int launch_tc_tf32x1(const TcLaunch &l);   // fp32 in/out, wgmma tf32, one pass (the tensor core ignores the low mantissa bits)
int launch_tc_tf32x3(const TcLaunch &l);   // fp32 in/out, wgmma tf32, hi/lo pieces, three passes
int launch_tc_bf16(const TcLaunch &l);     // bf16 in/out, wgmma bf16
int launch_tc_f16x3(const TcLaunch &l);    // two fp16 pieces of the scaled fp32 operands, three passes, fp32 out (default fp32 mode)

}  // namespace lb200
