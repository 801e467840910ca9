// tc_launch_impl.cuh -- the one launcher template behind tc_launch.h (included by tc_*.cu only)
#pragma once

#include <atomic>

#include "gemm_tc.cuh"
#include "tc_launch.h"

// tests/emu compiles this for the host with its own launch function (capi_host_prelude.h)
#ifndef LB200_LAUNCH_EX
#define LB200_LAUNCH_EX cudaLaunchKernelEx
#endif

namespace lb200 {

template <int ESZ, uint32_t FMT16, int NPASS, typename OutT, bool SCALED, bool A_MN, bool B_MN, bool BATCHED>
int launch_tc_one(const TcLaunch &l) {
  using Cfg = TcCfg<NPASS>;
  const int64_t units_total = tc_units(l.p);  // work units
  // persistent: one CTA per SM, never more CTAs than units
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<int>(units_total < l.sm_count ? units_total : l.sm_count));
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = l.stream;
  cudaLaunchAttribute attr[1];
  if (l.pdl) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  auto kfn = gemm_tc_kernel<ESZ, FMT16, NPASS, A_MN, B_MN, OutT, SCALED, BATCHED>;
  static std::atomic<uint32_t> attr_set{0};   // per device: function attributes live in the context
  if (!(attr_set.load(std::memory_order_acquire) & (1u << l.dev))) {
    const cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set.fetch_or(1u << l.dev, std::memory_order_release);
  }
  return static_cast<int>(LB200_LAUNCH_EX(&cfg, kfn, l.a0, l.a1, l.b0, l.b1, l.p));
}

template <int ESZ, uint32_t FMT16, int NPASS, typename OutT, bool SCALED>
int launch_tc_family(const TcLaunch &l) {
  if constexpr (ESZ == 4) {   // wgmma reads tf32 tiles K-major only: capi.cu prepares MN-major fp32 operands K-major
    if (l.a_mn || l.b_mn) return static_cast<int>(cudaErrorNotSupported);
    if (l.batched) return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, false, false, true>(l);
    return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, false, false, false>(l);
  }
#define LB200_MAJORS(BATCHED)                                                                                  \
  do {                                                                                                         \
    if (!l.a_mn && !l.b_mn) return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, false, false, BATCHED>(l);   \
    if (!l.a_mn && l.b_mn) return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, false, true, BATCHED>(l);     \
    if (l.a_mn && !l.b_mn) return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, true, false, BATCHED>(l);     \
    return launch_tc_one<ESZ, FMT16, NPASS, OutT, SCALED, true, true, BATCHED>(l);                             \
  } while (0)
  if constexpr (ESZ == 2) {
    // batched: the fp32 families only (F16X3 here; bf16 has no batched entry)
    if constexpr (SCALED) {
      if (l.batched) LB200_MAJORS(true);
    }
    if (l.batched) return static_cast<int>(cudaErrorNotSupported);
    LB200_MAJORS(false);
  }
#undef LB200_MAJORS
}

}  // namespace lb200
