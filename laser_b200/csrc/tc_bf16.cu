// tc_bf16.cu -- the eight instantiations (operand major-ness x single CTA / cluster of two) of gemm_tc_kernel<2, ptx::kFmtBF16, 1, uint16_t, false>
#include "tc_launch_impl.cuh"

namespace lb200 {
int launch_tc_bf16(const TcLaunch &l) { return launch_tc_family<2, ptx::kFmtBF16, 1, uint16_t, false>(l); }
}  // namespace lb200
