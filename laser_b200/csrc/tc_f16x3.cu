// tc_f16x3.cu -- the eight instantiations (operand major-ness x single CTA / cluster of two) of
// gemm_tc_kernel<2, ptx::kFmtF16, 3, float, true>, and the four of gemm_tc_batched_kernel (operand major-ness)
#include "tc_launch_impl.cuh"

namespace lb200 {
int launch_tc_f16x3(const TcLaunch &l) { return launch_tc_family<2, ptx::kFmtF16, 3, float, true>(l); }
}  // namespace lb200
