// tc_f16x3.cu -- the four instantiations (operand major-ness) of gemm_tc_kernel<2, ptx::kFmtF16, 3, ..., float, true>, and
// the four batched ones
#include "tc_launch_impl.cuh"

namespace lb200 {
int launch_tc_f16x3(const TcLaunch &l) { return launch_tc_family<2, ptx::kFmtF16, 3, float, true>(l); }
}  // namespace lb200
