// tc_tf32x3.cu -- the instantiation (K-major operands) of gemm_tc_kernel<4, ptx::kFmtBF16, 3, ..., float, false>, and the
// batched one
#include "tc_launch_impl.cuh"

namespace lb200 {
int launch_tc_tf32x3(const TcLaunch &l) { return launch_tc_family<4, ptx::kFmtBF16, 3, float, false>(l); }
}  // namespace lb200
