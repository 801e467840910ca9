// tc_tf32x1.cu -- the two instantiations (K-major operands x single CTA / cluster of two) of gemm_tc_kernel<4, ptx::kFmtBF16, 1, float, false>,
// and gemm_tc_batched_kernel
#include "tc_launch_impl.cuh"

namespace lb200 {
int launch_tc_tf32x1(const TcLaunch &l) { return launch_tc_family<4, ptx::kFmtBF16, 1, float, false>(l); }
}  // namespace lb200
