// prologue_emu.cpp -- TEST INFRASTRUCTURE: the prologue-fusion (HAS_OP = true) instantiations of the operand-preparation
// kernels of laser_b200/csrc/split.cuh compiled for the host (cuda_emu.h) behind a C interface for ctypes.  Aux element
// (r, c) of the kernel's [R][Cc] view is read at aux[r * aux_sr + c * aux_sc] (the row kernels: aux_sc = 1).
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

static OperandOp make_op(int op, const float *aux, int64_t aux_sr, int64_t aux_sc) {
  OperandOp o;
  o.op = op; o.aux = aux; o.aux_sr = aux_sr; o.aux_sc = aux_sc;
  return o;
}

extern "C" {

void emu_op_split_rows_tf32(int op, const float *aux, int64_t aux_ld, const float *src, int64_t R, int64_t Cc, int64_t src_ld,
                            float *hi, float *lo, int64_t dst_ld, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  emu::launch(grid, 256, [=]() { split_rows_tf32_kernel<true>(src, R, Cc, src_ld, hi, lo, dst_ld, o); });
}
// K-major operand, one scale per row: group = 32 (a warp per row) or 256 (the CTA)
void emu_op_f16x2_rows_fused(int group, int op, const float *aux, int64_t aux_ld, const float *src, int64_t R, int64_t Cc,
                             int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b, uint32_t *absmax, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  if (group == 32) emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<32, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o); });
  else emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<256, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o); });
}
// MN-major operand: one abs-max word per column, then the split
void emu_op_absmax_cols(int op, const float *aux, int64_t aux_ld, const float *src, int64_t R, int64_t Cc, int64_t src_ld,
                        uint32_t *out, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  emu::launch(grid, 256, [=]() { absmax_mn_kernel<true, true>(src, R, Cc, src_ld, out, o); });
}
void emu_op_split_cols_f16x2(int op, const float *aux, int64_t aux_ld, const float *src, int64_t R, int64_t Cc, int64_t src_ld,
                             uint16_t *hb, uint16_t *lb, int64_t ld_b, const uint32_t *absmax, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  emu::launch(grid, 256, [=]() { split_rows_f16x2_kernel<true, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o); });
}
// mode 0: copy, 1: tf32 hi/lo
void emu_op_pack_general_f32(int mode, int op, const float *aux, int64_t aux_sr, int64_t aux_sc, const float *src, int64_t R,
                             int64_t Cc, int64_t sr, int64_t sc, float *dst, float *dst_lo, int64_t ld, int read_along_r, int grid) {
  const OperandOp o = make_op(op, aux, aux_sr, aux_sc);
  if (mode == 0)
    emu::launch(grid, 256, [=]() { pack_general_kernel<float, 0, true>(src, R, Cc, sr, sc, dst, dst_lo, ld, read_along_r, o); });
  else
    emu::launch(grid, 256, [=]() { pack_general_kernel<float, 1, true>(src, R, Cc, sr, sc, dst, dst_lo, ld, read_along_r, o); });
}

}  // extern "C"
