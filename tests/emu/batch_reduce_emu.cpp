// batch_reduce_emu.cpp -- TEST INFRASTRUCTURE: the CONCAT instantiations of the operand-preparation kernels of
// laser_b200/csrc/split.cuh (with an op: op 0 is the identity) compiled for the host (cuda_emu.h) behind a C interface for
// ctypes.  n problems bs elements apart, their aux aux_bs apart, concatenated along k as split.cuh describes.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

static OperandOp make_op(int op, const float *aux, int64_t aux_sr, int64_t aux_sc) {
  OperandOp o;
  o.op = op; o.aux = aux; o.aux_sr = aux_sr; o.aux_sc = aux_sc;
  return o;
}
static Batch make_batch(int64_t n, int64_t bs, int64_t aux_bs) {
  Batch b;
  b.n = n; b.bs = bs; b.aux_bs = aux_bs;
  return b;
}

extern "C" {

// K-major: row r of [R][n * Cc] is the problems' rows r end to end
void emu_c_split_rows_tf32(int op, const float *aux, int64_t aux_ld, int64_t aux_bs, const float *src, int64_t R, int64_t Cc,
                           int64_t src_ld, int64_t bs, int64_t n, float *hi, float *lo, int64_t dst_ld, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  const Batch b = make_batch(n, bs, aux_bs);
  emu::launch(grid, 256, [=]() { split_rows_tf32_kernel<true, true, true>(src, R, Cc, src_ld, hi, lo, dst_ld, o, b); });
}
void emu_c_f16x2_rows_fused(int group, int op, const float *aux, int64_t aux_ld, int64_t aux_bs, const float *src, int64_t R,
                            int64_t Cc, int64_t src_ld, int64_t bs, int64_t n, uint16_t *hb, uint16_t *lb, int64_t ld_b,
                            uint32_t *absmax, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  const Batch b = make_batch(n, bs, aux_bs);
  if (group == 32)
    emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<32, true, true, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o, b); });
  else
    emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<256, true, true, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o, b); });
}
// MN-major: rows stacked [n * R][Cc], one word per column over every problem
void emu_c_absmax_cols(int op, const float *aux, int64_t aux_ld, int64_t aux_bs, const float *src, int64_t R, int64_t Cc,
                       int64_t src_ld, int64_t bs, int64_t n, uint32_t *out, int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  const Batch b = make_batch(n, bs, aux_bs);
  emu::launch(grid, 256, [=]() { absmax_mn_kernel<true, true, true, true>(src, R, Cc, src_ld, out, o, b); });
}
void emu_c_split_cols_f16x2(int op, const float *aux, int64_t aux_ld, int64_t aux_bs, const float *src, int64_t R, int64_t Cc,
                            int64_t src_ld, int64_t bs, int64_t n, uint16_t *hb, uint16_t *lb, int64_t ld_b, const uint32_t *absmax,
                            int grid) {
  const OperandOp o = make_op(op, aux, aux_ld, 1);
  const Batch b = make_batch(n, bs, aux_bs);
  emu::launch(grid, 256, [=]() { split_rows_f16x2_kernel<true, true, true, true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax, o, b); });
}
// the gather, problem b to columns b * Cc ..; mode 0: copy, 1: tf32 hi/lo
void emu_c_pack_general_f32(int mode, int op, const float *aux, int64_t aux_sr, int64_t aux_sc, int64_t aux_bs, const float *src,
                            int64_t R, int64_t Cc, int64_t sr, int64_t sc, int64_t bs, int64_t n, float *dst, float *dst_lo, int64_t ld,
                            int grid) {
  const OperandOp o = make_op(op, aux, aux_sr, aux_sc);
  const Batch b = make_batch(n, bs, aux_bs);
  if (mode == 0)
    emu::launch(grid, 256, [=]() { pack_general_kernel<float, 0, true, true, true>(src, R, Cc, sr, sc, dst, dst_lo, ld, 0, o, b); });
  else
    emu::launch(grid, 256, [=]() { pack_general_kernel<float, 1, true, true, true>(src, R, Cc, sr, sc, dst, dst_lo, ld, 0, o, b); });
}

}  // extern "C"
