// split_emu.cpp -- TEST INFRASTRUCTURE: the operand-preparation kernels of
// laser_b200/csrc/split.cuh (split_rows_tf32 / f16x2 preparation / pack_general / splitk_reduce /
// fill_uniform) compiled for the host (cuda_emu.h; cvt.rna.tf32 replaced by its software
// definition) behind a C interface for ctypes.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

void emu_split_rows_tf32(const float *src, int64_t R, int64_t Cc, int64_t src_ld, float *hi, float *lo, int64_t dst_ld,
                         int grid) {
  emu::launch(grid, 256, [=]() { split_rows_tf32_kernel(src, R, Cc, src_ld, hi, lo, dst_ld); });
}
// per_col 0: one abs-max word per row (K-major operand), 1: one per column (MN-major operand)
int emu_f16x2_rows_ring(const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
                        uint32_t *absmax, int grid) {
  if (!f16x2_rows_ring_ok(src, Cc, src_ld) || f16x2_rows_ring_smem(Cc) > emu::kDynSmemBytes) return 0;   // capi.cu: f16x2_prepare
  emu::reset_state();
  emu::launch(grid, 256, [=]() { f16x2_rows_ring_kernel(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
  return 1;
}
void emu_absmax_mn(int per_col, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint32_t *out, int grid) {
  if (per_col) emu::launch(grid, 256, [=]() { absmax_mn_kernel<true>(src, R, Cc, src_ld, out); });
  else emu::launch(grid, 256, [=]() { absmax_mn_kernel<false>(src, R, Cc, src_ld, out); });
}
void emu_split_rows_f16x2(int per_col, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb,
                          int64_t ld_b, const uint32_t *absmax, int grid) {
  if (per_col) emu::launch(grid, 256, [=]() { split_rows_f16x2_kernel<true>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
  else emu::launch(grid, 256, [=]() { split_rows_f16x2_kernel<false>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
}
// fused single-pass preparation of a K-major operand (one scale per row): group = 32 (a warp per row) or 256 (the CTA)
void emu_f16x2_rows_fused(int group, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb,
                          int64_t ld_b, uint32_t *absmax, int grid) {
  if (group == 32) emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<32>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
  else emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<256>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
}
// mode 0: copy, 1: tf32 hi/lo
void emu_pack_general_f32(int mode, const float *src, int64_t R, int64_t Cc, int64_t sr, int64_t sc, float *dst,
                          float *dst_lo, int64_t ld, int read_along_r, int grid) {
  if (mode == 0) emu::launch(grid, 256, [=]() { pack_general_kernel<float, 0>(src, R, Cc, sr, sc, dst, dst_lo, ld, read_along_r); });
  else emu::launch(grid, 256, [=]() { pack_general_kernel<float, 1>(src, R, Cc, sr, sc, dst, dst_lo, ld, read_along_r); });
}
void emu_pack_general_u16(const uint16_t *src, int64_t R, int64_t Cc, int64_t sr, int64_t sc, uint16_t *dst, int64_t ld,
                          int read_along_r, int grid) {
  emu::launch(grid, 256, [=]() { pack_general_kernel<uint16_t, 0>(src, R, Cc, sr, sc, dst, nullptr, ld, read_along_r); });
}
void emu_splitk_tail_reduce(const float *ws, int S, int n_tail, int n_direct, int num_m, int num_n, int raster_g,
                            int64_t M, int64_t N, float alpha, float beta, float *C, int64_t rsC, int64_t csC, const float *bias,
                            int bias_per_row, int act, int grid) {
  emu::launch(grid, 256, [=]() {
    splitk_tail_reduce_kernel(ws, S, n_tail, n_direct, num_m, num_n, raster_g, M, N, alpha, beta, C, rsC, csC, bias,
                              bias_per_row, act);
  });
}
void emu_fill_uniform_f32(float *dst, int64_t n, uint64_t seed, float lo, float hi, int grid) {
  emu::launch(grid, 256, [=]() { fill_uniform_f32_kernel(dst, n, seed, lo, hi); });
}

}  // extern "C"
