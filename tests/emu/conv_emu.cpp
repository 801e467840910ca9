// conv_emu.cpp -- TEST INFRASTRUCTURE: the im2col-source preparation kernel of laser_b200/csrc/split.cuh
// (im2col_rows_kernel, every mode and group) and the two row kernels whose output it must reproduce bit for bit
// (f16x2_rows_fused_kernel, split_rows_tf32_kernel) compiled for the host (cuda_emu.h) behind a C interface for ctypes.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

// geom = {C, H, W, kH, kW, pH, pW, sH, sW}; mode: IM2COL_*; outputs as split.cuh describes
void emu_im2col_rows(int mode, int group, const float *in, const int64_t *geom, int64_t images, float *dst, float *dst_lo,
                     uint16_t *hb, uint16_t *lb, int64_t ld, uint32_t *absmax, int grid) {
  ConvGeom g{};
  g.B = images; g.C = geom[0]; g.H = geom[1]; g.W = geom[2]; g.kH = geom[3]; g.kW = geom[4];
  g.pH = geom[5]; g.pW = geom[6]; g.sH = geom[7]; g.sW = geom[8];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  const Im2colSrc q = im2col_src(g);
#define EMU_IM2COL(MODE, GROUP) \
  emu::launch(grid, 256, [=]() { im2col_rows_kernel<MODE, GROUP>(in, q, images, dst, dst_lo, hb, lb, ld, absmax); })
  if (mode == IM2COL_F32) { if (group == 32) EMU_IM2COL(IM2COL_F32, 32); else EMU_IM2COL(IM2COL_F32, 256); }
  else if (mode == IM2COL_TF32) { if (group == 32) EMU_IM2COL(IM2COL_TF32, 32); else EMU_IM2COL(IM2COL_TF32, 256); }
  else { if (group == 32) EMU_IM2COL(IM2COL_F16X2, 32); else EMU_IM2COL(IM2COL_F16X2, 256); }
#undef EMU_IM2COL
}
void emu_f16x2_rows(int group, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
                    uint32_t *absmax, int grid) {
  if (group == 32)
    emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<32>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
  else
    emu::launch(grid, 256, [=]() { f16x2_rows_fused_kernel<256>(src, R, Cc, src_ld, hb, lb, ld_b, absmax); });
}
void emu_tf32_rows(const float *src, int64_t R, int64_t Cc, int64_t src_ld, float *hi, float *lo, int64_t ld, int grid) {
  emu::launch(grid, 256, [=]() { split_rows_tf32_kernel<>(src, R, Cc, src_ld, hi, lo, ld); });
}

}  // extern "C"
