// conv_nhwc_emu.cpp -- TEST INFRASTRUCTURE: the channels-last im2col source of laser_b200/csrc/split.cuh (im2col_rows_kernel
// with NHWC over an Im2colNhwcSrc, every mode and group) compiled for the host (cuda_emu.h) behind a C interface for ctypes.
// The row kernels it must reproduce are in conv_emu.cpp.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

// geom = {C, H, W, kH, kW, pH, pW, sH, sW}; in: [images][H][W][C]; the rows are the output pixels' windows in (kh, kw, c)
// order, [images * outH * outW][ld].  Returns the source's vec flag (split.cuh: im2col_nhwc_src decides it as the library does).
int emu_nhwc_rows(int mode, int group, const float *in, const int64_t *geom, int64_t images, float *dst, float *dst_lo,
                  uint16_t *hb, uint16_t *lb, int64_t ld, uint32_t *absmax, int grid) {
  ConvGeom g{};
  g.B = images; g.C = geom[0]; g.H = geom[1]; g.W = geom[2]; g.kH = geom[3]; g.kW = geom[4];
  g.pH = geom[5]; g.pW = geom[6]; g.sH = geom[7]; g.sW = geom[8];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  g.nhwc = true;
  const Im2colNhwcSrc q = im2col_nhwc_src(g, in);
#define EMU_NHWC(MODE, GROUP)                                                                                              \
  emu::launch(grid, 256, [=]() {                                                                                           \
    im2col_rows_kernel<MODE, GROUP, false, false, true>(in, q, images, dst, dst_lo, hb, lb, ld, absmax);                 \
  })
  if (mode == IM2COL_F32) { if (group == 32) EMU_NHWC(IM2COL_F32, 32); else EMU_NHWC(IM2COL_F32, 256); }
  else if (mode == IM2COL_TF32) { if (group == 32) EMU_NHWC(IM2COL_TF32, 32); else EMU_NHWC(IM2COL_TF32, 256); }
  else { if (group == 32) EMU_NHWC(IM2COL_F16X2, 32); else EMU_NHWC(IM2COL_F16X2, 256); }
#undef EMU_NHWC
  return q.vec;
}

}  // extern "C"
