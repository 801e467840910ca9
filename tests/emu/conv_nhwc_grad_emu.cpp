// conv_nhwc_grad_emu.cpp -- TEST INFRASTRUCTURE: the channels-last tap-row preparation kernel of laser_b200/csrc/split.cuh
// (im2col_nhwc_tap_rows_kernel, every mode; F16X2 as the host runs it: the abs-max pass, then the split pass) compiled for the
// host (cuda_emu.h) behind a C interface for ctypes.  The row kernels it must reproduce are in conv_emu.cpp.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

// geom = {C, H, W, kH, kW, pH, pW, sH, sW}; in: [images][H][W][C]; the rows are the taps in (kh, kw, c) order, [K][ld] over the
// pixels of every image end to end.  mode: IM2COL_*; absmax: K words, zeroed by the caller (F16X2).  Returns the source's vec
// flag (split.cuh: im2col_nhwc_src decides it as the library does).
int emu_nhwc_tap_rows(int mode, const float *in, const int64_t *geom, int64_t images, float *dst, float *dst_lo, uint16_t *hb,
                      uint16_t *lb, int64_t ld, uint32_t *absmax, int grid) {
  ConvGeom g{};
  g.B = images; g.C = geom[0]; g.H = geom[1]; g.W = geom[2]; g.kH = geom[3]; g.kW = geom[4];
  g.pH = geom[5]; g.pW = geom[6]; g.sH = geom[7]; g.sW = geom[8];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  g.nhwc = g.taps = true;
  const Im2colNhwcSrc q = im2col_nhwc_src(g, in);
  if (mode == IM2COL_F32) {
    emu::launch(grid, 256, [=]() { im2col_nhwc_tap_rows_kernel<IM2COL_F32>(in, q, images, dst, dst_lo, hb, lb, ld, absmax); });
  } else if (mode == IM2COL_TF32) {
    emu::launch(grid, 256, [=]() { im2col_nhwc_tap_rows_kernel<IM2COL_TF32>(in, q, images, dst, dst_lo, hb, lb, ld, absmax); });
  } else {
    emu::launch(grid, 256, [=]() { im2col_nhwc_tap_rows_kernel<IM2COL_F16X2, true>(in, q, images, dst, dst_lo, hb, lb, ld, absmax); });
    emu::launch(grid, 256, [=]() { im2col_nhwc_tap_rows_kernel<IM2COL_F16X2>(in, q, images, dst, dst_lo, hb, lb, ld, absmax); });
  }
  return q.vec;
}

// the ABSMAX pass alone (words zeroed by the caller)
void emu_nhwc_tap_absmax(const float *in, const int64_t *geom, int64_t images, int64_t ld, uint32_t *absmax, int grid) {
  ConvGeom g{};
  g.B = images; g.C = geom[0]; g.H = geom[1]; g.W = geom[2]; g.kH = geom[3]; g.kW = geom[4];
  g.pH = geom[5]; g.pW = geom[6]; g.sH = geom[7]; g.sW = geom[8];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  g.nhwc = g.taps = true;
  const Im2colNhwcSrc q = im2col_nhwc_src(g, in);
  emu::launch(grid, 256, [=]() {
    im2col_nhwc_tap_rows_kernel<IM2COL_F16X2, true>(in, q, images, nullptr, nullptr, nullptr, nullptr, ld, absmax);
  });
}

}  // extern "C"
