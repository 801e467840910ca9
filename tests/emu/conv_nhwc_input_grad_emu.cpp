// conv_nhwc_input_grad_emu.cpp -- TEST INFRASTRUCTURE: the channels-last transposed im2col source of laser_b200/csrc/split.cuh
// (im2col_rows_kernel with NHWC and DIL / HAS_OP over an Im2colNhwcGradSrc, every mode and group; without either, the NHWC
// forward instantiation the library runs at stride 1 without op) compiled for the host (cuda_emu.h) behind a C interface for
// ctypes.  The row kernels it must reproduce are in conv_emu.cpp.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

// geom = the FORWARD call's {C, H, W, kH, kW, pH, pW, sH, sW, c_out}; dy: NHWC [images][outH][outW][c_out]; the rows are the
// input pixels' transposed windows in (kh', kw', co) order, [images * H * W][ld] (capi.cu: conv2d_nhwc_input_grad_dev builds
// the same geometry).  dil: the DIL instantiation (the library takes it when the strides are not 1); op / aux: HAS_OP when
// op != 0.  Returns the source's vec flag, decided as the library's im2col_rows decides it.
int emu_nhwc_tconv_rows(int mode, int group, int dil, int op, const float *dy, const float *aux, const int64_t *geom,
                        int64_t images, float *dst, float *dst_lo, uint16_t *hb, uint16_t *lb, int64_t ld, uint32_t *absmax,
                        int grid) {
  const int64_t C = geom[0], H = geom[1], W = geom[2], kH = geom[3], kW = geom[4], pH = geom[5], pW = geom[6], sH = geom[7],
                sW = geom[8], Cout = geom[9];
  ConvGeom g{};
  g.B = images; g.C = Cout; g.Cout = C; g.kH = kH; g.kW = kW;
  g.H = 1 + (H + 2 * pH - kH) / sH;
  g.W = 1 + (W + 2 * pW - kW) / sW;
  g.pH = kH - 1 - pH; g.pW = kW - 1 - pW;
  g.sH = g.sW = 1;
  g.dH = sH; g.dW = sW;
  g.outH = H; g.outW = W;
  g.nhwc = true;
  Im2colNhwcGradSrc q{};
  static_cast<Im2colNhwcSrc &>(q) = im2col_nhwc_src(g, dy);
  q.vec = q.vec && (!op || !aux || (reinterpret_cast<uintptr_t>(aux) & 15) == 0);
  q.dH = static_cast<int>(sH);
  q.dW = static_cast<int>(sW);
  q.op.op = op;
  q.op.aux = aux;
  const Im2colNhwcSrc fq = q;   // (the forward source: no dilation, no op)
#define EMU_T(MODE, GROUP, DIL, HAS_OP) \
  emu::launch(grid, 256, [=]() { im2col_rows_kernel<MODE, GROUP, DIL, HAS_OP, true>(dy, q, images, dst, dst_lo, hb, lb, ld, absmax); })
#define EMU_T_FLAGS(MODE, GROUP)                                                                                                     \
  do {                                                                                                                               \
    if (dil && op) EMU_T(MODE, GROUP, true, true);                                                                                   \
    else if (dil) EMU_T(MODE, GROUP, true, false);                                                                                   \
    else if (op) EMU_T(MODE, GROUP, false, true);                                                                                    \
    else emu::launch(grid, 256, [=]() {                                                                                              \
      im2col_rows_kernel<MODE, GROUP, false, false, true>(dy, fq, images, dst, dst_lo, hb, lb, ld, absmax);                          \
    });                                                                                                                              \
  } while (0)
#define EMU_T_GROUP(MODE) \
  do { if (group == 32) EMU_T_FLAGS(MODE, 32); else EMU_T_FLAGS(MODE, 256); } while (0)
  if (mode == IM2COL_F32) EMU_T_GROUP(IM2COL_F32);
  else if (mode == IM2COL_TF32) EMU_T_GROUP(IM2COL_TF32);
  else EMU_T_GROUP(IM2COL_F16X2);
#undef EMU_T_GROUP
#undef EMU_T_FLAGS
#undef EMU_T
  return q.vec;
}

}  // extern "C"
