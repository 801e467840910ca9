// conv_input_grad_emu.cpp -- TEST INFRASTRUCTURE: the transposed im2col source of laser_b200/csrc/split.cuh
// (im2col_rows_kernel with DIL / HAS_OP over an Im2colGradSrc, every mode and group) compiled for the host (cuda_emu.h) behind
// a C interface for ctypes, and the library's operand op element by element.  The row kernels it must reproduce are in
// conv_emu.cpp.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

extern "C" {

// geom = the FORWARD call's {C, H, W, kH, kW, pH, pW, sH, sW, c_out}; dy: [images][c_out][outH][outW]; the rows are the input
// pixels' transposed windows (capi.cu: conv2d_input_grad_dev builds the same geometry).  dil: the DIL instantiation (it must
// be 1 when the strides are not 1); op / aux: HAS_OP when op != 0.
void emu_tconv_rows(int mode, int group, int dil, int op, const float *dy, const float *aux, const int64_t *geom, int64_t images,
                    float *dst, float *dst_lo, uint16_t *hb, uint16_t *lb, int64_t ld, uint32_t *absmax, int grid) {
  const int64_t C = geom[0], H = geom[1], W = geom[2], kH = geom[3], kW = geom[4], pH = geom[5], pW = geom[6], sH = geom[7],
                sW = geom[8], Cout = geom[9];
  ConvGeom g{};
  g.B = images; g.C = Cout; g.Cout = C; g.kH = kH; g.kW = kW;
  g.H = 1 + (H + 2 * pH - kH) / sH;
  g.W = 1 + (W + 2 * pW - kW) / sW;
  g.pH = kH - 1 - pH; g.pW = kW - 1 - pW;
  g.sH = g.sW = 1;
  g.outH = H; g.outW = W;
  Im2colGradSrc q{};
  static_cast<Im2colSrc &>(q) = im2col_src(g);
  q.dH = static_cast<int>(sH);
  q.dW = static_cast<int>(sW);
  q.op.op = op;
  q.op.aux = aux;
#define EMU_TCONV(MODE, GROUP, DIL, HAS_OP) \
  emu::launch(grid, 256, [=]() { im2col_rows_kernel<MODE, GROUP, DIL, HAS_OP>(dy, q, images, dst, dst_lo, hb, lb, ld, absmax); })
#define EMU_TCONV_FLAGS(MODE, GROUP)                                   \
  do {                                                                 \
    if (dil && op) EMU_TCONV(MODE, GROUP, true, true);                 \
    else if (dil) EMU_TCONV(MODE, GROUP, true, false);                 \
    else EMU_TCONV(MODE, GROUP, false, true);                          \
  } while (0)
#define EMU_TCONV_GROUP(MODE) \
  do { if (group == 32) EMU_TCONV_FLAGS(MODE, 32); else EMU_TCONV_FLAGS(MODE, 256); } while (0)
  if (mode == IM2COL_F32) EMU_TCONV_GROUP(IM2COL_F32);
  else if (mode == IM2COL_TF32) EMU_TCONV_GROUP(IM2COL_TF32);
  else EMU_TCONV_GROUP(IM2COL_F16X2);
#undef EMU_TCONV_GROUP
#undef EMU_TCONV_FLAGS
#undef EMU_TCONV
}

// out[i] = the library's operand op (split.cuh: operand_op) of x[i] with aux y[i] (y NULL: 0)
void emu_operand_op(int op, const float *x, const float *y, int64_t n, float *out) {
  for (int64_t i = 0; i < n; ++i) out[i] = operand_op(op, x[i], y ? y[i] : 0.0f);
}

}  // extern "C"
