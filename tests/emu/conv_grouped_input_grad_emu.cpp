// conv_grouped_input_grad_emu.cpp -- TEST INFRASTRUCTURE: the direct grouped-convolution kernel of laser_b200/csrc/gemm_simt.cuh
// in its input-gradient instantiation (conv_grouped_direct_kernel<MC, true>, the exact path of
// laser_b200_conv2d_grouped_input_grad_f32_fused_dev) compiled for the host (cuda_emu.h) behind a C interface for ctypes, launched
// with the tile the library plans (conv_grouped_plan) over the transposed geometry capi.cu builds.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/gemm_simt.cuh"

using namespace lb200;

extern "C" {

// geom = the FORWARD call's {n, C, H, W, Cout, kH, kW, pH, pW, sH, sW}; dx [n][C][H][W] (read when beta != 0), dy
// [n][Cout][outH][outW], kernel [Cout][C / groups][kH][kW], aux laid out like dy (NULL: none).  Returns the channels per thread
// (1, 2, 4) or 0 when the plan fails.
int emu_conv_grouped_input_grad(float *dx, const float *dy, const float *kernel, const int64_t *geom, int64_t groups, float alpha,
                                float beta, int op, const float *aux, int grid) {
  ConvGeom g{};
  g.B = geom[0]; g.C = geom[1]; g.H = geom[2]; g.W = geom[3]; g.Cout = geom[4]; g.kH = geom[5]; g.kW = geom[6];
  g.pH = geom[7]; g.pW = geom[8]; g.sH = geom[9]; g.sW = geom[10];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  // the transposed geometry of capi.cu: conv2d_grouped_input_grad_dev
  ConvGeom gt = g;
  gt.C = g.Cout; gt.H = g.outH; gt.W = g.outW; gt.Cout = g.C;
  gt.pH = g.kH - 1 - g.pH; gt.pW = g.kW - 1 - g.pW;
  gt.sH = gt.sW = 1;
  gt.dH = g.sH; gt.dW = g.sW;
  gt.outH = g.H; gt.outW = g.W;
  ConvGroupedGradParams p;
  int mc;
  size_t smem;
  const int threads = conv_grouped_plan(gt, groups, nullptr, 0, &p, &mc, &smem);
  if (threads == 0 || smem > emu::kDynSmemBytes) return 0;
  p.dH = static_cast<int>(g.sH);
  p.dW = static_cast<int>(g.sW);
  p.alpha = alpha;
  p.beta = beta;
  p.op = op;
  p.aux = aux;
  const unsigned blocks = static_cast<unsigned>(grid > 0 && grid < p.tiles ? grid : p.tiles);
  const unsigned block = static_cast<unsigned>(threads);   // (no warp operation: a partial last warp is fine)
  if (mc == 4) emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<4, true>(dx, dy, kernel, p); });
  else if (mc == 2) emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<2, true>(dx, dy, kernel, p); });
  else emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<1, true>(dx, dy, kernel, p); });
  return mc;
}

// out[i] = the library's operand op (split.cuh: operand_op) of x[i] with aux y[i] (y NULL: 0)
void emu_operand_op(int op, const float *x, const float *y, int64_t n, float *out) {
  for (int64_t i = 0; i < n; ++i) out[i] = operand_op(op, x[i], y ? y[i] : 0.0f);
}

}  // extern "C"
