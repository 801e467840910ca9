// conv_grouped_emu.cpp -- TEST INFRASTRUCTURE: the direct grouped-convolution kernel of laser_b200/csrc/gemm_simt.cuh (conv_grouped_direct_kernel)
// compiled for the host (cuda_emu.h) behind a C interface for ctypes, launched with the tile the library plans
// (conv_grouped_plan).
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include "../../laser_b200/csrc/gemm_simt.cuh"

using namespace lb200;

extern "C" {

// geom = {n, C, H, W, Cout, kH, kW, pH, pW, sH, sW}; returns the channels per thread (1, 2, 4) or 0 when the plan fails
int emu_conv_grouped(float *out, const float *in, const float *kernel, const int64_t *geom, int64_t groups, const float *bias,
                     int act, int grid) {
  ConvGeom g{};
  g.B = geom[0]; g.C = geom[1]; g.H = geom[2]; g.W = geom[3]; g.Cout = geom[4]; g.kH = geom[5]; g.kW = geom[6];
  g.pH = geom[7]; g.pW = geom[8]; g.sH = geom[9]; g.sW = geom[10];
  g.outH = 1 + (g.H + 2 * g.pH - g.kH) / g.sH;
  g.outW = 1 + (g.W + 2 * g.pW - g.kW) / g.sW;
  ConvGroupedParams p;
  int mc;
  size_t smem;
  const int threads = conv_grouped_plan(g, groups, bias, act, &p, &mc, &smem);
  if (threads == 0 || smem > emu::kDynSmemBytes) return 0;
  const unsigned blocks = static_cast<unsigned>(grid > 0 && grid < p.tiles ? grid : p.tiles);
  const unsigned block = static_cast<unsigned>(threads);   // (no warp operation: a partial last warp is fine)
  if (mc == 4) emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<4>(out, in, kernel, p); });
  else if (mc == 2) emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<2>(out, in, kernel, p); });
  else emu::launch(blocks, block, [=]() { conv_grouped_direct_kernel<1>(out, in, kernel, p); });
  return mc;
}

// the exact kernel's bias + activation over x[rows][cols] (bias one per row), in place
void emu_bias_act(float *x, int64_t rows, int64_t cols, const float *bias, int act) {
  for (int64_t r = 0; r < rows; ++r)
    for (int64_t c = 0; c < cols; ++c) x[r * cols + c] = simt_bias_act(x[r * cols + c], bias, 1, act, r, c);
}

}  // extern "C"
