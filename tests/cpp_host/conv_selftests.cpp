// conv_selftests.cpp -- the reference's convolution self-check (`conv_impl_check`,
// benchmarks/convolution/conv2d_common.nim:128-283) and a transposition check (swapaxes.nim:16-112)
// re-stated against the C++ host mirror (include/laser_b200.hpp).  Needs an H100 to run; with
// --link-only it only proves that the mirror compiles and links.
#include <cstdio>
#include <cstring>
#include <vector>

#include "laser_b200.hpp"

using namespace laser;

static int conv_case(const char *src, TensorShape ishape, KernelShape kshape, Padding padding, Strides strides,
                     const std::vector<float> &input, const std::vector<float> &kernel, const std::vector<float> &target) {
  const TensorShape oshape = conv2d_out_shape(ishape, kshape, padding, strides);
  std::vector<float> output(static_cast<size_t>(oshape.n * oshape.c * oshape.h * oshape.w), 99.0f);
  conv2d_im2col(output.data(), oshape, input.data(), ishape, kernel.data(), kshape, padding, strides);
  const bool ok = output == target;   // doAssert target == output
  std::printf("%s %s\n", ok ? "SUCCESS" : "FAILURE", src);
  return ok ? 0 : 1;
}

int main(int argc, char **argv) {
  if (argc > 1 && std::strcmp(argv[1], "--instantiate") == 0) {   // never run: instantiates the tensor-level templates
    CudaTensor<float> a = newTensor<float>({2, 3}), b = newTensor<float>({2, 3}), o = newTensor<float>({2, 3});
    forEach(LASER_B200_FOREACH_FMA, o, &o, &a, &b);
    copyFrom(o, a);
    return 0;
  }
  if (argc > 1 && std::strcmp(argv[1], "--link-only") == 0) {
    std::printf("laser_b200 %d workspace %lld\n", laser_b200_version(),
                (long long)im2col_workspace_size({1, 3, 5, 5}, {2, 3, 3, 3}, {1, 1}, {2, 2}));
    return 0;
  }
  int bad = 0;
  try {
    bad += conv_case("conv2d_common.nim:137-178", {1, 1, 4, 4}, {1, 1, 3, 3}, {1, 1}, {1, 1},
                     {1, 2, 0, 0, 5, 3, 0, 4, 0, 0, 0, 7, 9, 3, 0, 0}, {1, 1, 1, 1, 1, 0, 1, 0, 0},
                     {1, 8, 5, 0, 8, 11, 5, 4, 8, 17, 10, 11, 9, 12, 10, 7});
    bad += conv_case("conv2d_common.nim:180-283", {1, 3, 5, 5}, {2, 3, 3, 3}, {1, 1}, {2, 2},
                     {2, 2, 0, 2, 1, 0, 1, 1, 0, 2, 1, 2, 1, 2, 1, 2, 2, 0, 0, 2, 2, 1, 1, 1, 2,
                      2, 0, 1, 1, 1, 2, 2, 0, 0, 2, 2, 2, 1, 0, 0, 1, 1, 2, 2, 0, 2, 1, 1, 1, 0,
                      0, 1, 2, 2, 0, 1, 1, 1, 1, 0, 2, 1, 2, 2, 0, 0, 2, 2, 2, 1, 0, 0, 2, 2, 1},
                     {-1, -1, -1, 1, 0, 1, 0, -1, 0, 1, 0, -1, 1, -1, 1, 0, 1, 0, 0, 0, 1, -1, -1, -1, -1, 0, 0,
                      0, 1, 0, 1, -1, -1, 1, 1, -1, -1, 0, 1, -1, -1, 1, 1, 1, 0, 0, 1, 1, -1, 1, -1, -1, -1, 0},
                     {1, -3, -1, -4, 1, -6, -3, -2, -1, -7, 1, 0, 3, -3, 2, 1, 3, -2});
    // transposition: 4000 x 2000 float32, the reference bench shape (transpose_bench.nim:54-55)
    const int64_t NR = 4000, NC = 2000;
    std::vector<float> a(static_cast<size_t>(NR * NC)), t(a.size()), back(a.size());
    for (size_t i = 0; i < a.size(); ++i) a[i] = static_cast<float>(i % 8191);
    transpose2D_copy(t.data(), a.data(), NR, NC);
    transpose2D_copy(back.data(), t.data(), NC, NR);
    bool ok = back == a;
    for (int64_t i = 0; ok && i < NR; i += 97)
      for (int64_t j = 0; j < NC; j += 89) ok = ok && t[static_cast<size_t>(j * NR + i)] == a[static_cast<size_t>(i * NC + j)];
    std::printf("%s swapaxes.nim:16-54\n", ok ? "SUCCESS" : "FAILURE");
    bad += ok ? 0 : 1;
  } catch (const LaserB200Error &e) {
    std::printf("FAILURE %s\n", e.what());
    return 2;
  }
  return bad;
}
