// tc_emu.cpp -- TEST INFRASTRUCTURE: the wgmma GEMM kernel (laser_b200/csrc/gemm_tc.cuh) compiled
// by g++ on top of ptx_emu.h (a functional model of mbarrier / TMA / wgmma / clusters of two CTAs) and
// launched on host threads with the library's own planning (tc_plan) and the tensor-map parameters
// capi.cu passes to cuTensorMapEncodeTiled (operand_map).  See ptx_emu.h for what this can and
// cannot prove.
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include <vector>

#include "../../laser_b200/csrc/gemm_tc.cuh"
#include "../../laser_b200/csrc/split.cuh"

using namespace lb200;

static CUtensorMap make_map(int esz, const void *base, int64_t inner, int64_t outer, int64_t outer_stride_elems,
                            int box_inner, int box_outer) {
  CUtensorMap out;
  std::memset(&out, 0, sizeof out);
  if (!base) return out;
  emu::TensorMap2D m;
  m.magic = emu::kMapMagic;
  m.base = static_cast<const unsigned char *>(base);
  m.dim0 = inner; m.dim1 = outer;
  m.stride1_bytes = outer_stride_elems * esz;
  m.esz = esz; m.box0 = box_inner; m.box1 = box_outer;
  std::memcpy(&out, &m, sizeof m);
  return out;
}
// capi.cu: operand_map -- an operand seen as [mn][k]; K-major: array [mn][ld], MN-major: array [k][ld]
static CUtensorMap operand_map(int esz, const void *base, bool mn_major, int64_t mn, int64_t k, int64_t ld, int block_mn) {
  const int block_k = TC_ROW_BYTES / esz, mn_atom = TC_ROW_BYTES / esz;
  if (!mn_major) return make_map(esz, base, k, mn, ld, block_k, block_mn);
  return make_map(esz, base, mn, k, ld, mn_atom, block_k);
}

struct Args {
  int64_t M, N, K;
  float alpha, beta;
  const void *A[2], *B[2];   // piece 0 / piece 1, see capi.cu: OperandMaps
  int64_t ldA, ldB;
  void *C;
  int64_t rsC, csC;
  int kc_faithful, raster_g, splitk_enabled, sm_count;
  const float *bias;
  int bias_per_row, act;
  float *splitk_ws;          // tile-local planes of the split tiles (tc_params.h: tc_split_ws_floats)
  int64_t splitk_ws_floats;
  int *out_k_splits, *out_grid;
  const uint32_t *amax_a, *amax_b;   // SCALED: abs-max words per row of A / column of B (f16_scale.cuh)
  int tail_min_k;            // TcPlanCfg::tail_min_k (0: the library's default)
  int dyn_sched;             // 1: tiles drawn from an atomic counter (capi.cu: Ctx::sched), 0: static round-robin
};

static unsigned int g_sched[2] = {0u, 0u};

template <int ESZ, uint32_t FMT16, int NPASS, typename OutT, bool SCALED, bool A_MN, bool B_MN, bool PAIR>
static int run(const Args &a) {
  TcParams p;
  p.M = a.M; p.N = a.N; p.K = a.K; p.alpha = a.alpha; p.beta = a.beta;
  p.C = a.C; p.rsC = a.rsC; p.csC = a.csC; p.zero = 0;
  p.epi.bias = a.bias; p.epi.bias_per_row = a.bias_per_row; p.epi.act = a.act;
  p.amax_a = a.amax_a; p.amax_b = a.amax_b;
  TcPlanCfg cfg{a.kc_faithful, a.raster_g, a.splitk_enabled != 0, a.sm_count};
  if (a.tail_min_k > 0) cfg.tail_min_k = a.tail_min_k;
  tc_plan<ESZ, std::is_same<OutT, float>::value>(p, NPASS, PAIR, cfg);
  if (a.out_k_splits) { a.out_k_splits[0] = p.k_splits; a.out_k_splits[1] = p.n_direct; }
  if (p.k_splits > 1) {   // capi.cu: tc_run -- raw partial sums of the split tiles into the planes, reduced by splitk_tail_reduce_kernel
    if (!a.splitk_ws || a.splitk_ws_floats < tc_split_ws_floats(p, PAIR)) return -2;
    p.split_ws = a.splitk_ws;
  }
  if (a.dyn_sched) {
    if (g_sched[0] != 0u || g_sched[1] != 0u) return -4;   // the previous launch must have re-armed its slot
    p.sched = g_sched;
  }
  const int b_block = TC_BLOCK_N;
  const CUtensorMap mA0 = operand_map(ESZ, a.A[0], A_MN, a.M, a.K, a.ldA, TC_BLOCK_M), mA1 = operand_map(ESZ, a.A[1], A_MN, a.M, a.K, a.ldA, TC_BLOCK_M);
  const CUtensorMap mB0 = operand_map(ESZ, a.B[0], B_MN, a.N, a.K, a.ldB, b_block), mB1 = operand_map(ESZ, a.B[1], B_MN, a.N, a.K, a.ldB, b_block);
  // tc_launch_impl.cuh: launch_tc_one -- persistent: one CTA (pair) per SM (pair of SMs), never more than work units
  const int64_t units_total = tc_units(p);
  const int units = PAIR ? a.sm_count / 2 : a.sm_count;
  const int sched = static_cast<int>(units_total < units ? units_total : units);
  const unsigned grid = PAIR ? 2 * sched : sched;
  if (a.out_grid) *a.out_grid = static_cast<int>(grid);
  if (TcCfg<NPASS, PAIR>::SMEM_BYTES > static_cast<int>(emu::kDynSmemBytes)) return -3;
  emu::reset_state();
  emu::launch(grid, TC_THREADS,
              [=]() { gemm_tc_kernel<ESZ, FMT16, NPASS, A_MN, B_MN, OutT, PAIR, SCALED>(mA0, mA1, mB0, mB1, p); },
              PAIR ? 2 : 1);
  if (p.k_splits > 1) {
    if constexpr (std::is_same<OutT, float>::value) {
      const int n_tail = p.num_m_blocks * p.num_n_blocks - p.n_direct;
      const int tile_m = PAIR ? 2 * TC_BLOCK_M : TC_BLOCK_M;
      const float *ws = a.splitk_ws;
      const TcParams q = p;
      float *C = static_cast<float *>(a.C);
      const Args b = a;
      emu::launch(3, 256, [=]() {
        splitk_tail_reduce_kernel(ws, q.k_splits, n_tail, q.n_direct, q.num_m_blocks, q.num_n_blocks, q.raster_g, tile_m, b.M, b.N,
                                  b.alpha, b.beta, C, b.rsC, b.csC, b.bias, b.bias_per_row, b.act);
      });
    } else {
      return -5;
    }
  }
  return 0;
}

// capi.cu: prepare_operand -- the tf32 modes gather an MN-major fp32 operand ([k][ld]) into compact K-major rows
static const void *to_k_major(const void *src, int64_t mn, int64_t k, int64_t ld, int64_t ld_out, std::vector<float> &dst) {
  if (!src) return nullptr;
  dst.assign(static_cast<size_t>(mn * ld_out), 0.0f);
  const float *s = static_cast<const float *>(src);
  for (int64_t i = 0; i < mn; ++i)
    for (int64_t kk = 0; kk < k; ++kk) dst[i * ld_out + kk] = s[kk * ld + i];
  return dst.data();
}

template <int ESZ, uint32_t FMT16, int NPASS, typename OutT, bool SCALED>
static int dispatch(int a_mn, int b_mn, int pair, const Args &a_in) {
#define GO(AMN, BMN) (pair ? run<ESZ, FMT16, NPASS, OutT, SCALED, AMN, BMN, true>(a) : run<ESZ, FMT16, NPASS, OutT, SCALED, AMN, BMN, false>(a))
  Args a = a_in;
  if constexpr (ESZ == 4) {
    std::vector<float> ka[2], kb[2];
    const int64_t ld_k = (a.K + 3) / 4 * 4;
    if (a_mn) {
      for (int i = 0; i < 2; ++i) a.A[i] = to_k_major(a_in.A[i], a.M, a.K, a_in.ldA, ld_k, ka[i]);
      a.ldA = ld_k;
    }
    if (b_mn) {
      for (int i = 0; i < 2; ++i) a.B[i] = to_k_major(a_in.B[i], a.N, a.K, a_in.ldB, ld_k, kb[i]);
      a.ldB = ld_k;
    }
    return GO(false, false);
  } else {
    if (!a_mn && !b_mn) return GO(false, false);
    if (!a_mn && b_mn) return GO(false, true);
    if (a_mn && !b_mn) return GO(true, false);
    return GO(true, true);
  }
#undef GO
}

// kind: 0 tf32x1, 1 tf32x3, 2 bf16, 3 f16x3 (tc_launch.h: the four kernel families)
extern "C" int emu_gemm_tc(int kind, int a_mn, int b_mn, int pair, int64_t M, int64_t N, int64_t K, float alpha, float beta,
                           const void *A0, const void *A1, int64_t ldA, const void *B0, const void *B1, int64_t ldB,
                           void *C, int64_t rsC, int64_t csC, int kc_faithful, int raster_g, int splitk_enabled,
                           int sm_count, const float *bias, int bias_per_row, int act, float *splitk_ws, int64_t splitk_ws_floats, int *out_k_splits,
                           int *out_grid, const uint32_t *amax_a, const uint32_t *amax_b, int dyn_sched, int tail_min_k) {
  Args a{M, N, K, alpha, beta, {A0, A1}, {B0, B1}, ldA, ldB, C, rsC, csC, kc_faithful,
         raster_g, splitk_enabled, sm_count, bias, bias_per_row, act, splitk_ws, splitk_ws_floats, out_k_splits, out_grid, amax_a, amax_b, tail_min_k, dyn_sched};
  switch (kind) {
    case 0: return dispatch<4, ptx::kFmtBF16, 1, float, false>(a_mn, b_mn, pair, a);
    case 1: return dispatch<4, ptx::kFmtBF16, 3, float, false>(a_mn, b_mn, pair, a);
    case 2: return dispatch<2, ptx::kFmtBF16, 1, uint16_t, false>(a_mn, b_mn, pair, a);
    case 3: return dispatch<2, ptx::kFmtF16, 3, float, true>(a_mn, b_mn, pair, a);
    default: return -1;
  }
}
