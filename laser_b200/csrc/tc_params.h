// tc_params.h -- host-visible part of the tensor-core GEMM: tile constants, the kernel's parameter block and the launch
// planning (no device code: capi.cu includes this without instantiating the kernel, see tc_launch.h)
#pragma once

#include <stdint.h>

#if defined(__CUDACC__) || defined(LB200_HOST_EMULATION)
#define LB200_HD __host__ __device__
#else
#define LB200_HD
#endif

namespace lb200 {

constexpr int TC_BLOCK_M = 128;
constexpr int TC_BLOCK_N = 128;
constexpr int TC_ROW_BYTES = 128;  // one swizzle row; BLOCK_K = 128 / sizeof(element)
constexpr int TC_A_TILE_BYTES = TC_BLOCK_M * TC_ROW_BYTES;  // 16 KB: 128 rows x 128 B
template <int NPASS> struct TcCfg {
  static constexpr int PIECES = (NPASS == 3) ? 2 : 1;
  static constexpr int B_TILE_BYTES = TC_BLOCK_N * TC_ROW_BYTES;
  static constexpr int A_STAGE_BYTES = PIECES * TC_A_TILE_BYTES;
  static constexpr int B_STAGE_BYTES = PIECES * B_TILE_BYTES;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;  // 32 KB (1 pass), 64 KB (3 passes)
#ifdef TC_STAGES_OVERRIDE
  static constexpr int STAGES = TC_STAGES_OVERRIDE;
#else
  static constexpr int STAGES = (NPASS == 3) ? 3 : 6;   // 192 KB of tiles in every variant (227 KB per block on sm_90)
#endif
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 512 /*barriers, scheduler slot*/;
};
// warpgroup 0: warp 0 TMA, warp 3 tile scheduler | warpgroups 1, 2: wgmma + epilogue, 64 rows each
constexpr int TC_THREADS = 384;
constexpr int TC_EPI_THREADS = 256;
constexpr int TC_EPI_WARPS = TC_EPI_THREADS / 32;
constexpr int TC_ACC_REGS = 64 * TC_BLOCK_N / 128;   // fp32 accumulators per thread of an m64 x n128 wgmma
constexpr int TC_REGS_CTRL = 40;   // setmaxnreg for the producer / scheduler warpgroup
constexpr int TC_REGS_EPI = 232;   // ... and for the consumer warpgroups (accumulators + running sums): 128 x 40 + 256 x 232 <= 65536

// fused epilogue: v -> act(v + bias)   (gemm.nim:196 "elementwise epilogue fusion")
struct Epilogue {
  const float *bias = nullptr;
  int bias_per_row = 0;
  int act = 0;  // 0 none, 1 relu, 2 tanh, 3 sigmoid
};
struct TcParams {
  int64_t M, N, K;
  float alpha, beta;
  void *C;
  int64_t rsC, csC;
  int kb_per_block;   // k-tiles per accumulation block of the wgmma registers (>= 1)
  int raster_g;       // m-blocks per raster group (see tile_coords)
  Epilogue epi;
  // split-K.  Tiles [0, n_direct) (raster order, tile_coords) are computed over all of K and stored through the epilogue
  // into C.  Each of the remaining `num tiles - n_direct` tiles is cut in k_splits K-ranges of kb_per_split k-tiles; unit
  // n_direct + i * k_splits + s computes range s of tile n_direct + i and writes its raw partial sums (scales undone, no
  // alpha / beta / bias / activation) to the tile-local plane [s][i] of split_ws; splitk_tail_reduce_kernel then adds the
  // planes in order and applies alpha / beta / epilogue.  Two uses: few output tiles and a long K (n_direct = 0: every
  // tile is split), and the partial last wave of a persistent launch (n_direct = the tiles of the full waves: the
  // remainder of at most half a wave runs as twice as many half-K units, which the idle SMs take up)
  int n_direct;          // == num_m_blocks * num_n_blocks when nothing is split
  int k_splits;          // >= 1
  int kb_per_split;      // k-tiles per split
  float *split_ws = nullptr;   // [k_splits][split tiles][TC_BLOCK_M][TC_BLOCK_N] fp32
  int num_m_blocks, num_n_blocks;  // output tiles of 128 x 128
  // SCALED: fp32 bits of the largest finite |a| of row i of A / |b| of column j of B (f16_scale.cuh)
  const uint32_t *amax_a = nullptr, *amax_b = nullptr;
  // tile scheduler: word 0 = next unit (atomicAdd), word 1 = CTAs that have drawn their last unit (the last one zeroes
  // both words for the next launch that uses this slot).  nullptr: static round-robin (unit = CTA index + i * CTAs)
  unsigned int *sched = nullptr;
  // batched launch (gemm_tc_kernel<..., BATCHED = true>): `batch` problems of M x N x K.  Tile t of the launch is tile
  // t % (num_m_blocks * num_n_blocks) of problem t / (num_m_blocks * num_n_blocks); split-K and the raster order apply to
  // these tiles as above.  Problem b reads slice b * map_b_a (b * map_b_b) of A's (B's) rank-3 tensor maps -- 0 for an
  // operand the batch shares --, writes C + b * bsC and reads its scale words b * amax_bs_a (b * amax_bs_b) further on.
  int batch = 1;
  int map_b_a = 0, map_b_b = 0;
  int64_t bsC = 0;
  int64_t amax_bs_a = 0, amax_bs_b = 0;
};

// raster order of the output tiles: groups of G m-blocks sweep n together, so that the concurrently resident tiles (132 of
// 128 x 128 on an H100 SXM) cover a compact patch, which limits the A + B panels one wave pulls through L2 (G = 16 tiles =
// 2048 rows)
LB200_HD inline void tile_coords(int t, int num_m, int num_n, int G, int &mb, int &nb) {
  const int per_group = G * num_n;
  const int g = t / per_group;
  const int first_m = g * G;
  const int gsz = (G < num_m - first_m) ? G : (num_m - first_m);
  const int r = t - g * per_group;
  mb = first_m + r % gsz;
  nb = r / gsz;
}

// host side: the part of TcParams that depends only on the problem (p.M, p.N, p.K set by the
// caller) and on the configuration
struct TcPlanCfg {
  int kc_faithful;      // K extent per accumulator block in the fp32-faithful modes
  int raster_g;         // 0 = default
  bool splitk_enabled;
  int sm_count;
  int tail_min_k = 2048;   // shortest K for which the remainder behind full waves is split
};
template <int ESZ, bool OUT_F32>
inline void tc_plan(TcParams &p, int npass, const TcPlanCfg &cfg) {
  const int block_k = TC_ROW_BYTES / ESZ;  // k-tile
  const int num_kb = static_cast<int>((p.K + block_k - 1) / block_k);
  {
    // K extent accumulated inside the tensor core before the epilogue warps add the block
    // to their fp32 running sums (the analogue of the reference's kc, gemm_tiling.nim:310).
    // Only the fp32-faithful modes need short chains.
    const int kc = (npass == 3) ? cfg.kc_faithful : 0;
    p.kb_per_block = (kc > 0) ? (kc + block_k - 1) / block_k : num_kb;
    if (p.kb_per_block < 1) p.kb_per_block = 1;
    if (p.kb_per_block > num_kb) p.kb_per_block = num_kb;
  }
  p.raster_g = cfg.raster_g > 0 ? cfg.raster_g : 16;
  p.num_m_blocks = static_cast<int>((p.M + TC_BLOCK_M - 1) / TC_BLOCK_M);
  p.num_n_blocks = static_cast<int>((p.N + TC_BLOCK_N - 1) / TC_BLOCK_N);
  // ---- split-K (fp32 output only): too few output tiles to fill the machine and a long K, or a thin last wave ----
  const int64_t tiles = static_cast<int64_t>(p.num_m_blocks) * p.num_n_blocks * p.batch;
  p.k_splits = 1;
  p.kb_per_split = num_kb;
  p.n_direct = static_cast<int>(tiles);
  p.split_ws = nullptr;
  const int units = cfg.sm_count;
  if constexpr (OUT_F32) {
    const int blocks = (num_kb + p.kb_per_block - 1) / p.kb_per_block;   // accumulation blocks along K
    // every split keeps >= 512 K-elements
    const int min_tiles = 512 / block_k;
    const int min_blocks = (min_tiles + p.kb_per_block - 1) / p.kb_per_block;
    const int max_s = blocks / min_blocks < 16 ? blocks / min_blocks : 16;
    // tiles that do not fill a wave of their own: all of them when there are fewer than `units`, else the remainder
    const int64_t rem = tiles < units ? tiles : tiles % units;
    int S = rem > 0 ? static_cast<int>(units / rem) : 1;
    if (S > max_s) S = max_s;
    // a remainder behind full waves (S >= 2: at most half a wave of tiles) is split when a tile is long enough for half
    // of it to outweigh the reduce kernel
    const bool worth = S >= 2 && (tiles < units || p.K >= cfg.tail_min_k);
    if (cfg.splitk_enabled && worth && units > 0) {
      const int blocks_per_split = (blocks + S - 1) / S;
      p.k_splits = (blocks + blocks_per_split - 1) / blocks_per_split;
      p.kb_per_split = blocks_per_split * p.kb_per_block;
      if (p.k_splits >= 2) p.n_direct = static_cast<int>(tiles - rem);
      else { p.k_splits = 1; p.kb_per_split = num_kb; }
    }
  }
}
// work units of a planned launch, and the fp32 words of its split-K workspace (0: nothing is split)
inline int64_t tc_units(const TcParams &p) {
  const int64_t tiles = static_cast<int64_t>(p.num_m_blocks) * p.num_n_blocks * p.batch;
  return p.n_direct + (tiles - p.n_direct) * p.k_splits;
}
inline int64_t tc_split_ws_floats(const TcParams &p) {
  const int64_t tiles = static_cast<int64_t>(p.num_m_blocks) * p.num_n_blocks * p.batch;
  return (tiles - p.n_direct) * p.k_splits * TC_BLOCK_M * TC_BLOCK_N;
}

}  // namespace lb200
