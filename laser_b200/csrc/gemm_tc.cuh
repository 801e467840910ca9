// gemm_tc.cuh -- the wgmma / TMA strided GEMM for sm_90a (ONE kernel template).
//
// What it replaces in the reference (mratsim/laser, paths relative to
// laser/primitives/matrix_multiplication/):
//   pack_A_mc_kc / pack_B_kc_nc (gemm_packing.nim:24-94)  -> TMA tensor maps: the
//       copy engine resolves the operand's strides and lands 128-byte-swizzled
//       tiles in shared memory; no packing buffers exist.
//   gebb_ukernel register micro-kernel (gemm_ukernel_generator.nim:140-250)
//       -> wgmma.mma_async (tf32 / f16 / bf16) issued by two consumer warpgroups per CTA, each
//       owning 64 rows x 128 columns of the 128 x 128 output tile, accumulators in registers.
//   gemm_impl loop pc (gemm.nim:150-158: K is cut in kc blocks, every block's partial
//       product is ADDED to C in fp32) -> K is cut in accumulation blocks of `kb_per_block`
//       k-tiles: the tensor core accumulates one block in the wgmma accumulator registers, which
//       are then added (IEEE round-to-nearest FADD) to running sums held in other registers.
//       This matters numerically: the tensor core's own accumulation does not round to nearest,
//       so long chains must not live in the accumulator.
//   gebp_mkernel loops jr/ir + loop ic (gemm.nim:48-176; `omp for` over ic blocks)
//       -> persistent CTAs that DRAW output tiles from an atomic counter in device memory (a scheduler
//       thread per CTA publishes the unit through shared memory): tiles go to whichever
//       CTA is free, so SMs that start late (another kernel -- e.g. the NCCL broadcast of the
//       row-sharded driver -- still holds them) or run slower simply take fewer tiles.
//   epilogues (gemm_ukernel_generic.nim:53-126)
//       -> alpha/beta in fp32 from the running sums; beta == 0 never reads C; optional fused
//       bias + activation (the reference's TODO at gemm.nim:196).
//
// Warp roles (384 threads): warp 0 lane 0 issues the TMA loads into a ring of stages, warp 3 lane 0 runs the tile
// scheduler, warpgroups 1 and 2 issue the MMAs and store their rows of C.
//
// Template parameters:
//   ESZ     element size of the tiles (4: fp32 containers read as tf32, 2: 16-bit)
//   FMT16   ptx::kFmtBF16 or ptx::kFmtF16 (ESZ == 2)
//   NPASS   1: one MMA pass over (A, B).  3: fp32-faithful product of two-piece operands
//           x = hi + lo: per k-tile the stage holds FOUR tiles (A_hi, A_lo, B_hi, B_lo), each loaded
//           ONCE, and feeds three passes hi*lo', lo*hi', hi*hi'
//   A_MN/B_MN operand major-ness (wgmma reads K-major and MN-major 16-bit tiles natively, so A^T*B,
//           A*B^T ... need no data movement; tf32 tiles must be K-major)
//   OutT    float or uint16_t (bf16 bits)
//   SCALED  F16X3 mode: the operands are fp16 pieces of A's rows / B's columns scaled by powers of
//           two (f16_scale.cuh); the epilogue multiplies output (i, j) by 2^-sA[i] * 2^-sB[j]
//   BATCHED p.batch problems in one launch (tc_params.h): rank-3 tensor maps {inner, outer, problem} with a box depth
//           of 1, so that TMA zero-fills past M, N and K within each problem
#pragma once

#include <type_traits>

#include "f16_scale.cuh"
#include "ptx.cuh"
#include "tc_params.h"

namespace lb200 {

// (out of line: inlined into the unrolled stores the tanhf / expf bodies would multiply the kernel's code size, and the
// consumer warps would miss the instruction cache on every tile)
#ifndef LB200_HOST_EMULATION
static __device__ __noinline__ float epi_act(float v, int act) {
#else
inline float epi_act(float v, int act) {
#endif
  if (act == 1) return fmaxf(v, 0.0f);
  if (act == 2) return tanhf(v);
  if (act == 3) return 1.0f / (1.0f + expf(-v));
  return v;
}

__device__ __forceinline__ float bf16_bits_to_f32(uint16_t h) {
  return __uint_as_float(static_cast<uint32_t>(h) << 16);
}
__device__ __forceinline__ uint16_t f32_to_bf16_bits(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}

// Tensor maps of the kernel: piece 0 (hi, or the operand itself) and piece 1 (lo; unused when NPASS == 1)
template <int ESZ, uint32_t FMT16, int NPASS, bool A_MN, bool B_MN, typename OutT, bool SCALED, bool BATCHED>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
               const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1,
               const TcParams p) {
  static_assert(NPASS == 1 || NPASS == 3, "one pass, or the three passes of a two-piece product");
  static_assert(ESZ == 2 || (!A_MN && !B_MN), "wgmma reads tf32 operands K-major only (capi.cu transposes MN-major fp32)");
  using Cfg = TcCfg<NPASS>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int BLOCK_K = TC_ROW_BYTES / ESZ;             // 32 or 64 k-elements per k-tile
  const int sched_id = static_cast<int>(blockIdx.x);
  const int sched_stride = static_cast<int>(gridDim.x);

  LB200_DYN_SMEM(uint8_t, smem_raw);
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                              ~static_cast<uintptr_t>(1023));
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t *full_bar = bars;                        // [STAGES]
  uint64_t *empty_bar = bars + STAGES;              // [STAGES]
  uint64_t *sched_full = bars + 2 * STAGES;         // the scheduler published a unit (one slot)
  uint64_t *sched_empty = sched_full + 1;           // every consumer has read it
  int *sched_unit = reinterpret_cast<int *>(sched_empty + 1);

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_pp = p.num_m_blocks * p.num_n_blocks;   // output tiles of one problem
  const int num_tiles = BATCHED ? tiles_pp * p.batch : tiles_pp;
  const int num_kb = static_cast<int>((p.K + BLOCK_K - 1) / BLOCK_K);
  // work units of the persistent scheduler: the direct tiles, then k_splits K-ranges of each of the other tiles (tc_params.h)
  const int num_units = p.n_direct + (num_tiles - p.n_direct) * p.k_splits;
  // unit -> tile t, K range [kb_lo, kb_hi) in k-tiles, split index sp (-1: a direct tile)
  auto decode_unit = [&](int u, int &t, int &sp, int &kb_lo, int &kb_hi) {
    if (u < p.n_direct) {
      t = u; sp = -1; kb_lo = 0; kb_hi = num_kb;
    } else {
      const int v = u - p.n_direct;
      const int i = v / p.k_splits;
      t = p.n_direct + i;
      sp = v - i * p.k_splits;
      kb_lo = min(num_kb, sp * p.kb_per_split);
      kb_hi = min(num_kb, kb_lo + p.kb_per_split);
    }
  };
  // consumers of the scheduler slot: the producer thread and lane 0 of each consumer warp
  constexpr int SCHED_CONSUMERS = 1 + TC_EPI_WARPS;
  // next unit of this CTA, or -1.  One thread per consumer calls it; `ph` is that consumer's phase bit.
  auto next_unit = [&](uint32_t &ph) -> int {
    ptx::mbar_wait(sched_full, ph);
    const int u = *reinterpret_cast<volatile int *>(sched_unit);
    ptx::mbar_arrive(sched_empty);   // slot read
    ph ^= 1u;
    return u;
  };

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&mapA0);
    ptx::prefetch_tensormap(&mapB0);
    if constexpr (NPASS == 3) {
      ptx::prefetch_tensormap(&mapA1);
      ptx::prefetch_tensormap(&mapB1);
    }
  }
  if (threadIdx.x == 32) {
    for (int i = 0; i < STAGES; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], TC_EPI_WARPS);   // lane 0 of every consumer warp releases the stage
    }
    ptx::mbar_init(sched_full, 1);
    ptx::mbar_init(sched_empty, SCHED_CONSUMERS);
    ptx::fence_barrier_init();
  }
  __syncthreads();   // barrier inits visible to all warps
  // programmatic dependent launch: everything above overlapped the tail of the preceding kernel of the stream (the operand
  // preparation); its results (prepared tiles, abs-max words) are visible from here on.  No-op for an ordinary launch.
  ptx::griddep_wait();

  if (warp_idx < 4) {
    ptx::setmaxnreg_dec<TC_REGS_CTRL>();  // hand registers to the consumer warpgroups
    if (warp_idx == 3 && lane == 0) {
      // ===================== tile scheduler (one thread) =====================
      uint32_t phase = 0;
      int next_static = sched_id;
      for (;;) {
        ptx::mbar_wait(sched_empty, phase ^ 1);
        int u;
        if (p.sched) {
          u = static_cast<int>(atomicAdd(p.sched, 1u));
        } else {
          u = next_static;
          next_static += sched_stride;
        }
        if (u >= num_units) u = -1;
        *reinterpret_cast<volatile int *>(sched_unit) = u;
        ptx::mbar_arrive(sched_full);
        phase ^= 1u;
        if (u < 0) {
          if (p.sched) {   // the last CTA to run dry re-arms the counter for the next launch on this slot
            __threadfence();
            if (atomicAdd(p.sched + 1, 1u) == static_cast<unsigned int>(sched_stride - 1)) {
              p.sched[0] = 0u;
              p.sched[1] = 0u;
              __threadfence();
            }
          }
          break;
        }
      }
    } else if (warp_idx == 0 && lane == 0) {
      // ===================== TMA producer (one thread) =====================
      int stage = 0;
      uint32_t phase = 0, sched_phase = 0;
      constexpr int MN_ATOM = TC_ROW_BYTES / ESZ;             // elements per 128-byte MN chunk
      constexpr int MN_BOX_BYTES = BLOCK_K * TC_ROW_BYTES;    // one [BLOCK_K][128 B] TMA box
      // BATCHED: z is the problem's slice of the map (0 for a shared operand)
      auto load_a = [&](uint8_t *dst, const CUtensorMap *m, uint64_t *bar, int m0, int k0, int z) {
        if constexpr (!A_MN) {
          if constexpr (BATCHED) ptx::tma_load_3d(dst, m, bar, k0, m0, z);
          else ptx::tma_load_2d(dst, m, bar, k0, m0);  // box {BLOCK_K, 128}
        } else {
#pragma unroll
          for (int c = 0; c < TC_BLOCK_M / MN_ATOM; ++c) {  // boxes {MN_ATOM, BLOCK_K}
            if constexpr (BATCHED) ptx::tma_load_3d(dst + c * MN_BOX_BYTES, m, bar, m0 + c * MN_ATOM, k0, z);
            else ptx::tma_load_2d(dst + c * MN_BOX_BYTES, m, bar, m0 + c * MN_ATOM, k0);
          }
        }
      };
      auto load_b = [&](uint8_t *dst, const CUtensorMap *m, uint64_t *bar, int n0, int k0, int z) {
        if constexpr (!B_MN) {
          if constexpr (BATCHED) ptx::tma_load_3d(dst, m, bar, k0, n0, z);
          else ptx::tma_load_2d(dst, m, bar, k0, n0);  // box {BLOCK_K, TC_BLOCK_N}
        } else {
#pragma unroll
          for (int c = 0; c < TC_BLOCK_N / MN_ATOM; ++c) {
            if constexpr (BATCHED) ptx::tma_load_3d(dst + c * MN_BOX_BYTES, m, bar, n0 + c * MN_ATOM, k0, z);
            else ptx::tma_load_2d(dst + c * MN_BOX_BYTES, m, bar, n0 + c * MN_ATOM, k0);
          }
        }
      };
      for (;;) {
        const int u = next_unit(sched_phase);
        if (u < 0) break;
        int t, sp, mb, nb, kb_lo, kb_hi;
        decode_unit(u, t, sp, kb_lo, kb_hi);
        int za = 0, zb = 0;   // slices of A's and B's maps read by this tile's problem
        if constexpr (BATCHED) {
          const int bz = t / tiles_pp;
          t -= bz * tiles_pp;
          za = bz * p.map_b_a;
          zb = bz * p.map_b_b;
        }
        tile_coords(t, p.num_m_blocks, p.num_n_blocks, p.raster_g, mb, nb);
        const int m0 = mb * TC_BLOCK_M;
        const int n0 = nb * TC_BLOCK_N;
        for (int kb = kb_lo; kb < kb_hi; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          ptx::mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          uint8_t *sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t *sb = sa + Cfg::A_STAGE_BYTES;
          const int k0 = kb * BLOCK_K;
          load_a(sa, &mapA0, &full_bar[stage], m0, k0, za);
          if constexpr (NPASS == 3) load_a(sa + TC_A_TILE_BYTES, &mapA1, &full_bar[stage], m0, k0, za);
          load_b(sb, &mapB0, &full_bar[stage], n0, k0, zb);
          if constexpr (NPASS == 3) load_b(sb + Cfg::B_TILE_BYTES, &mapB1, &full_bar[stage], n0, k0, zb);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============ consumers: warpgroup g = 0, 1 multiplies and stores rows [64 g, 64 g + 64) of the CTA's 128 ============
    ptx::setmaxnreg_inc<TC_REGS_EPI>();
    const int g = (warp_idx - 4) >> 2;
    const int wq = warp_idx & 3;          // warp of the warpgroup: rows 16 wq .. 16 wq + 15 of the warpgroup's 64
    const int lr = lane >> 2;             // fragment row (and row + 8)
    const int lc = 2 * (lane & 3);        // fragment column pair 8 i + lc, 8 i + lc + 1
    constexpr int MMA_K = 32 / ESZ;                        // 8 (tf32) or 16 (16-bit) k-elements = 32 bytes per instruction
    constexpr int K_STEPS = BLOCK_K / MMA_K;               // 4
    constexpr int MN_BOX_BYTES = BLOCK_K * TC_ROW_BYTES;
    // the warpgroup's 64 rows of A: 8 KB into the tile both for K-major (64 rows of 128 B) and MN-major (the second box)
    constexpr uint32_t A_WG_BYTES = 64 * TC_ROW_BYTES;
    int stage = 0;
    uint32_t phase = 0, sched_phase = 0;
    // (BATCHED: the paired stores must stay aligned in every problem's C)
    const bool vec_ok_c = (p.csC == 1) && ((p.rsC & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & (2 * sizeof(OutT) - 1)) == 0) &&
                          (!BATCHED || (p.bsC & 1) == 0);
    float acc[TC_ACC_REGS];
#pragma unroll
    for (int j = 0; j < TC_ACC_REGS; ++j) acc[j] = 0.0f;
    for (;;) {
      int u = 0;
      if (lane == 0) u = next_unit(sched_phase);
      u = __shfl_sync(0xffffffffu, u, 0);
      if (u < 0) break;
      int t, sp, mb, nb, kb_lo, kb_hi;
      decode_unit(u, t, sp, kb_lo, kb_hi);
      int bz = 0;   // problem of the tile
      if constexpr (BATCHED) {
        bz = t / tiles_pp;
        int tl = t - bz * tiles_pp;
        tile_coords(tl, p.num_m_blocks, p.num_n_blocks, p.raster_g, mb, nb);
      } else {
        tile_coords(t, p.num_m_blocks, p.num_n_blocks, p.raster_g, mb, nb);
      }
      const int num_blocks = (kb_hi - kb_lo + p.kb_per_block - 1) / p.kb_per_block;  // accumulation blocks
      const int r_tile = 64 * g + 16 * wq + lr;                            // first row, tile-local
      const int64_t row0 = static_cast<int64_t>(mb) * TC_BLOCK_M + r_tile;  // of the product (+ 8: second)
      const int64_t col0 = static_cast<int64_t>(nb) * TC_BLOCK_N + lc;                     // column of acc[4 i] is col0 + 8 i
      const bool split_unit = sp >= 0;
      // SCALED: the abs-max words were written by earlier kernels of this stream; this thread's two row words and 32 column
      // words are fetched now and used only by the store after the K loop, so their latency hides behind the MMAs
      uint32_t amax_row[2] = {0u, 0u}, amax_col[2 * TC_BLOCK_N / 8];
      if constexpr (SCALED) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (row0 + 8 * h < p.M) amax_row[h] = p.amax_a[(BATCHED ? bz * p.amax_bs_a : 0) + row0 + 8 * h];
#pragma unroll
        for (int j = 0; j < 2 * TC_BLOCK_N / 8; ++j) {
          const int64_t c = col0 + 8 * (j >> 1) + (j & 1);
          amax_col[j] = c < p.N ? p.amax_b[(BATCHED ? bz * p.amax_bs_b : 0) + c] : 0u;
        }
      }
      float run[TC_ACC_REGS];  // running sums of this thread's fragment (registers)
#pragma unroll
      for (int j = 0; j < TC_ACC_REGS; ++j) run[j] = 0.0f;
      for (int blk = 0; blk < num_blocks; ++blk) {
        const int kb0 = kb_lo + blk * p.kb_per_block;
        const int kb1 = min(kb_hi, kb0 + p.kb_per_block);
        int prev_stage = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
          ptx::mbar_wait(&full_bar[stage], phase);
          ptx::wgmma_fence();
          const uint32_t a_addr = ptx::smem_u32(smem + stage * Cfg::STAGE_BYTES) + g * A_WG_BYTES;
          const uint32_t b_addr = ptx::smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_STAGE_BYTES);
          // three passes: the small cross terms hi*lo', lo*hi' first, then hi*hi'
#pragma unroll
          for (int pass = 0; pass < NPASS; ++pass) {
            const uint32_t a_tile = a_addr + ((NPASS == 3 && pass == 1) ? TC_A_TILE_BYTES : 0);
            const uint32_t b_tile = b_addr + ((NPASS == 3 && pass == 0) ? Cfg::B_TILE_BYTES : 0);
#pragma unroll
            for (int k = 0; k < K_STEPS; ++k) {
              // K-major: step 32 bytes inside the 128-byte swizzle row.  MN-major: step MMA_K k-rows of 128 bytes.
              const uint64_t ad = A_MN ? ptx::make_smem_desc(a_tile + k * MMA_K * TC_ROW_BYTES, MN_BOX_BYTES, 1024, ptx::kLayoutSw128)
                                       : ptx::make_smem_desc(a_tile + k * 32, 0, 1024, ptx::kLayoutSw128);
              const uint64_t bd = B_MN ? ptx::make_smem_desc(b_tile + k * MMA_K * TC_ROW_BYTES, MN_BOX_BYTES, 1024, ptx::kLayoutSw128)
                                       : ptx::make_smem_desc(b_tile + k * 32, 0, 1024, ptx::kLayoutSw128);
              const uint32_t accum = (kb == kb0 && pass == 0 && k == 0) ? 0u : 1u;
              if constexpr (ESZ == 4) ptx::wgmma_m64n128k8_tf32(acc, ad, bd, accum);
              else if constexpr (FMT16 == ptx::kFmtF16) ptx::wgmma_m64n128k16_f16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd, accum);
              else ptx::wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, ad, bd, accum);
            }
          }
          ptx::wgmma_commit();
          // at most this k-tile's group still runs: the previous k-tile's stage goes back to the producer
          ptx::wgmma_wait<1>();
          if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        ptx::wgmma_wait<0>();
        ptx::wgmma_hold(acc);
        if (prev_stage >= 0 && lane == 0) ptx::mbar_arrive(&empty_bar[prev_stage]);
        // block complete: added (IEEE round-to-nearest) to the running sums, see the top of this file
#pragma unroll
        for (int j = 0; j < TC_ACC_REGS; ++j) run[j] = __fadd_rn(run[j], acc[j]);
      }
      // where this thread's sums go.  Direct tile: C, with alpha / beta / bias / activation.  Split unit: plane
      // [sp][t - n_direct] of the workspace, tile-local rows / columns, raw (only the operand scales are undone).
      float alpha_r[2] = {split_unit ? 1.0f : p.alpha, split_unit ? 1.0f : p.alpha};
      if constexpr (SCALED) {
#pragma unroll
        for (int h = 0; h < 2; ++h) alpha_r[h] *= f16x2_unscale(amax_row[h]);
      }
      const float beta_u = split_unit ? 0.0f : p.beta;
      const bool has_epi = !split_unit && ((p.epi.bias != nullptr) || (p.epi.act != 0));
      float *ws_base = nullptr;
      if (split_unit) {
        const int64_t plane = static_cast<int64_t>(sp) * (num_tiles - p.n_direct) + (t - p.n_direct);
        ws_base = p.split_ws + (plane * TC_BLOCK_M + r_tile) * TC_BLOCK_N + lc;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = row0 + 8 * h;
        if (!split_unit && row >= p.M) continue;
        const float row_bias = (has_epi && p.epi.bias && p.epi.bias_per_row) ? p.epi.bias[row] : 0.0f;
        OutT *crow = split_unit ? nullptr : reinterpret_cast<OutT *>(p.C) + (BATCHED ? bz * p.bsC : 0) + row * p.rsC;
#pragma unroll
        for (int i = 0; i < TC_BLOCK_N / 8; ++i) {
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            v[e] = alpha_r[h] * run[4 * i + 2 * h + e];
            if constexpr (SCALED) v[e] *= f16x2_unscale(amax_col[2 * i + e]);
          }
          if (split_unit) {   // (rows past M: zeros into the workspace)
            *reinterpret_cast<float2 *>(ws_base + 8 * h * TC_BLOCK_N + 8 * i) = make_float2(v[0], v[1]);
            continue;
          }
          const int64_t c = col0 + 8 * i;
          if (c >= p.N) continue;
          const bool pair_ok = vec_ok_c && c + 1 < p.N;
          OutT *dst = crow + c * p.csC;
          if (beta_u != 0.0f) {
            float o[2] = {0.0f, 0.0f};
            if constexpr (sizeof(OutT) == 4) {
              if (pair_ok) { const float2 w = *reinterpret_cast<const float2 *>(dst); o[0] = w.x; o[1] = w.y; }
              else { o[0] = dst[0]; if (c + 1 < p.N) o[1] = dst[p.csC]; }
            } else {
              o[0] = bf16_bits_to_f32(dst[0]);
              if (c + 1 < p.N) o[1] = bf16_bits_to_f32(dst[pair_ok ? 1 : p.csC]);
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) v[e] = fmaf(beta_u, o[e], v[e]);
          }
          if (has_epi) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float bv = (p.epi.bias && !p.epi.bias_per_row) ? (c + e < p.N ? p.epi.bias[c + e] : 0.0f) : row_bias;
              v[e] = epi_act(v[e] + bv, p.epi.act);
            }
          }
          if constexpr (sizeof(OutT) == 4) {
            if (pair_ok) *reinterpret_cast<float2 *>(dst) = make_float2(v[0], v[1]);
            else { dst[0] = v[0]; if (c + 1 < p.N) dst[p.csC] = v[1]; }
          } else {
            if (pair_ok) *reinterpret_cast<uint32_t *>(dst) = f32_to_bf16_bits(v[0]) | (static_cast<uint32_t>(f32_to_bf16_bits(v[1])) << 16);
            else { dst[0] = f32_to_bf16_bits(v[0]); if (c + 1 < p.N) dst[p.csC] = f32_to_bf16_bits(v[1]); }
          }
        }
      }
    }
  }

  __syncthreads();
}

}  // namespace lb200
