// split.cuh -- HBM-bound operand preparation kernels.
//
//  split_rows_tf32 : elementwise hi/lo split of an operand that TMA can read as is
//                    (one stride == 1): hi = tf32_rna(x), lo = tf32_rna(x - hi).  The
//                    operand keeps its major-ness; outputs are compact [R][ld].
//  pack_general    : gather of an operand with arbitrary (row, col) element strides
//                    (neither is 1, misaligned base, odd leading dimension, negative
//                    strides ...) into a compact row-major [R][ld] array, optionally
//                    hi/lo split on the way.  This is the one place where the
//                    reference's pack_A_mc_kc / pack_B_kc_nc (gemm_packing.nim:24-94)
//                    survives: as a single coalesced pass for the operands the TMA
//                    engine cannot address.
// Both are pure streaming kernels: grid = multiple of the SM count, 16-byte
// accesses where alignment allows.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "f16_scale.cuh"
#include "ptx.cuh"
#include "tc_params.h"

namespace lb200 {

#ifndef LB200_HOST_EMULATION
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
#else   // tests/emu: round to nearest, ties away from zero, onto 10 mantissa bits (finite inputs)
inline float tf32_rna(float x) {
  uint32_t u = __float_as_uint(x);
  if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & 0xffffe000u;
  return __uint_as_float(u);
}
#endif

// low piece of the hi/lo split; 0 when hi is not finite (x = +-inf, or |x| so close to FLT_MAX that hi rounded up to inf:
// x - hi would be NaN and poison the whole row / column of C, where the reference's FMA chain gives +-inf)
__device__ __forceinline__ float tf32_lo(float x, float hi) {
  return ((__float_as_uint(hi) & 0x7f800000u) == 0x7f800000u) ? 0.0f : tf32_rna(x - hi);
}

// ---- prologue fusion: an elementwise op applied to the operand while it is prepared ---------------------------------
// The kernels below take `template <bool HAS_OP>` (false: the plain kernel, which never reads `op`) and an OperandOp.
// Element (r, c) of the kernel's [R][Cc] view has its aux element at aux[r * aux_sr + c * aux_sc]; the row kernels read aux
// with the operand's own offsets (aux_sr = src_ld, aux_sc = 1, 16-byte aligned), the gather with any strides.
struct OperandOp {
  int op = 0;                   // LASER_B200_OP_* (1 .. 6)
  const float *aux = nullptr;   // derivative ops (4 .. 6) only
  int64_t aux_sr = 0, aux_sc = 0;
};
// Ops 1-3: the formulas of the epilogue's activations (gemm_tc.cuh: epi_act).  Ops 4-6: every operation rounded on its
// own, in the order written (no contraction), so that the exact path is bit-identical to a step-by-step restatement.
// (tanhf / expf out of line: inlined into every element of the unrolled row kernels they make them spill)
#ifndef LB200_HOST_EMULATION
static __device__ __noinline__ float operand_act(int op, float x) {
#else
inline float operand_act(int op, float x) {
#endif
  return op == 2 ? tanhf(x) : 1.0f / (1.0f + expf(-x));
}
__device__ __forceinline__ float operand_op(int op, float x, float y) {
  switch (op) {
    case 1: return fmaxf(x, 0.0f);
    case 2:
    case 3: return operand_act(op, x);
    case 4: return y > 0.0f ? x : 0.0f;                               // a select: inf * 0 never happens
    case 5: return __fmul_rn(x, __fsub_rn(1.0f, __fmul_rn(y, y)));
    case 6: return __fmul_rn(x, __fmul_rn(y, __fsub_rn(1.0f, y)));
    default: return x;
  }
}
__device__ __forceinline__ float4 load_row_vec(const float *row, int64_t c, int64_t Cc) {
  float4 v;
  if (c + 4 <= Cc) {
    v = *reinterpret_cast<const float4 *>(row + c);
  } else {   // ragged end of the row: one to three elements
    v.x = row[c];
    v.y = (c + 1 < Cc) ? row[c + 1] : 0.0f;
    v.z = (c + 2 < Cc) ? row[c + 2] : 0.0f;
    v.w = 0.0f;
  }
  return v;
}
// the op on four consecutive elements c .. c+3 of row r (v: the operand's values, 0 past Cc); elements past Cc stay 0 (they
// are the padding of the prepared arrays)
__device__ __forceinline__ float4 op_vec(const OperandOp &op, float4 v, int64_t r, int64_t c, int64_t Cc) {
  const float4 y = op.aux ? load_row_vec(op.aux + r * op.aux_sr, c, Cc) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  v.x = operand_op(op.op, v.x, y.x);
  v.y = (c + 1 < Cc) ? operand_op(op.op, v.y, y.y) : 0.0f;
  v.z = (c + 2 < Cc) ? operand_op(op.op, v.z, y.z) : 0.0f;
  v.w = (c + 3 < Cc) ? operand_op(op.op, v.w, y.w) : 0.0f;
  return v;
}

// ---- batched preparation: the operands of bt.n problems in one launch ------------------------------------------------
// The kernels below also take `template <bool BATCHED>` (false: one problem, `bt` never read).  A BATCHED kernel prepares bt.n
// problems whose [R][Cc] views are bt.bs elements apart (aux: bt.aux_bs), and writes what one problem's launch writes,
// stacked: pieces [bt.n * R][ld], per-row scale words [bt.n * R], per-column scale words [bt.n][Cc].
struct Batch {
  int64_t n = 1;
  int64_t bs = 0, aux_bs = 0;
};
// stacked row g -> its problem's source (and aux) and the row within the problem
template <bool BATCHED>
__device__ __forceinline__ int64_t batch_row(int64_t g, int64_t R, const Batch &bt, const float *&src, OperandOp &op) {
  if constexpr (BATCHED) {
    const int64_t b = g / R;
    src += b * bt.bs;
    if (op.aux) op.aux += b * bt.aux_bs;
    return g - b * R;
  } else {
    return g;
  }
}

// src: R rows of Cc contiguous floats, leading dimension src_ld (16-byte aligned rows).
// hi/lo: compact, leading dimension dst_ld (multiple of 4).
template <bool HAS_OP = false, bool BATCHED = false>
__global__ void __launch_bounds__(256)
split_rows_tf32_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld,
                       float *__restrict__ hi, float *__restrict__ lo, int64_t dst_ld, OperandOp op = OperandOp(),
                       Batch bt = Batch()) {
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int64_t vec_per_row = (Cc + 3) >> 2;
  const int64_t total = (BATCHED ? bt.n * R : R) * vec_per_row;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / vec_per_row;
    const int64_t c = (i - r * vec_per_row) << 2;
    const float *sp = src;
    OperandOp o = op;
    const int64_t rl = batch_row<BATCHED>(r, R, bt, sp, o);
    const float *s = sp + rl * src_ld + c;
    float4 v;
    if (c + 4 <= Cc) {
      v = *reinterpret_cast<const float4 *>(s);
    } else {
      v.x = s[0];
      v.y = (c + 1 < Cc) ? s[1] : 0.0f;
      v.z = (c + 2 < Cc) ? s[2] : 0.0f;
      v.w = 0.0f;
    }
    if constexpr (HAS_OP && BATCHED) v = op_vec(o, v, rl, c, Cc);
    else if constexpr (HAS_OP) v = op_vec(op, v, r, c, Cc);
    float4 h, l;
    h.x = tf32_rna(v.x); l.x = tf32_lo(v.x, h.x);
    h.y = tf32_rna(v.y); l.y = tf32_lo(v.y, h.y);
    h.z = tf32_rna(v.z); l.z = tf32_lo(v.z, h.z);
    h.w = tf32_rna(v.w); l.w = tf32_lo(v.w, h.w);
    *reinterpret_cast<float4 *>(hi + r * dst_ld + c) = h;
    *reinterpret_cast<float4 *>(lo + r * dst_ld + c) = l;
  }
}

// ---- LASER_B200_PATH_F16X3: two fp16 pieces of the SCALED operand (f16_scale.cuh) -------------------------
// One scale per mn index of the operand (row of A / column of B), i.e. one abs-max over k per mn.  The prepared
// layout is [R][Cc] with contiguous rows (as for the other split kernels); mn runs along R for a K-major operand
// (PER_COL = false: one word per row) and along Cc for an MN-major one (PER_COL = true: one word per column).
// out[] holds fp32 bit patterns of non-negative finite numbers (ordered like unsigned integers), zeroed by the
// host before the launch, combined with atomicMax after a local reduction.
__device__ __forceinline__ uint32_t finite_abs_bits(float f) {
  const uint32_t a = __float_as_uint(f) & 0x7fffffffu;
  return a < 0x7f800000u ? a : 0u;     // infinities and NaNs do not set a scale (they propagate as such)
}
constexpr int ABSMAX_ROW_CHUNK = 1024;   // floats of one row reduced by one warp pass (32 lanes x 8 x float4)
constexpr int ABSMAX_COL_ROWS = 64;      // rows of a 4-column strip reduced by one thread
template <bool PER_COL, bool HAS_OP = false, bool BATCHED = false>
__global__ void __launch_bounds__(256)
absmax_mn_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld, uint32_t *__restrict__ out,
                 OperandOp op = OperandOp(), Batch bt = Batch()) {
  static_assert(PER_COL || !HAS_OP, "a K-major operand with an op takes the fused row kernel");
  static_assert(PER_COL || !BATCHED, "a K-major operand takes the fused row kernel");
  if constexpr (!PER_COL) {
    // warp w takes (row, chunk) items; lanes read float4s 128 floats apart; butterfly max; one atomic per item
    const int lane = threadIdx.x & 31;
    const int64_t chunks = (Cc + ABSMAX_ROW_CHUNK - 1) / ABSMAX_ROW_CHUNK;
    const int64_t items = R * chunks;
    const int64_t warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t it = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; it < items; it += warps) {
      const int64_t r = it / chunks;
      const int64_t c0 = (it - r * chunks) * ABSMAX_ROW_CHUNK;
      const float *row = src + r * src_ld;
      uint32_t m = 0u;
#pragma unroll
      for (int i = 0; i < ABSMAX_ROW_CHUNK / 128; ++i) {
        const int64_t c = c0 + i * 128 + lane * 4;
        if (c + 4 <= Cc) {
          const float4 v = *reinterpret_cast<const float4 *>(row + c);
          m = max(max(m, finite_abs_bits(v.x)), max(finite_abs_bits(v.y), max(finite_abs_bits(v.z), finite_abs_bits(v.w))));
        } else if (c < Cc) {   // ragged end of the row: one to three elements
          m = max(m, finite_abs_bits(row[c]));
          if (c + 1 < Cc) m = max(m, finite_abs_bits(row[c + 1]));
          if (c + 2 < Cc) m = max(m, finite_abs_bits(row[c + 2]));
        }
      }
      float mf = __uint_as_float(m);     // non-negative finite: fmaxf orders them like the integers
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o));
      if (lane == 0) atomicMax(out + r, __float_as_uint(mf));
    }
  } else {
    // thread takes (4-column strip, block of ABSMAX_COL_ROWS rows) items: adjacent threads read adjacent float4s
    // (BATCHED: row blocks of one problem at a time, rb counting over the problems' blocks)
    const int64_t strips = (Cc + 3) >> 2;
    const int64_t rblocks = (R + ABSMAX_COL_ROWS - 1) / ABSMAX_COL_ROWS;
    const int64_t items = strips * (BATCHED ? bt.n * rblocks : rblocks);
    for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < items;
         it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
      int64_t rb = it / strips;
      const int64_t c = (it - rb * strips) << 2;
      const float *src_b = src;
      OperandOp o = op;
      uint32_t *out_b = out;
      if constexpr (BATCHED) {
        const int64_t b = rb / rblocks;
        rb -= b * rblocks;
        batch_row<true>(b * R, R, bt, src_b, o);
        out_b += b * Cc;
      }
      const int64_t r1 = (rb + 1) * ABSMAX_COL_ROWS < R ? (rb + 1) * ABSMAX_COL_ROWS : R;
      uint32_t m0 = 0u, m1 = 0u, m2 = 0u, m3 = 0u;
      for (int64_t r = rb * ABSMAX_COL_ROWS; r < r1; ++r) {
        const float *s = src_b + r * src_ld + c;
        if constexpr (HAS_OP) {   // the scale is taken over the op's output (padding lanes are 0)
          const float4 v = op_vec(BATCHED ? o : op, load_row_vec(src_b + r * src_ld, c, Cc), r, c, Cc);
          m0 = max(m0, finite_abs_bits(v.x)); m1 = max(m1, finite_abs_bits(v.y));
          m2 = max(m2, finite_abs_bits(v.z)); m3 = max(m3, finite_abs_bits(v.w));
        } else if (c + 4 <= Cc) {
          const float4 v = *reinterpret_cast<const float4 *>(s);
          m0 = max(m0, finite_abs_bits(v.x)); m1 = max(m1, finite_abs_bits(v.y));
          m2 = max(m2, finite_abs_bits(v.z)); m3 = max(m3, finite_abs_bits(v.w));
        } else {
          m0 = max(m0, finite_abs_bits(s[0]));
          if (c + 1 < Cc) m1 = max(m1, finite_abs_bits(s[1]));
          if (c + 2 < Cc) m2 = max(m2, finite_abs_bits(s[2]));
        }
      }
      atomicMax(out_b + c, m0);
      if (c + 1 < Cc) atomicMax(out_b + c + 1, m1);
      if (c + 2 < Cc) atomicMax(out_b + c + 2, m2);
      if (c + 3 < Cc) atomicMax(out_b + c + 3, m3);
    }
  }
}

__device__ __forceinline__ void store_f16x2_vec4(float4 v, float sx, float sy, float sz, float sw, uint16_t *hrow, uint16_t *lrow,
                                                 int64_t c) {
  uint2 h, l;
  f16x2_pieces2(__fmul_rn(v.x, sx), __fmul_rn(v.y, sy), h.x, l.x);
  f16x2_pieces2(__fmul_rn(v.z, sz), __fmul_rn(v.w, sw), h.y, l.y);
  *reinterpret_cast<uint2 *>(hrow + c) = h;
  *reinterpret_cast<uint2 *>(lrow + c) = l;
}
__device__ __forceinline__ void store_f16x2_vec(float4 v, float s, uint16_t *hrow, uint16_t *lrow, int64_t c) {
  store_f16x2_vec4(v, s, s, s, s, hrow, lrow, c);
}

// K-major operand (rows contiguous, ONE scale per row): abs-max, scale and split in a single pass over HBM.  A group
// of threads -- a warp for short rows, the whole CTA otherwise -- reads its row into registers (F16ROWS_MAXV float4 per
// thread; what is left of a longer row is read twice, the second time from L2), reduces the abs-max, writes the word and
// both fp16 pieces: 4 bytes read + 4 written per element, against 8 + 4 for abs-max and split as two kernels.
constexpr int F16ROWS_MAXV = 8;
template <int GROUP, bool HAS_OP = false, bool BATCHED = false>
__global__ void __launch_bounds__(256, 4)
f16x2_rows_fused_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *__restrict__ hb,
                        uint16_t *__restrict__ lb, int64_t ld_b, uint32_t *__restrict__ absmax, OperandOp op = OperandOp(),
                        Batch bt = Batch()) {
  static_assert(GROUP == 32 || GROUP == 256, "a warp or the CTA per row");
  __shared__ uint32_t red[2][8];
  ptx::griddep_launch_dependents();
  const int tid = static_cast<int>(threadIdx.x) % GROUP;
  const int64_t per_cta = 256 / GROUP;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * per_cta + static_cast<int64_t>(threadIdx.x) / GROUP;
  const int64_t step = static_cast<int64_t>(gridDim.x) * per_cta;
  const int64_t nvec = (Cc + 3) >> 2;
  int parity = 0;
  // GROUP == 256: every thread of the CTA runs the same number of iterations (the loop holds a __syncthreads)
  const int64_t rows = BATCHED ? bt.n * R : R;
  for (int64_t r = first; r < rows; r += step) {
    const float *sp = src;
    OperandOp o = op;
    const int64_t rl = batch_row<BATCHED>(r, R, bt, sp, o);
    const float *row = sp + rl * src_ld;
    float4 v[F16ROWS_MAXV];
    uint32_t m = 0u;
#pragma unroll
    for (int i = 0; i < F16ROWS_MAXV; ++i) {
      const int64_t idx = tid + static_cast<int64_t>(i) * GROUP;
      if (idx < nvec) {
        v[i] = load_row_vec(row, idx << 2, Cc);
        if constexpr (HAS_OP) v[i] = op_vec(o, v[i], rl, idx << 2, Cc);
        m = max(max(m, finite_abs_bits(v[i].x)), max(finite_abs_bits(v[i].y), max(finite_abs_bits(v[i].z), finite_abs_bits(v[i].w))));
      }
    }
    for (int64_t idx = tid + static_cast<int64_t>(F16ROWS_MAXV) * GROUP; idx < nvec; idx += GROUP) {
      float4 t = load_row_vec(row, idx << 2, Cc);
      if constexpr (HAS_OP) t = op_vec(o, t, rl, idx << 2, Cc);
      m = max(max(m, finite_abs_bits(t.x)), max(finite_abs_bits(t.y), max(finite_abs_bits(t.z), finite_abs_bits(t.w))));
    }
    float mf = __uint_as_float(m);     // non-negative finite: fmaxf orders them like the integers
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o));
    m = __float_as_uint(mf);
    if constexpr (GROUP == 256) {
      if ((threadIdx.x & 31) == 0) red[parity][threadIdx.x >> 5] = m;
      __syncthreads();
#pragma unroll
      for (int w = 0; w < 8; ++w) m = max(m, red[parity][w]);
      parity ^= 1;   // the next row uses the other buffer: one barrier per row is enough
    }
    if (tid == 0) absmax[r] = m;
    const float s = f16x2_scale(m);
    uint16_t *hrow = hb + r * ld_b, *lrow = lb + r * ld_b;
#pragma unroll
    for (int i = 0; i < F16ROWS_MAXV; ++i) {
      const int64_t idx = tid + static_cast<int64_t>(i) * GROUP;
      if (idx < nvec) store_f16x2_vec(v[i], s, hrow, lrow, idx << 2);
    }
    for (int64_t idx = tid + static_cast<int64_t>(F16ROWS_MAXV) * GROUP; idx < nvec; idx += GROUP) {
      if constexpr (HAS_OP) store_f16x2_vec(op_vec(o, load_row_vec(row, idx << 2, Cc), rl, idx << 2, Cc), s, hrow, lrow, idx << 2);
      else store_f16x2_vec(load_row_vec(row, idx << 2, Cc), s, hrow, lrow, idx << 2);
    }
  }
}

// The same single pass with the rows PREFETCHED by the copy engine: thread 0 keeps F16RING_BUFS rows of the CTA in flight as
// bulk copies into a shared-memory ring (cp.async.bulk, one instruction per row, completion on an mbarrier), the CTA picks a
// landed row up into registers, reduces its abs-max (the one __syncthreads per row doubles as "the buffer is free again":
// every thread has read its part by then), scales, splits and stores.  The register-only kernel above alternates between
// "all loads in flight" and "converting": 47 % of the HBM rate at 8192 x 8192 (ncu, round 2); here the loads of the next
// rows never stop.  Needs 16-byte aligned rows of at most 256 * F16ROWS_MAXV float4 (the host checks).
constexpr int F16RING_BUFS = 3;
__global__ void __launch_bounds__(256, 2)
f16x2_rows_ring_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *__restrict__ hb,
                       uint16_t *__restrict__ lb, int64_t ld_b, uint32_t *__restrict__ absmax) {
  LB200_DYN_SMEM(uint8_t, ring_raw);
  __shared__ uint32_t red[2][8];
  __shared__ uint64_t full[F16RING_BUFS];   // (8-byte aligned by type)
  ptx::griddep_launch_dependents();
  uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ring_raw) + 127) & ~static_cast<uintptr_t>(127));
  const uint32_t row_bytes = static_cast<uint32_t>(Cc) * 4u;
  const uint32_t buf_bytes = (row_bytes + 127u) & ~127u;
  const int tid = static_cast<int>(threadIdx.x);
  const int64_t first = blockIdx.x, step = gridDim.x;
  const int nvec = static_cast<int>(Cc >> 2);
  if (tid == 0) {
    for (int i = 0; i < F16RING_BUFS; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_barrier_init();
    for (int i = 0; i < F16RING_BUFS; ++i) {
      const int64_t r = first + i * step;
      if (r < R) {
        ptx::mbar_arrive_expect_tx(&full[i], row_bytes);
        ptx::bulk_load_1d(ring + i * buf_bytes, src + r * src_ld, row_bytes, &full[i]);
      }
    }
  }
  __syncthreads();
  int b = 0, parity = 0;
  uint32_t phase = 0;
  for (int64_t r = first; r < R; r += step) {
    ptx::mbar_wait(&full[b], phase);
    const float4 *row = reinterpret_cast<const float4 *>(ring + b * buf_bytes);
    float4 v[F16ROWS_MAXV];
    uint32_t m = 0u;
#pragma unroll
    for (int i = 0; i < F16ROWS_MAXV; ++i) {
      const int idx = tid + i * 256;
      if (idx < nvec) {
        v[i] = row[idx];
        m = max(max(m, finite_abs_bits(v[i].x)), max(finite_abs_bits(v[i].y), max(finite_abs_bits(v[i].z), finite_abs_bits(v[i].w))));
      }
    }
    float mf = __uint_as_float(m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o));
    if ((tid & 31) == 0) red[parity][tid >> 5] = __float_as_uint(mf);
    __syncthreads();   // the maxima of the eight warps are there AND every thread has taken its part of the row out of the ring
    if (tid == 0) {
      const int64_t rn = r + F16RING_BUFS * step;
      if (rn < R) {
        ptx::mbar_arrive_expect_tx(&full[b], row_bytes);
        ptx::bulk_load_1d(ring + b * buf_bytes, src + rn * src_ld, row_bytes, &full[b]);
      }
    }
    m = 0u;
#pragma unroll
    for (int w = 0; w < 8; ++w) m = max(m, red[parity][w]);
    parity ^= 1;
    if (tid == 0) absmax[r] = m;
    const float s = f16x2_scale(m);
    uint16_t *hrow = hb + r * ld_b, *lrow = lb + r * ld_b;
#pragma unroll
    for (int i = 0; i < F16ROWS_MAXV; ++i) {
      const int idx = tid + i * 256;
      if (idx < nvec) store_f16x2_vec(v[i], s, hrow, lrow, static_cast<int64_t>(idx) << 2);
    }
    if (++b == F16RING_BUFS) { b = 0; phase ^= 1u; }
  }
}
inline size_t f16x2_rows_ring_smem(int64_t Cc) { return static_cast<size_t>(F16RING_BUFS) * ((Cc * 4 + 127) / 128 * 128) + 128; }
inline bool f16x2_rows_ring_ok(const float *src, int64_t Cc, int64_t src_ld) {
  return Cc % 4 == 0 && src_ld % 4 == 0 && Cc > 4 * 32 * F16ROWS_MAXV && Cc <= 4 * 256 * F16ROWS_MAXV &&
         (reinterpret_cast<uintptr_t>(src) & 15) == 0;
}

// hb = fp16(x * 2^s), lb = fp16(x * 2^s - hb) with s from the abs-max word of the element's mn index
// (f16_scale.cuh): x * 2^s = hb + lb + r, |r| <= 2^-22 |x * 2^s| for elements within 2^-17 of their row's /
// column's maximum.  [R][Cc] row-contiguous arrays in and out.  Work item = (strip of 256 columns, block of
// SPLIT_ROWS rows): a thread owns 4 columns of the strip -- for PER_COL their four scales are computed once -- and walks
// the rows of the block, adjacent threads reading adjacent float4s.
constexpr int SPLIT_ROWS = 64;
template <bool PER_COL, bool HAS_OP = false, bool BATCHED = false>
__global__ void __launch_bounds__(256)
split_rows_f16x2_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld,
                        uint16_t *__restrict__ hb, uint16_t *__restrict__ lb, int64_t ld_b,
                        const uint32_t *__restrict__ absmax, OperandOp op = OperandOp(), Batch bt = Batch()) {
  static_assert(PER_COL || !BATCHED, "a K-major operand takes the fused row kernel");
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int tx = static_cast<int>(threadIdx.x) & 63, ty = static_cast<int>(threadIdx.x) >> 6;   // 64 float4 columns x 4 row lanes
  const int64_t strips = (Cc + 255) >> 8;
  const int64_t rblocks = (R + SPLIT_ROWS - 1) / SPLIT_ROWS;
  for (int64_t it = blockIdx.x; it < strips * (BATCHED ? bt.n * rblocks : rblocks); it += gridDim.x) {
    int64_t rb = it / strips;
    const int64_t c = ((it - rb * strips) << 8) + (tx << 2);
    if (c >= Cc) continue;
    // (BATCHED: row block rb of problem b; its pieces are rows b * R + r of hb / lb, its words absmax[b * Cc ..])
    const float *src_b = src;
    OperandOp o = op;
    const uint32_t *absmax_b = absmax;
    uint16_t *hb_b = hb, *lb_b = lb;
    if constexpr (BATCHED) {
      const int64_t b = rb / rblocks;
      rb -= b * rblocks;
      batch_row<true>(b * R, R, bt, src_b, o);
      absmax_b += b * Cc;
      hb_b += b * R * ld_b;
      lb_b += b * R * ld_b;
    }
    float sx = 1.0f, sy = 1.0f, sz = 1.0f, sw = 1.0f;
    if constexpr (PER_COL) {
      sx = f16x2_scale(absmax_b[c]);
      sy = (c + 1 < Cc) ? f16x2_scale(absmax_b[c + 1]) : 1.0f;
      sz = (c + 2 < Cc) ? f16x2_scale(absmax_b[c + 2]) : 1.0f;
      sw = (c + 3 < Cc) ? f16x2_scale(absmax_b[c + 3]) : 1.0f;
    }
    const int64_t r1 = (rb + 1) * SPLIT_ROWS < R ? (rb + 1) * SPLIT_ROWS : R;
#pragma unroll 4
    for (int64_t r = rb * SPLIT_ROWS + ty; r < r1; r += 4) {
      float4 v = load_row_vec(src_b + r * src_ld, c, Cc);
      if constexpr (HAS_OP) v = op_vec(o, v, r, c, Cc);
      if constexpr (!PER_COL) sx = sy = sz = sw = f16x2_scale(absmax_b[r]);
      store_f16x2_vec4(v, sx, sy, sz, sw, hb_b + r * ld_b, lb_b + r * ld_b, c);
    }
  }
}

// dst[r*ld + c] = src[r*sr + c*sc] for r < R, c < Cc.  32 x 32 tiles through shared
// memory so that both the gather (along whichever source stride is smaller) and the
// store (along c) are coalesced.  SPLIT: also write lo (fp32 only).
// MODE 0: plain copy; 1: fp32 hi/lo pieces (dst, dst_lo).
// HAS_OP (fp32): the op is applied to each element as it is gathered (aux read with its own strides).
template <typename T, int MODE, bool HAS_OP = false, bool BATCHED = false>
__global__ void __launch_bounds__(256)
pack_general_kernel(const T *__restrict__ src, int64_t R, int64_t Cc, int64_t sr, int64_t sc,
                    T *__restrict__ dst, T *__restrict__ dst_lo, int64_t ld, int read_along_r, OperandOp op = OperandOp(),
                    Batch bt = Batch()) {
  static_assert(!HAS_OP || sizeof(T) == 4, "operand ops are fp32 only");
  static_assert(!BATCHED || sizeof(T) == 4, "batched operands are fp32 only");
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  __shared__ T tile[32][33];
  const int64_t tiles_c = (Cc + 31) >> 5;
  const int64_t tiles_r = (R + 31) >> 5;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int64_t t = blockIdx.x; t < tiles_r * tiles_c * (BATCHED ? bt.n : 1); t += gridDim.x) {
    int64_t r0 = (t / tiles_c) << 5;
    const int64_t c0 = (t % tiles_c) << 5;
    const T *src_t = src;
    T *dst_t = dst, *dlo_t = dst_lo;
    OperandOp o = op;
    if constexpr (BATCHED) {   // a tile of problem b: read from its operand and aux, written to rows b * R + r of dst
      const int64_t b = (t / tiles_c) / tiles_r;
      r0 -= (b * tiles_r) << 5;
      src_t += b * bt.bs;
      if (o.aux) o.aux += b * bt.aux_bs;
      dst_t += b * R * ld;
      if constexpr (MODE == 1) dlo_t += b * R * ld;
    }
    if (read_along_r) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t c = c0 + ty + i * 8, r = r0 + tx;
        if constexpr (HAS_OP) {
          if (r < R && c < Cc)
            tile[tx][ty + i * 8] = operand_op(o.op, src_t[r * sr + c * sc], o.aux ? o.aux[r * o.aux_sr + c * o.aux_sc] : 0.0f);
        } else {
          if (r < R && c < Cc) tile[tx][ty + i * 8] = src_t[r * sr + c * sc];
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t r = r0 + ty + i * 8, c = c0 + tx;
        if constexpr (HAS_OP) {
          if (r < R && c < Cc)
            tile[ty + i * 8][tx] = operand_op(o.op, src_t[r * sr + c * sc], o.aux ? o.aux[r * o.aux_sr + c * o.aux_sc] : 0.0f);
        } else {
          if (r < R && c < Cc) tile[ty + i * 8][tx] = src_t[r * sr + c * sc];
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty + i * 8, c = c0 + tx;
      if (r < R && c < Cc) {
        const T v = tile[ty + i * 8][tx];
        if constexpr (MODE == 1) {
          const float h = tf32_rna(v);
          dst_t[r * ld + c] = h;
          dlo_t[r * ld + c] = tf32_lo(v, h);
        } else {
          dst_t[r * ld + c] = v;
        }
      }
    }
    __syncthreads();
  }
}

// Second half of a split-K GEMM (tc_params.h): C <- act(alpha * sum_s ws[s][i] + beta * C + bias) over the split tiles
// n_direct + i, i < n_tail, planes added in the fixed order s = 0 .. S-1 (deterministic).  ws: [S][n_tail][TC_BLOCK_M][TC_BLOCK_N]
// fp32, tile-local.  Item = four consecutive columns of one tile row.  BATCHED: tile t of the launch is tile t % (num_m * num_n)
// of problem t / (num_m * num_n), whose C starts bsC elements after the previous problem's (tc_params.h).
template <bool BATCHED = false>
__global__ void __launch_bounds__(256)
splitk_tail_reduce_kernel(const float *__restrict__ ws, int S, int n_tail, int n_direct, int num_m, int num_n, int raster_g,
                          int64_t M, int64_t N, float alpha, float beta, float *__restrict__ C, int64_t rsC,
                          int64_t csC, const float *__restrict__ bias, int bias_per_row, int act, int64_t bsC = 0) {
  constexpr int V = TC_BLOCK_N / 4;   // float4 per tile row
  const int64_t per_tile = static_cast<int64_t>(TC_BLOCK_M) * V;
  const int64_t total = static_cast<int64_t>(n_tail) * per_tile;
  const int64_t plane = total * 4;    // floats between consecutive split planes
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ti = static_cast<int>(i / per_tile);
    const int64_t rem = i - ti * per_tile;
    const int r_l = static_cast<int>(rem / V), c4 = static_cast<int>(rem - static_cast<int64_t>(r_l) * V);
    int mb, nb, t = n_direct + ti;
    float *Cb = C;
    if constexpr (BATCHED) {
      const int b = t / (num_m * num_n);
      t -= b * (num_m * num_n);
      Cb += b * bsC;
    }
    tile_coords(t, num_m, num_n, raster_g, mb, nb);
    const int64_t r = static_cast<int64_t>(mb) * TC_BLOCK_M + r_l, c = static_cast<int64_t>(nb) * TC_BLOCK_N + 4 * c4;
    if (r >= M || c >= N) continue;
    const float *src = ws + i * 4;
    float4 sum = *reinterpret_cast<const float4 *>(src);
    for (int sp = 1; sp < S; ++sp) {
      const float4 t = *reinterpret_cast<const float4 *>(src + sp * plane);
      sum.x = __fadd_rn(sum.x, t.x); sum.y = __fadd_rn(sum.y, t.y); sum.z = __fadd_rn(sum.z, t.z); sum.w = __fadd_rn(sum.w, t.w);
    }
    const float sv[4] = {sum.x, sum.y, sum.z, sum.w};
    float *dst = Cb + r * rsC + c * csC;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (c + e < N) {
        float v = alpha * sv[e];
        if (beta != 0.0f) v = fmaf(beta, dst[e * csC], v);
        if (bias != nullptr || act != 0) {
          if (bias) v += bias_per_row ? bias[r] : bias[c + e];
          if (act == 1) v = fmaxf(v, 0.0f);
          else if (act == 2) v = tanhf(v);
          else if (act == 3) v = 1.0f / (1.0f + expf(-v));
        }
        dst[e * csC] = v;
      }
    }
  }
}

// counter-based uniform fill, bit-identical to oracle_fill_uniform_f32
__device__ __forceinline__ uint64_t splitmix64_dev(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void __launch_bounds__(256)
fill_uniform_f32_kernel(float *__restrict__ dst, int64_t n, uint64_t seed, float lo, float hi) {
  const float span = __fsub_rn(hi, lo);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint64_t h = splitmix64_dev(seed * 0xD1342543DE82EF95ull + static_cast<uint64_t>(i));
    const float u = __fmul_rn(static_cast<float>(static_cast<uint32_t>(h >> 40)), 1.0f / 16777216.0f);
    dst[i] = __fmaf_rn(u, span, lo);
  }
}

}  // namespace lb200
