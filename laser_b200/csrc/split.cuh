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

#include <type_traits>

#include "f16_scale.cuh"
#include "layers.cuh"
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

// ---- batch-reduced preparation: the problems concatenated along k ----------------------------------------------------
// The kernels below also take `template <bool CONCAT>` (only with BATCHED; false: the kernels above and their batched
// twins).  A CONCAT kernel prepares ONE operand of extent bt.n * k, whose b-th k-segment is problem b's operand: the operand
// of a sum of products over the batch.  A kernel whose rows run along mn (K-major) writes row r as the problems' rows r laid
// end to end, [R][bt.n * Cc]; one whose rows run along k (MN-major) writes the problems' rows stacked as BATCHED does,
// [bt.n * R][Cc], with ONE scale word per column for all of them.
// Elements c .. c+3 of row r of the rows laid end to end (0 past bt.n * Cc), op applied: one vector load where the four lie
// in one problem at a 16-byte boundary (the host passes 16-byte aligned rows, aux rows and problem offsets), element by
// element across a boundary.  int32 positions: the tensor-core path bounds bt.n * Cc by 2^31.
template <bool HAS_OP>
__device__ __forceinline__ float4 concat_vec(const float *src, int64_t src_ld, const OperandOp &op, const Batch &bt, int64_t r,
                                             int64_t c, int64_t Cc) {
  const int seg = static_cast<int>(Cc);
  int b = static_cast<int>(c) / seg;
  int k = static_cast<int>(c) - b * seg;
  if ((k & 3) == 0 && k + 4 <= seg) {
    float4 v = *reinterpret_cast<const float4 *>(src + b * bt.bs + r * src_ld + k);
    if constexpr (HAS_OP) {
      float4 y = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      if (op.aux) y = *reinterpret_cast<const float4 *>(op.aux + b * bt.aux_bs + r * op.aux_sr + k);
      v.x = operand_op(op.op, v.x, y.x); v.y = operand_op(op.op, v.y, y.y);
      v.z = operand_op(op.op, v.z, y.z); v.w = operand_op(op.op, v.w, y.w);
    }
    return v;
  }
  float e[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    while (k >= seg) { k -= seg; ++b; }   // (segments shorter than 4 floats: more than one boundary)
    float x = 0.0f;
    if (b < bt.n) {
      x = src[b * bt.bs + r * src_ld + k];
      if constexpr (HAS_OP) x = operand_op(op.op, x, op.aux ? op.aux[b * bt.aux_bs + r * op.aux_sr + k] : 0.0f);
    }
    e[i] = x;
    ++k;
  }
  return make_float4(e[0], e[1], e[2], e[3]);
}

// src: R rows of Cc contiguous floats, leading dimension src_ld (16-byte aligned rows).
// hi/lo: compact, leading dimension dst_ld (multiple of 4).
template <bool HAS_OP = false, bool BATCHED = false, bool CONCAT = false>
__global__ void __launch_bounds__(256)
split_rows_tf32_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld,
                       float *__restrict__ hi, float *__restrict__ lo, int64_t dst_ld, OperandOp op = OperandOp(),
                       Batch bt = Batch()) {
  static_assert(!CONCAT || BATCHED, "a concatenation is of a batch");
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int64_t vec_per_row = ((CONCAT ? bt.n * Cc : Cc) + 3) >> 2;
  const int64_t total = (BATCHED && !CONCAT ? bt.n * R : R) * vec_per_row;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / vec_per_row;
    const int64_t c = (i - r * vec_per_row) << 2;
    float4 v;
    if constexpr (CONCAT) {
      v = concat_vec<HAS_OP>(src, src_ld, op, bt, r, c, Cc);
    } else {
      const float *sp = src;
      OperandOp o = op;
      const int64_t rl = batch_row<BATCHED>(r, R, bt, sp, o);
      const float *s = sp + rl * src_ld + c;
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
    }
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
template <bool PER_COL, bool HAS_OP = false, bool BATCHED = false, bool CONCAT = false>
__global__ void __launch_bounds__(256)
absmax_mn_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld, uint32_t *__restrict__ out,
                 OperandOp op = OperandOp(), Batch bt = Batch()) {
  static_assert(PER_COL || !HAS_OP, "a K-major operand with an op takes the fused row kernel");
  static_assert(PER_COL || !BATCHED, "a K-major operand takes the fused row kernel");
  static_assert(!CONCAT || BATCHED, "a concatenation is of a batch");
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
        if constexpr (!CONCAT) out_b += b * Cc;   // (CONCAT: one word per column over every problem)
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
template <int GROUP, bool HAS_OP = false, bool BATCHED = false, bool CONCAT = false>
__global__ void __launch_bounds__(256, 4)
f16x2_rows_fused_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *__restrict__ hb,
                        uint16_t *__restrict__ lb, int64_t ld_b, uint32_t *__restrict__ absmax, OperandOp op = OperandOp(),
                        Batch bt = Batch()) {
  static_assert(GROUP == 32 || GROUP == 256, "a warp or the CTA per row");
  static_assert(!CONCAT || BATCHED, "a concatenation is of a batch");
  __shared__ uint32_t red[2][8];
  ptx::griddep_launch_dependents();
  const int tid = static_cast<int>(threadIdx.x) % GROUP;
  const int64_t per_cta = 256 / GROUP;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * per_cta + static_cast<int64_t>(threadIdx.x) / GROUP;
  const int64_t step = static_cast<int64_t>(gridDim.x) * per_cta;
  const int64_t nvec = ((CONCAT ? bt.n * Cc : Cc) + 3) >> 2;
  int parity = 0;
  // GROUP == 256: every thread of the CTA runs the same number of iterations (the loop holds a __syncthreads)
  const int64_t rows = BATCHED && !CONCAT ? bt.n * R : R;
  for (int64_t r = first; r < rows; r += step) {
    const float *sp = src;
    OperandOp o = op;
    const int64_t rl = batch_row<BATCHED && !CONCAT>(r, R, bt, sp, o);
    const float *row = sp + rl * src_ld;
    float4 v[F16ROWS_MAXV];
    uint32_t m = 0u;
#pragma unroll
    for (int i = 0; i < F16ROWS_MAXV; ++i) {
      const int64_t idx = tid + static_cast<int64_t>(i) * GROUP;
      if (idx < nvec) {
        if constexpr (CONCAT) {
          v[i] = concat_vec<HAS_OP>(src, src_ld, op, bt, r, idx << 2, Cc);
        } else {
          v[i] = load_row_vec(row, idx << 2, Cc);
          if constexpr (HAS_OP) v[i] = op_vec(o, v[i], rl, idx << 2, Cc);
        }
        m = max(max(m, finite_abs_bits(v[i].x)), max(finite_abs_bits(v[i].y), max(finite_abs_bits(v[i].z), finite_abs_bits(v[i].w))));
      }
    }
    for (int64_t idx = tid + static_cast<int64_t>(F16ROWS_MAXV) * GROUP; idx < nvec; idx += GROUP) {
      float4 t;
      if constexpr (CONCAT) {
        t = concat_vec<HAS_OP>(src, src_ld, op, bt, r, idx << 2, Cc);
      } else {
        t = load_row_vec(row, idx << 2, Cc);
        if constexpr (HAS_OP) t = op_vec(o, t, rl, idx << 2, Cc);
      }
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
      if constexpr (CONCAT) store_f16x2_vec(concat_vec<HAS_OP>(src, src_ld, op, bt, r, idx << 2, Cc), s, hrow, lrow, idx << 2);
      else if constexpr (HAS_OP) store_f16x2_vec(op_vec(o, load_row_vec(row, idx << 2, Cc), rl, idx << 2, Cc), s, hrow, lrow, idx << 2);
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
template <bool PER_COL, bool HAS_OP = false, bool BATCHED = false, bool CONCAT = false>
__global__ void __launch_bounds__(256)
split_rows_f16x2_kernel(const float *__restrict__ src, int64_t R, int64_t Cc, int64_t src_ld,
                        uint16_t *__restrict__ hb, uint16_t *__restrict__ lb, int64_t ld_b,
                        const uint32_t *__restrict__ absmax, OperandOp op = OperandOp(), Batch bt = Batch()) {
  static_assert(PER_COL || !BATCHED, "a K-major operand takes the fused row kernel");
  static_assert(!CONCAT || BATCHED, "a concatenation is of a batch");
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
      if constexpr (!CONCAT) absmax_b += b * Cc;
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

// ---- im2col source: a convolution's B operand prepared straight from the NCHW images ---------------------------------
// Row n * outHW + p -- image n of the launch, output pixel p = oh * outW + ow -- is the pixel's receptive field in the
// reference's im2col order k = (c * kH + krow) * kW + kcol (conv2d_im2col.nim:69-93), 0 where the window leaves the padded
// image: the im2col matrix transposed, K-major, stacked [images][outHW][ld] like a gathered batched operand.  Each row is
// written in the format of the preparation step it replaces, bit for bit:
//   IM2COL_F32   the values, ld = round_up(K, 4)                                (TF32X1, exact path)
//   IM2COL_TF32  hi / lo pieces as split_rows_tf32_kernel, ld = round_up(K, 4)  (TF32X3)
//   IM2COL_F16X2 abs-max word + both fp16 pieces as f16x2_rows_fused_kernel, ld = round_up(K, 8)  (F16X3): one pass, the row
//                held in registers (F16ROWS_MAXV float4 per thread) while its abs-max is reduced
// Every column up to ld is written (zeros past K).  The window is read with plain cached loads: the 256 / GROUP rows of a
// CTA are neighbouring pixels, whose windows overlap, and the image is small enough to stay in L2 between CTAs.
// GROUP: a warp per row (ld <= 1024), the CTA per row otherwise (the part of the row past the registers is read twice).
enum Im2colMode { IM2COL_F32 = 0, IM2COL_TF32 = 1, IM2COL_F16X2 = 2 };
struct Im2colSrc {   // int32 geometry of one launch (conv_geom bounds K, outHW and H * W by 2^31)
  int C, H, W, kH, kW, pH, pW, sH, sW, outW, K;
  int64_t outHW, image;   // pixels per image, floats per input image
};
inline Im2colSrc im2col_src(const ConvGeom &g) {
  return Im2colSrc{static_cast<int>(g.C), static_cast<int>(g.H), static_cast<int>(g.W), static_cast<int>(g.kH),
                   static_cast<int>(g.kW), static_cast<int>(g.pH), static_cast<int>(g.pW), static_cast<int>(g.sH),
                   static_cast<int>(g.sW), static_cast<int>(g.outW), static_cast<int>(g.K()), g.outHW(), g.C * g.H * g.W};
}
// elements k .. k+3 of the window of output pixel (oh, ow) of image `img` (0 past K)
__device__ __forceinline__ float4 window_vec(const float *__restrict__ img, const Im2colSrc &q, int oh, int ow, int k) {
  const int khw = q.kH * q.kW;
  int c = k / khw;
  int kr = (k - c * khw) / q.kW;
  int kc = k - c * khw - kr * q.kW;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int h = oh * q.sH - q.pH + kr, w = ow * q.sW - q.pW + kc;
    const bool inside = k + e < q.K && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) &&
                        static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
    v[e] = inside ? img[(static_cast<int64_t>(c) * q.H + h) * q.W + w] : 0.0f;
    if (++kc == q.kW) { kc = 0; if (++kr == q.kH) { kr = 0; ++c; } }
  }
  return make_float4(v[0], v[1], v[2], v[3]);
}

// ---- transposed source: a convolution's input gradient, B prepared straight from the output gradients --------------
// The input gradient dX_n = W' * B_n is the forward product over another source (W': the filters rotated by 180 degrees, the
// channel axes swapped).  Row ih * W + iw of B_n is input pixel (ih, iw)'s window over the output gradient dY_n, zero-dilated
// by the forward strides, padded by kH - 1 - pH (which may be negative) and windowed at stride 1, in the forward im2col
// order (co, kh', kw'): the forward windows with Im2colSrc's geometry over dY (C = c_out, H x W = outH x outW, pH = kH - 1 -
// pH, sH = sW = 1, outW = the input's W, outHW = its H * W), read where the dilated position is a source value:
//   h = ih - p' + kh' in the dilated plane; a source row when h >= 0, h % dH == 0 and h / dH < outH (columns likewise)
// Everything else is a structural zero -- also the input rows and columns no window covers, (H + 2pH - kH) mod sH of them.
// HAS_OP applies the operand op to the values read (aux at the same NCHW offset as the dY element); holes stay 0, never op(0).
// A parameter struct of its own, so that Im2colSrc -- and every forward instantiation -- keeps its layout.
struct Im2colGradSrc : Im2colSrc {
  int dH, dW;     // source dilation: the forward strides (1: none)
  OperandOp op;   // HAS_OP: the op on the source values
};
// ---- channels-last source: A of the NHWC forward convolution, prepared straight from the NHWC images ----------------
// Row n * outHW + p -- image n of the launch, output pixel p = oh * outW + ow -- is the pixel's window in the filter matrix's
// row order k = (kh * kW + kw) * C + ci: kH * kW runs of C contiguous floats,
//   row[k] = in[((n * H + h) * W + w) * C + ci],  h = oh * sH - pH + kh,  w = ow * sW - pW + kw   (0 outside the image)
// -- the im2col matrix of every image of the launch, one row per output pixel, K-major: the A operand of ONE product with the
// [K][c_out] filter matrix, whose C is the NHWC output.  vec (C % 4 == 0 and a 16-byte aligned input): every float4 of a row
// lies inside one tap, so it is one 16-byte load (or zeros) with the tap decoded once; otherwise element by element with
// running (ci, kw, kh) counters.  A parameter struct of its own, so that Im2colSrc keeps its layout.
struct Im2colNhwcSrc : Im2colSrc {
  int vec;
};
inline Im2colNhwcSrc im2col_nhwc_src(const ConvGeom &g, const float *in) {
  Im2colNhwcSrc q{};
  static_cast<Im2colSrc &>(q) = im2col_src(g);
  q.vec = g.C % 4 == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0;
  return q;
}
// elements k .. k+3 of the channels-last window of output pixel (oh, ow) of image `img` (0 past K)
__device__ __forceinline__ float4 nhwc_window_vec(const float *__restrict__ img, const Im2colNhwcSrc &q, int oh, int ow, int k) {
  const int tap = k / q.C;
  int ci = k - tap * q.C;
  int kr = tap / q.kW, kc = tap - kr * q.kW;
  if (q.vec) {   // k % 4 == 0 and C % 4 == 0: k .. k+3 are channels ci .. ci+3 of one tap
    const int h = oh * q.sH - q.pH + kr, w = ow * q.sW - q.pW + kc;
    if (k < q.K && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) && static_cast<unsigned>(w) < static_cast<unsigned>(q.W))
      return *reinterpret_cast<const float4 *>(img + (static_cast<int64_t>(h) * q.W + w) * q.C + ci);
    return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int h = oh * q.sH - q.pH + kr, w = ow * q.sW - q.pW + kc;
    const bool inside = k + e < q.K && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) &&
                        static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
    v[e] = inside ? img[(static_cast<int64_t>(h) * q.W + w) * q.C + ci] : 0.0f;
    if (++ci == q.C) { ci = 0; if (++kc == q.kW) { kc = 0; ++kr; } }
  }
  return make_float4(v[0], v[1], v[2], v[3]);
}

// ---- channels-last transposed source: A of the NHWC input gradient, prepared straight from the NHWC output gradients ------
// Row n * outHW + p -- input pixel p = ih * W + iw of image n -- is the pixel's window over dY zero-dilated by the forward
// strides, in the order k' = (kh' * kW + kw') * c_out + co: the transposed geometry of Im2colGradSrc (C = c_out, H x W = outH x
// outW, pH = kH - 1 - pH, stride 1, outW = the input's W), laid out like Im2colNhwcSrc's windows,
//   row[k'] = op(dY)[n][h / dH][w / dW][co],  h = ih - pH' + kh', w = iw - pW' + kw'  when both are source positions, else 0
// (holes are 0, never op(0); the aux at the same NHWC offset as the dY element).  vec (c_out % 4 == 0, dY and the aux 16-byte
// aligned): every float4 of a row lies inside one tap, so the hole test and the h / dH decode run once per float4 and a
// source value is one 16-byte load (and one of the aux).  A parameter struct of its own, so that Im2colNhwcSrc keeps its
// layout.
struct Im2colNhwcGradSrc : Im2colNhwcSrc {
  int dH, dW;     // source dilation: the forward strides (1: none)
  OperandOp op;   // HAS_OP: the op on the source values
};
// (h, w) of the dilated plane -> the source pixel, and whether there is one
template <bool DIL>
__device__ __forceinline__ bool dilated_source(const Im2colNhwcGradSrc &q, int &h, int &w) {
  if constexpr (DIL) {   // h >= 0 is tested, and the quotient used, before any remainder of a negative h could matter
    const unsigned hq = static_cast<unsigned>(h) / static_cast<unsigned>(q.dH), wq = static_cast<unsigned>(w) / static_cast<unsigned>(q.dW);
    const bool inside = h >= 0 && w >= 0 && hq * q.dH == static_cast<unsigned>(h) && wq * q.dW == static_cast<unsigned>(w) &&
                        hq < static_cast<unsigned>(q.H) && wq < static_cast<unsigned>(q.W);
    h = static_cast<int>(hq);
    w = static_cast<int>(wq);
    return inside;
  } else {
    return static_cast<unsigned>(h) < static_cast<unsigned>(q.H) && static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
  }
}
// elements k .. k+3 of the channels-last transposed window of input pixel (oh, ow) of image `img` (aux: its aux image, HAS_OP)
template <bool DIL, bool HAS_OP>
__device__ __forceinline__ float4 nhwc_grad_window_vec(const float *__restrict__ img, const float *__restrict__ aux,
                                                       const Im2colNhwcGradSrc &q, int oh, int ow, int k) {
  const int tap = k / q.C;
  int co = k - tap * q.C;
  int kr = tap / q.kW, kc = tap - kr * q.kW;
  if (q.vec) {   // k % 4 == 0 and c_out % 4 == 0: k .. k+3 are channels co .. co+3 of one tap
    int h = oh - q.pH + kr, w = ow - q.pW + kc;
    if (k < q.K && dilated_source<DIL>(q, h, w)) {
      const int64_t off = (static_cast<int64_t>(h) * q.W + w) * q.C + co;
      float4 v = *reinterpret_cast<const float4 *>(img + off);
      if constexpr (HAS_OP) {
        const float4 y = aux ? *reinterpret_cast<const float4 *>(aux + off) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        v = make_float4(operand_op(q.op.op, v.x, y.x), operand_op(q.op.op, v.y, y.y), operand_op(q.op.op, v.z, y.z),
                        operand_op(q.op.op, v.w, y.w));
      }
      return v;
    }
    return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    int h = oh - q.pH + kr, w = ow - q.pW + kc;
    float x = 0.0f;
    if (k + e < q.K && dilated_source<DIL>(q, h, w)) {
      const int64_t off = (static_cast<int64_t>(h) * q.W + w) * q.C + co;
      x = img[off];
      if constexpr (HAS_OP) x = operand_op(q.op.op, x, aux ? aux[off] : 0.0f);
    }
    v[e] = x;
    if (++co == q.C) { co = 0; if (++kc == q.kW) { kc = 0; ++kr; } }
  }
  return make_float4(v[0], v[1], v[2], v[3]);
}

template <bool GRAD, bool NHWC = false>
using Im2colSrcOf = typename std::conditional<
    NHWC, typename std::conditional<GRAD, Im2colNhwcGradSrc, Im2colNhwcSrc>::type,
    typename std::conditional<GRAD, Im2colGradSrc, Im2colSrc>::type>::type;
// elements k .. k+3 of the transposed window of pixel (oh, ow) of image `img` (aux: its aux image, HAS_OP)
template <bool DIL, bool HAS_OP>
__device__ __forceinline__ float4 grad_window_vec(const float *__restrict__ img, const float *__restrict__ aux, const Im2colGradSrc &q,
                                                  int oh, int ow, int k) {
  const int khw = q.kH * q.kW;
  int c = k / khw;
  int kr = (k - c * khw) / q.kW;
  int kc = k - c * khw - kr * q.kW;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    int h = oh * q.sH - q.pH + kr, w = ow * q.sW - q.pW + kc;
    bool inside = k + e < q.K;
    if constexpr (DIL) {   // h >= 0 is tested, and the quotient used, before any remainder of a negative h could matter
      const unsigned hq = static_cast<unsigned>(h) / static_cast<unsigned>(q.dH), wq = static_cast<unsigned>(w) / static_cast<unsigned>(q.dW);
      inside = inside && h >= 0 && w >= 0 && hq * q.dH == static_cast<unsigned>(h) && wq * q.dW == static_cast<unsigned>(w) &&
               hq < static_cast<unsigned>(q.H) && wq < static_cast<unsigned>(q.W);
      h = static_cast<int>(hq);
      w = static_cast<int>(wq);
    } else {
      inside = inside && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) && static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
    }
    float x = 0.0f;
    if (inside) {
      const int64_t off = (static_cast<int64_t>(c) * q.H + h) * q.W + w;
      x = img[off];
      if constexpr (HAS_OP) x = operand_op(q.op.op, x, aux ? aux[off] : 0.0f);
    }
    v[e] = x;
    if (++kc == q.kW) { kc = 0; if (++kr == q.kH) { kr = 0; ++c; } }
  }
  return make_float4(v[0], v[1], v[2], v[3]);
}
template <bool DIL, bool HAS_OP, bool NHWC, typename Src>
__device__ __forceinline__ float4 source_vec(const float *__restrict__ img, const float *__restrict__ aux, const Src &q, int oh, int ow,
                                             int k) {
  if constexpr (NHWC && (DIL || HAS_OP)) return nhwc_grad_window_vec<DIL, HAS_OP>(img, aux, q, oh, ow, k);
  else if constexpr (NHWC) return nhwc_window_vec(img, q, oh, ow, k);
  else if constexpr (DIL || HAS_OP) return grad_window_vec<DIL, HAS_OP>(img, aux, q, oh, ow, k);
  else return window_vec(img, q, oh, ow, k);
}

// (F16X2: the row in registers next to the geometry needs more than the 64 registers of 4 CTAs per SM -- it spills there)
// DIL / HAS_OP (an Im2colGradSrc): the transposed source of the input gradient, dilated / with an op; NHWC (an Im2colNhwcSrc):
// the channels-last source of the NHWC forward call, with DIL / HAS_OP (an Im2colNhwcGradSrc) the channels-last transposed
// source of the NHWC input gradient; the NCHW forward call's instantiations are <MODE, GROUP, false, false>.
template <int MODE, int GROUP, bool DIL = false, bool HAS_OP = false, bool NHWC = false>
__global__ void __launch_bounds__(256, MODE == IM2COL_F16X2 ? 3 : 4)
im2col_rows_kernel(const float *__restrict__ in, Im2colSrcOf<DIL || HAS_OP, NHWC> q, int64_t images, float *__restrict__ dst,
                   float *__restrict__ dst_lo, uint16_t *__restrict__ hb, uint16_t *__restrict__ lb, int64_t ld,
                   uint32_t *__restrict__ absmax) {
  static_assert(GROUP == 32 || GROUP == 256, "a warp or the CTA per row");
  __shared__ uint32_t red[2][8];
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int tid = static_cast<int>(threadIdx.x) % GROUP;
  const int64_t per_cta = 256 / GROUP;
  const int64_t first = static_cast<int64_t>(blockIdx.x) * per_cta + static_cast<int64_t>(threadIdx.x) / GROUP;
  const int64_t step = static_cast<int64_t>(gridDim.x) * per_cta;
  const int nvec = static_cast<int>(ld >> 2);   // float4 groups written per row, padding included
  int parity = 0;
  // GROUP == 256: every thread of the CTA runs the same number of iterations (the loop holds a __syncthreads)
  for (int64_t r = first; r < images * q.outHW; r += step) {
    const int64_t n = r / q.outHW;
    const int p = static_cast<int>(r - n * q.outHW);
    const int oh = p / q.outW, ow = p - oh * q.outW;
    const float *img = in + n * q.image;
    const float *aux = nullptr;
    if constexpr (HAS_OP) aux = q.op.aux ? q.op.aux + n * q.image : nullptr;
    if constexpr (MODE != IM2COL_F16X2) {
      for (int idx = tid; idx < nvec; idx += GROUP) {
        const float4 v = source_vec<DIL, HAS_OP, NHWC>(img, aux, q, oh, ow, idx << 2);
        if constexpr (MODE == IM2COL_F32) {
          *reinterpret_cast<float4 *>(dst + r * ld + (idx << 2)) = v;
        } else {
          float4 h, l;
          h.x = tf32_rna(v.x); l.x = tf32_lo(v.x, h.x);
          h.y = tf32_rna(v.y); l.y = tf32_lo(v.y, h.y);
          h.z = tf32_rna(v.z); l.z = tf32_lo(v.z, h.z);
          h.w = tf32_rna(v.w); l.w = tf32_lo(v.w, h.w);
          *reinterpret_cast<float4 *>(dst + r * ld + (idx << 2)) = h;
          *reinterpret_cast<float4 *>(dst_lo + r * ld + (idx << 2)) = l;
        }
      }
    } else {
      float4 v[F16ROWS_MAXV];
      uint32_t m = 0u;
#pragma unroll
      for (int i = 0; i < F16ROWS_MAXV; ++i) {
        const int idx = tid + i * GROUP;
        if (idx < nvec) {
          v[i] = source_vec<DIL, HAS_OP, NHWC>(img, aux, q, oh, ow, idx << 2);
          m = max(max(m, finite_abs_bits(v[i].x)), max(finite_abs_bits(v[i].y), max(finite_abs_bits(v[i].z), finite_abs_bits(v[i].w))));
        }
      }
      for (int idx = tid + F16ROWS_MAXV * GROUP; idx < nvec; idx += GROUP) {
        const float4 t = source_vec<DIL, HAS_OP, NHWC>(img, aux, q, oh, ow, idx << 2);
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
      uint16_t *hrow = hb + r * ld, *lrow = lb + r * ld;
#pragma unroll
      for (int i = 0; i < F16ROWS_MAXV; ++i) {
        const int idx = tid + i * GROUP;
        if (idx < nvec) store_f16x2_vec(v[i], s, hrow, lrow, static_cast<int64_t>(idx) << 2);
      }
      for (int idx = tid + F16ROWS_MAXV * GROUP; idx < nvec; idx += GROUP)
        store_f16x2_vec(source_vec<DIL, HAS_OP, NHWC>(img, aux, q, oh, ow, idx << 2), s, hrow, lrow, static_cast<int64_t>(idx) << 2);
    }
  }
}

// ---- concatenated im2col source: a convolution's filter-gradient B prepared straight from the NCHW images -------------
// Tap row t = (c * kH + krow) * kW + kcol holds the tap's shifted input plane of every image of the launch, end to end:
//   row[t][n * P + oh * outW + ow] = in[n][c][oh * sH - pH + krow][ow * sW - pW + kcol]   (0 outside the image), P = outHW
// -- the images' im2col matrices [K][P] laid side by side, which is what the batch-reduce entry prepares from materialised
// matrices read transposed (a K-major operand concatenated along k).  Each row is written in the format of the row kernel it
// replaces over that concatenation, bit for bit (im2col_rows_kernel's modes):
//   IM2COL_F32   the values, ld = round_up(n * P, 4)
//   IM2COL_TF32  hi / lo as split_rows_tf32_kernel, ld = round_up(n * P, 4)
//   IM2COL_F16X2 both fp16 pieces as f16x2_rows_fused_kernel against the row's abs-max word, ld = round_up(n * P, 8); the word
//                comes from an ABSMAX launch of the same tiles first (words zeroed by the host, combined with atomicMax)
// Every column up to ld is written (zeros past n * P).  The rows are few and very long (576 x 100352 floats for 32 images of
// a 56 x 56, 64-channel layer), so a work item is a tile of TAP_SEG columns of one row: the tap is decoded once per tile, the
// pixel once per float4, and adjacent threads take adjacent float4, so a warp reads consecutive ow -- consecutive addresses
// when sW = 1.  Both passes read the images, which are small enough to stay in L2 between them.
constexpr int TAP_VEC = 4;                     // float4 per thread of a tile
constexpr int TAP_SEG = 256 * 4 * TAP_VEC;     // columns of one tile
template <int MODE, bool ABSMAX = false>
__global__ void __launch_bounds__(256)
im2col_tap_rows_kernel(const float *__restrict__ in, Im2colSrc q, int64_t images, float *__restrict__ dst, float *__restrict__ dst_lo,
                       uint16_t *__restrict__ hb, uint16_t *__restrict__ lb, int64_t ld, uint32_t *__restrict__ absmax) {
  static_assert(!ABSMAX || MODE == IM2COL_F16X2, "only the f16x2 rows carry a scale word");
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int64_t segs = (ld + TAP_SEG - 1) / TAP_SEG;
  const int khw = q.kH * q.kW, HW = q.H * q.W;
  const uint32_t P = static_cast<uint32_t>(q.outHW);
  const int outH = static_cast<int>(q.outHW / q.outW);
  for (int64_t it = blockIdx.x; it < q.K * segs; it += gridDim.x) {
    const int t = static_cast<int>(it / segs);
    const int64_t j0 = (it - t * segs) * TAP_SEG;
    const int c = t / khw, kr = (t - c * khw) / q.kW, kc = t - c * khw - kr * q.kW;
    const int64_t n0 = j0 / P;
    const uint32_t p0 = static_cast<uint32_t>(j0 - n0 * P);                 // (p0 + d < 2^32: conv_geom bounds P by 2^31)
    const float *plane0 = in + n0 * q.image + static_cast<int64_t>(c) * HW;   // channel c of image n0
    float s = 1.0f;
    if constexpr (MODE == IM2COL_F16X2 && !ABSMAX) s = f16x2_scale(absmax[t]);
    uint32_t m = 0u;
#pragma unroll
    for (int i = 0; i < TAP_VEC; ++i) {
      const uint32_t d = (static_cast<uint32_t>(threadIdx.x) + 256u * i) * 4u;   // this float4's column in the tile
      if (j0 + d < ld) {
        const uint32_t dn = (p0 + d) / P, p = p0 + d - dn * P;
        int oh = static_cast<int>(p) / q.outW, ow = static_cast<int>(p) - oh * q.outW;
        int64_t n = n0 + dn;
        const float *plane = plane0 + dn * q.image;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h = oh * q.sH - q.pH + kr, w = ow * q.sW - q.pW + kc;
          const bool inside = n < images && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) &&
                              static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
          v[e] = inside ? plane[h * q.W + w] : 0.0f;
          if (++ow == q.outW) { ow = 0; if (++oh == outH) { oh = 0; ++n; plane += q.image; } }
        }
        const float4 x = make_float4(v[0], v[1], v[2], v[3]);
        const int64_t j = j0 + d;
        if constexpr (ABSMAX) {
          m = max(max(m, finite_abs_bits(x.x)), max(finite_abs_bits(x.y), max(finite_abs_bits(x.z), finite_abs_bits(x.w))));
        } else if constexpr (MODE == IM2COL_F32) {
          *reinterpret_cast<float4 *>(dst + t * ld + j) = x;
        } else if constexpr (MODE == IM2COL_TF32) {
          float4 h, l;
          h.x = tf32_rna(x.x); l.x = tf32_lo(x.x, h.x);
          h.y = tf32_rna(x.y); l.y = tf32_lo(x.y, h.y);
          h.z = tf32_rna(x.z); l.z = tf32_lo(x.z, h.z);
          h.w = tf32_rna(x.w); l.w = tf32_lo(x.w, h.w);
          *reinterpret_cast<float4 *>(dst + t * ld + j) = h;
          *reinterpret_cast<float4 *>(dst_lo + t * ld + j) = l;
        } else {
          store_f16x2_vec(x, s, hb + t * ld, lb + t * ld, j);
        }
      }
    }
    if constexpr (ABSMAX) {
      float mf = __uint_as_float(m);     // non-negative finite: fmaxf orders them like the integers
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o));
      if ((threadIdx.x & 31) == 0) atomicMax(absmax + t, __float_as_uint(mf));
    }
  }
}

// ---- channels-last tap rows: the filter-gradient B of an NHWC convolution, prepared straight from the NHWC images -------
// Tap row k = (kh * kW + kw) * C + ci -- the filter matrix's row order -- holds the tap's value at every output pixel of every
// image of the launch, end to end along the NHWC gradients' row index j = n * P + p (P = outHW, p = oh * outW + ow):
//   row[k][j] = in[((n * H + h) * W + w) * C + ci],  h = oh * sH - pH + kh,  w = ow * sW - pW + kw   (0 outside the image)
// -- the NHWC forward's window rows transposed: the K-major B of ONE product dWmat^T = op(dY)^T * rows.  Consecutive columns of
// a row lie sW * C floats apart in the images, so a work item is a tile of NHWC_TAPS consecutive taps x NHWC_PIX consecutive
// columns, transposed through shared memory: the reads go along the channels (vec: one 16-byte load per 4 taps of one pixel,
// a warp reading 4 pixels x 32 taps; otherwise element by element), the writes along the pixels, a warp per tap row segment.
// The pixels (n, oh, ow) are decoded once per column and the taps (kh, kw, ci) once per tap, per tile.  The modes write what
// im2col_tap_rows_kernel's write over the same rows, bit for bit (F16X2: the words come from an ABSMAX launch of the same tiles
// first, zeroed by the host, one atomicMax per tap per tile).  Every column up to ld is written (zeros past n * P).
// Shared tile [tap][column]: the float4 slot of columns 4s .. 4s+3 of tap t sits at slot s ^ (t / 4), so that the staging
// stores (4 columns x 8 tap quads per warp) and the row reads (one float4 per lane) are both free of bank conflicts.
// NHWC_PER_SM CTAs per SM: the launch bounds the registers to what that many CTAs leave, and the host sizes the grid to it;
// six is also what the 37 KB of shared memory of a 256-column tile allows.  NHWC_PIX = 256 was the fastest of 64, 128 and 256
// on an H100 (DESIGN.md section 4); a wider tile no longer fits the 48 KB of static shared memory.
constexpr int NHWC_TAPS = 32;     // taps of one tile
constexpr int NHWC_PIX = 256;     // columns of one tile
constexpr int NHWC_PER_SM = 6;    // resident CTAs per SM
template <int MODE, bool ABSMAX = false>
__global__ void __launch_bounds__(256, NHWC_PER_SM)
im2col_nhwc_tap_rows_kernel(const float *__restrict__ in, Im2colNhwcSrc q, int64_t images, float *__restrict__ dst,
                            float *__restrict__ dst_lo, uint16_t *__restrict__ hb, uint16_t *__restrict__ lb, int64_t ld,
                            uint32_t *__restrict__ absmax) {
  static_assert(!ABSMAX || MODE == IM2COL_F16X2, "only the f16x2 rows carry a scale word");
  static_assert(NHWC_TAPS == 32 && NHWC_PIX % 32 == 0 && NHWC_PIX >= 32 && NHWC_PIX + NHWC_TAPS <= 512,
                "8 tap quads per column, 8 warps x 4 rows, whole float4 slots for the swizzle, two decode items per thread at most");
  __shared__ __align__(16) float tile[NHWC_TAPS * NHWC_PIX];
  __shared__ int64_t col_off[NHWC_PIX];        // the pixel's window corner (n, h0, w0) in floats from `in`
  __shared__ int col_h[NHWC_PIX], col_w[NHWC_PIX];
  __shared__ int tap_off[NHWC_TAPS], tap_h[NHWC_TAPS], tap_w[NHWC_TAPS];
  ptx::griddep_launch_dependents();   // the next kernel of the stream may start its prologue (it waits for our results)
  const int tid = static_cast<int>(threadIdx.x), lane = tid & 31, warp = tid >> 5;
  const int64_t cols = images * q.outHW;
  const int64_t tap_tiles = (q.K + NHWC_TAPS - 1) / NHWC_TAPS, col_tiles = (ld + NHWC_PIX - 1) / NHWC_PIX;
  // the tap tiles of one column block are neighbours in the loop: CTAs running together read the same pixels' windows
  for (int64_t it = blockIdx.x; it < tap_tiles * col_tiles; it += gridDim.x) {
    const int64_t cb = it / tap_tiles;
    const int t0 = static_cast<int>(it - cb * tap_tiles) * NHWC_TAPS;
    const int64_t j0 = cb * NHWC_PIX;
    for (int d = tid; d < NHWC_PIX + NHWC_TAPS; d += 256) {
      if (d < NHWC_PIX) {
        const int64_t j = j0 + d;
        int h0 = -(1 << 30), w0 = 0;   // past the images: no tap is inside
        int64_t off = 0;
        if (j < cols) {
          const int64_t n = j / q.outHW;
          const int p = static_cast<int>(j - n * q.outHW), oh = p / q.outW, ow = p - oh * q.outW;
          h0 = oh * q.sH - q.pH;
          w0 = ow * q.sW - q.pW;
          off = n * q.image + (static_cast<int64_t>(h0) * q.W + w0) * q.C;
        }
        col_h[d] = h0; col_w[d] = w0; col_off[d] = off;
      } else {
        const int t = t0 + d - NHWC_PIX;
        int kr = 0, kc = 0, off = 0;   // (past K: every read is skipped)
        if (t < q.K) {
          const int tap = t / q.C, ci = t - tap * q.C;
          kr = tap / q.kW;
          kc = tap - kr * q.kW;
          off = (kr * q.W + kc) * q.C + ci;
        }
        tap_h[d - NHWC_PIX] = kr; tap_w[d - NHWC_PIX] = kc; tap_off[d - NHWC_PIX] = off;
      }
    }
    __syncthreads();   // (also: every warp has read the previous tile out of `tile`)
#pragma unroll
    for (int i = 0; i < NHWC_TAPS * NHWC_PIX / 4 / 256; ++i) {
      const int item = tid + 256 * i, cl = item >> 3, tq = item & 7;   // column cl, taps 4 tq .. 4 tq + 3 of the tile
      const int h0 = col_h[cl], w0 = col_w[cl];
      const float *px = in + col_off[cl];
      float v[4];
      if (q.vec) {   // C % 4 == 0: the four taps are channels ci .. ci + 3 of one (kh, kw), K % 4 == 0
        const int t = 4 * tq;
        const int h = h0 + tap_h[t], w = w0 + tap_w[t];
        float4 x = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (t0 + t < q.K && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) && static_cast<unsigned>(w) < static_cast<unsigned>(q.W))
          x = *reinterpret_cast<const float4 *>(px + tap_off[t]);
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int t = 4 * tq + e;
          const int h = h0 + tap_h[t], w = w0 + tap_w[t];
          const bool inside = t0 + t < q.K && static_cast<unsigned>(h) < static_cast<unsigned>(q.H) &&
                              static_cast<unsigned>(w) < static_cast<unsigned>(q.W);
          v[e] = inside ? px[tap_off[t]] : 0.0f;
        }
      }
      const int slot = (((cl >> 2) ^ tq) << 2) + (cl & 3);
#pragma unroll
      for (int e = 0; e < 4; ++e) tile[(4 * tq + e) * NHWC_PIX + slot] = v[e];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NHWC_TAPS / 8; ++i) {
      const int r = warp + 8 * i, t = t0 + r;
      if (t >= q.K) break;   // (uniform over the warp)
      uint32_t m = 0u;
      for (int c4 = lane; c4 < NHWC_PIX / 4; c4 += 32) {   // this lane's float4 of the row segment
        const int64_t j = j0 + 4 * c4;
        const float4 x = *reinterpret_cast<const float4 *>(tile + r * NHWC_PIX + ((c4 ^ (r >> 2)) << 2));
        if constexpr (ABSMAX) {   // (columns past ld are zeros)
          m = max(max(m, max(finite_abs_bits(x.x), finite_abs_bits(x.y))), max(finite_abs_bits(x.z), finite_abs_bits(x.w)));
        } else if (j < ld) {
          if constexpr (MODE == IM2COL_F32) {
            *reinterpret_cast<float4 *>(dst + t * ld + j) = x;
          } else if constexpr (MODE == IM2COL_TF32) {
            float4 h, l;
            h.x = tf32_rna(x.x); l.x = tf32_lo(x.x, h.x);
            h.y = tf32_rna(x.y); l.y = tf32_lo(x.y, h.y);
            h.z = tf32_rna(x.z); l.z = tf32_lo(x.z, h.z);
            h.w = tf32_rna(x.w); l.w = tf32_lo(x.w, h.w);
            *reinterpret_cast<float4 *>(dst + t * ld + j) = h;
            *reinterpret_cast<float4 *>(dst_lo + t * ld + j) = l;
          } else {
            store_f16x2_vec(x, f16x2_scale(absmax[t]), hb + t * ld, lb + t * ld, j);
          }
        }
      }
      if constexpr (ABSMAX) {   // every lane takes part, with 0 where it had no column
        float mf = __uint_as_float(m);   // non-negative finite: fmaxf orders them like the integers
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mf = fmaxf(mf, __shfl_xor_sync(0xffffffffu, mf, o));
        if (lane == 0) atomicMax(absmax + t, __float_as_uint(mf));
      }
    }
  }
}

// dst[r*ld + c] = src[r*sr + c*sc] for r < R, c < Cc.  32 x 32 tiles through shared
// memory so that both the gather (along whichever source stride is smaller) and the
// store (along c) are coalesced.  SPLIT: also write lo (fp32 only).
// MODE 0: plain copy; 1: fp32 hi/lo pieces (dst, dst_lo).
// HAS_OP (fp32): the op is applied to each element as it is gathered (aux read with its own strides).
// CONCAT: problem b's [R][Cc] is written to columns b * Cc .. of the rows [R][ld] (ld >= bt.n * Cc).
template <typename T, int MODE, bool HAS_OP = false, bool BATCHED = false, bool CONCAT = false>
__global__ void __launch_bounds__(256)
pack_general_kernel(const T *__restrict__ src, int64_t R, int64_t Cc, int64_t sr, int64_t sc,
                    T *__restrict__ dst, T *__restrict__ dst_lo, int64_t ld, int read_along_r, OperandOp op = OperandOp(),
                    Batch bt = Batch()) {
  static_assert(!HAS_OP || sizeof(T) == 4, "operand ops are fp32 only");
  static_assert(!BATCHED || sizeof(T) == 4, "batched operands are fp32 only");
  static_assert(!CONCAT || BATCHED, "a concatenation is of a batch");
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
      dst_t += CONCAT ? b * Cc : b * R * ld;   // (CONCAT: to columns b * Cc + c)
      if constexpr (MODE == 1) dlo_t += CONCAT ? b * Cc : b * R * ld;
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
// of problem t / (num_m * num_n), whose C starts bsC elements after the previous problem's and whose bias starts
// (problem % period_a) * bias_bs elements into `bias` (tc_params.h).
template <bool BATCHED = false>
__global__ void __launch_bounds__(256)
splitk_tail_reduce_kernel(const float *__restrict__ ws, int S, int n_tail, int n_direct, int num_m, int num_n, int raster_g,
                          int64_t M, int64_t N, float alpha, float beta, float *__restrict__ C, int64_t rsC,
                          int64_t csC, const float *__restrict__ bias, int bias_per_row, int act, int64_t bsC = 0, int period_a = 1,
                          int64_t bias_bs = 0) {
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
    const float *bb = bias;
    if constexpr (BATCHED) {
      const int b = t / (num_m * num_n);
      t -= b * (num_m * num_n);
      Cb += b * bsC;
      if (bb) bb += (b % period_a) * bias_bs;
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
        if (bb != nullptr || act != 0) {
          if (bb) v += bias_per_row ? bb[r] : bb[c + e];
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
