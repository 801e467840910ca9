// layers.cuh -- the HBM-bound steps either side of the GEMM in the reference's intended use
// (SURVEY.md section 8f, rank 4): physical transposition / NCHW<->NHWC
// (laser/primitives/swapaxes.nim:16-112), im2col (benchmarks/convolution/conv2d_im2col.nim:44-93)
// and the strided N-d copy behind copyFrom (laser/tensor/initialization.nim:80-112).
// All of them move each byte once: coalesced 16-byte global accesses where the shapes allow,
// shared-memory tiles for the transposition, grids sized from the SM count by the host.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace lb200 {

// ---- batched 2-d transposition: dst[n][j][i] = src[n][i][j], src = N x [NR][NC] contiguous ----
// 64 x 64 element tiles through shared memory (row pitch 65 elements: the transposed read hits
// 2-way bank conflicts at worst, far from limiting an HBM-bound kernel).  V = elements per
// global access (4 when NR, NC are multiples of 4 and both bases are aligned to 4 elements,
// else 1).  256 threads: 16 accesses of V=4 per tile row, 16 rows per pass.
template <typename T>
struct alignas(sizeof(T) * 4 > 16 ? 16 : sizeof(T) * 4) Vec4 {
  T v[4];
};

// host side: may the 4-element accesses be used?
template <typename T>
inline bool transpose_can_vec(const void *dst, const void *src, int64_t NR, int64_t NC) {
  const uintptr_t align = sizeof(T) * 4 > 16 ? 16 : sizeof(T) * 4;
  return (NR % 4 == 0) && (NC % 4 == 0) && (reinterpret_cast<uintptr_t>(dst) % align == 0) &&
         (reinterpret_cast<uintptr_t>(src) % align == 0);
}
inline int64_t transpose_tiles(int64_t N, int64_t NR, int64_t NC) { return N * ((NR + 63) / 64) * ((NC + 63) / 64); }

template <typename T, int V>
__global__ void __launch_bounds__(256)
transpose_batched_kernel(T *__restrict__ dst, const T *__restrict__ src, int64_t N, int64_t NR, int64_t NC) {
  constexpr int TILE = 64;
  __shared__ T tile[TILE][TILE + 1];
  const int64_t tiles_r = (NR + TILE - 1) / TILE, tiles_c = (NC + TILE - 1) / TILE;
  const int64_t per_mat = tiles_r * tiles_c, total = per_mat * N;
  const int tid = threadIdx.x;
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int64_t n = t / per_mat, rem = t - n * per_mat;
    const int64_t r0 = (rem / tiles_c) * TILE, c0 = (rem % tiles_c) * TILE;
    const T *s = src + n * NR * NC;
    T *d = dst + n * NR * NC;
    if constexpr (V == 4) {
      const int q = tid & 15, rr = tid >> 4;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int r = p * 16 + rr;
        if (r0 + r < NR && c0 + 4 * q < NC) {
          const Vec4<T> v = *reinterpret_cast<const Vec4<T> *>(s + (r0 + r) * NC + c0 + 4 * q);
#pragma unroll
          for (int e = 0; e < 4; ++e) tile[r][4 * q + e] = v.v[e];
        }
      }
      __syncthreads();
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int j = p * 16 + rr;  // row of dst inside the tile = column of src
        if (c0 + j < NC && r0 + 4 * q < NR) {
          Vec4<T> v;
#pragma unroll
          for (int e = 0; e < 4; ++e) v.v[e] = tile[4 * q + e][j];
          *reinterpret_cast<Vec4<T> *>(d + (c0 + j) * NR + r0 + 4 * q) = v;
        }
      }
    } else {
      const int x = tid & 63, y = tid >> 6;  // 64 x 4
#pragma unroll 4
      for (int p = 0; p < 16; ++p) {
        const int r = p * 4 + y;
        if (r0 + r < NR && c0 + x < NC) tile[r][x] = s[(r0 + r) * NC + c0 + x];
      }
      __syncthreads();
#pragma unroll 4
      for (int p = 0; p < 16; ++p) {
        const int j = p * 4 + y;
        if (c0 + j < NC && r0 + x < NR) d[(c0 + j) * NR + r0 + x] = tile[x][j];
      }
    }
    __syncthreads();
  }
}

// ---- convolution geometry (conv2d_common.nim:6-45): NCHW images, [Cout][C][kH][kW] filters ----
struct ConvGeom {
  int64_t B, C, H, W, Cout, kH, kW, pH, pW, sH, sW, outH, outW;
  // dilation of the source (an im2col source only): the transposed geometry of the input gradient reads the output gradient
  // zero-dilated by the forward strides (split.cuh: Im2colGradSrc)
  int64_t dH = 1, dW = 1;
  // channels-last images [B][H][W][C] (an im2col source only): the windows are rows in the (kh, kw, c) order of the NHWC
  // forward call (split.cuh: Im2colNhwcSrc)
  bool nhwc = false;
  // with nhwc: the windows oriented as tap rows (an im2col source only) -- the operand's mn is the tap (kh, kw, c), its k the
  // pixel index n * outH * outW + p: B of the NHWC filter gradient (split.cuh: im2col_nhwc_tap_rows_kernel)
  bool taps = false;
  __host__ __device__ int64_t K() const { return C * kH * kW; }
  __host__ __device__ int64_t outHW() const { return outH * outW; }
};

// ---- im2col: images x [C][H][W] -> images x [C*kH*kW][outH*outW], zero outside the image ----
struct Im2colParams {
  int C, H, W, kH, kW, pH, pW, sH, sW, outH, outW;
  int K;         // C * kH * kW  (rows of the workspace matrix)
  int outHW;     // columns
  int64_t rows;  // K * images
  int64_t in_image_stride, ws_image_stride;  // elements
  int tx_log2;   // threads along the columns = 1 << tx_log2 (each owns 4 consecutive columns)
  int chunks;    // column chunks of (4 * quads_per_thread << tx_log2) per row
  int quads_per_thread;   // consecutive groups of 4 columns one thread writes (row and column decoded once for all of them)
};

// host side: launch geometry.  geom = {C, H, W, kH, kW, pH, pW, sH, sW, outH, outW} (all < 2^31).
// Returns the number of blocks of 256 threads; *vec4 says whether the float4 store variant applies.
inline int64_t im2col_plan(const int64_t geom[11], int64_t images, const void *workspace, Im2colParams *p,
                           bool *vec4) {
  p->C = (int)geom[0]; p->H = (int)geom[1]; p->W = (int)geom[2]; p->kH = (int)geom[3]; p->kW = (int)geom[4];
  p->pH = (int)geom[5]; p->pW = (int)geom[6]; p->sH = (int)geom[7]; p->sW = (int)geom[8];
  p->outH = (int)geom[9]; p->outW = (int)geom[10];
  p->K = p->C * p->kH * p->kW;
  p->outHW = p->outH * p->outW;
  p->rows = static_cast<int64_t>(p->K) * images;
  p->in_image_stride = geom[0] * geom[1] * geom[2];
  p->ws_image_stride = static_cast<int64_t>(p->K) * p->outHW;
  const int quads = (p->outHW + 3) / 4;
  int tx_log2 = 0;
  while ((1 << tx_log2) < quads && tx_log2 < 8) ++tx_log2;
  p->tx_log2 = tx_log2;
  p->quads_per_thread = quads >= 1024 ? 4 : 1;
  const int per_chunk = p->quads_per_thread << tx_log2;
  p->chunks = (quads + per_chunk - 1) / per_chunk;
  const int rows_per_block = 256 >> tx_log2;
  *vec4 = (p->outHW % 4 == 0) && (reinterpret_cast<uintptr_t>(workspace) % 16 == 0);
  return ((p->rows + rows_per_block - 1) / rows_per_block) * p->chunks;
}

// thread (tx, ty): row = block_row_group * rows_per_block + ty, columns 4*((chunk*U + u)*TX + tx) .. +3 for u < U =
// quads_per_thread.  The row is decoded once per thread (kk -> c, krow, kcol), the column once per 4 outputs.
template <bool VEC4>
__global__ void __launch_bounds__(256)
im2col_kernel(float *__restrict__ ws, const float *__restrict__ in, Im2colParams p) {
  const int tx = threadIdx.x & ((1 << p.tx_log2) - 1), ty = threadIdx.x >> p.tx_log2;
  const int rows_per_block = 256 >> p.tx_log2;
  const int64_t blk = blockIdx.x;
  const int chunk = static_cast<int>(blk % p.chunks);
  const int64_t row = (blk / p.chunks) * rows_per_block + ty;
  if (row >= p.rows) return;
  const int64_t img = row / p.K;
  const int kk = static_cast<int>(row - img * p.K);
  const int khw = p.kH * p.kW;
  const int c = kk / khw, r2 = kk - c * khw;
  const int krow = r2 / p.kW, kcol = r2 - krow * p.kW;
  const float *src = in + img * p.in_image_stride + static_cast<int64_t>(c) * p.H * p.W;
  float *wrow = ws + img * p.ws_image_stride + static_cast<int64_t>(kk) * p.outHW;
  // quad u of this thread: lanes stay next to each other in every store instruction (the row was decoded once above)
  for (int u = 0; u < p.quads_per_thread; ++u) {
    const int p0 = (((chunk * p.quads_per_thread + u) << p.tx_log2) + tx) * 4;
    if (p0 >= p.outHW) return;
    int oh = p0 / p.outW, ow = p0 - oh * p.outW;
    float *dst = wrow + p0;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = oh * p.sH - p.pH + krow, cc = ow * p.sW - p.pW + kcol;
      const bool inside = (p0 + e < p.outHW) && static_cast<unsigned>(r) < static_cast<unsigned>(p.H) &&
                          static_cast<unsigned>(cc) < static_cast<unsigned>(p.W);
      v[e] = inside ? src[static_cast<int64_t>(r) * p.W + cc] : 0.0f;
      if (++ow == p.outW) { ow = 0; ++oh; }
    }
    if constexpr (VEC4) {
      *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (p0 + e < p.outHW) dst[e] = v[e];
    }
  }
}

// ---- strided N-d copy (copyFrom): dst[idx] = src[idx] over a common shape, rank <= 6 ----
struct CopyParams {
  int rank;
  int64_t shape[6], dst_strides[6], src_strides[6];  // elements; innermost dimension last
  int64_t total;
};
// host side: merge neighbouring dimensions that are contiguous in both views, drop extents of 1
inline void copy_plan(int rank, const int64_t *shape, const int64_t *dst_strides, const int64_t *src_strides,
                      CopyParams *p) {
  p->rank = 0;
  p->total = 1;
  for (int d = 0; d < rank; ++d) {
    p->total *= shape[d];
    if (shape[d] == 1) continue;
    if (p->rank > 0 && p->dst_strides[p->rank - 1] == dst_strides[d] * shape[d] &&
        p->src_strides[p->rank - 1] == src_strides[d] * shape[d]) {
      p->shape[p->rank - 1] *= shape[d];
      p->dst_strides[p->rank - 1] = dst_strides[d];
      p->src_strides[p->rank - 1] = src_strides[d];
    } else {
      p->shape[p->rank] = shape[d];
      p->dst_strides[p->rank] = dst_strides[d];
      p->src_strides[p->rank] = src_strides[d];
      ++p->rank;
    }
  }
  for (int d = p->rank; d < 6; ++d) { p->shape[d] = 1; p->dst_strides[d] = 0; p->src_strides[d] = 0; }
}

template <typename T>
__global__ void __launch_bounds__(256)
copy_strided_kernel(T *__restrict__ dst, const T *__restrict__ src, CopyParams p) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < p.total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t rem = i, od = 0, os = 0;
#pragma unroll
    for (int d = 5; d >= 0; --d) {
      if (d < p.rank) {
        const int64_t q = rem / p.shape[d], x = rem - q * p.shape[d];
        od += x * p.dst_strides[d];
        os += x * p.src_strides[d];
        rem = q;
      }
    }
    dst[od] = src[os];
  }
}


// ---- forEach over up to four equal-shape strided views (laser/strided_iteration/foreach.nim:229-251) ----
// `forEach o in out, x in a, y in b, z in c: <body>` -- the body cannot cross a C ABI, so the bodies
// the reference's own code, docs and iteration benchmark use are provided as opcodes.
enum ForeachOp : int {
  FE_COPY = 0,    // o = x                      (copyFrom / deepCopy, initialization.nim:68,104)
  FE_FILL = 1,    // o = alpha
  FE_SCALE = 2,   // o = alpha * x
  FE_ADD = 3,     // o = x + y
  FE_SUB = 4,     // o = x - y
  FE_MUL = 5,     // o = x * y
  FE_FMA = 6,     // o = x + y * z               (`x += y * z`, foreach.nim:231-232, with o aliasing x)
  FE_AXPY = 7,    // o = alpha * x + y
  FE_BENCH = 8,   // o = x + y - sin(z)          (benchmarks/loop_iteration/iter_bench_prod.nim:88-90)
  FE_NUM_OPS = 9
};
struct ForeachParams {
  int rank;
  int64_t shape[6];
  int64_t strides[4][6];   // o, x, y, z (elements; 0 for unused operands)
  int64_t total;
};
// host side: merge neighbouring dimensions contiguous in every operand, drop extents of 1
inline void foreach_plan(int rank, const int64_t *shape, const int64_t *const strides[4], ForeachParams *p) {
  p->rank = 0;
  p->total = 1;
  for (int d = 0; d < rank; ++d) {
    p->total *= shape[d];
    if (shape[d] == 1) continue;
    bool merge = p->rank > 0;
    for (int t = 0; t < 4 && merge; ++t)
      merge = p->strides[t][p->rank - 1] == (strides[t] ? strides[t][d] : 0) * shape[d];
    if (merge) {
      p->shape[p->rank - 1] *= shape[d];
      for (int t = 0; t < 4; ++t) p->strides[t][p->rank - 1] = strides[t] ? strides[t][d] : 0;
    } else {
      p->shape[p->rank] = shape[d];
      for (int t = 0; t < 4; ++t) p->strides[t][p->rank] = strides[t] ? strides[t][d] : 0;
      ++p->rank;
    }
  }
  for (int d = p->rank; d < 6; ++d) {
    p->shape[d] = 1;
    for (int t = 0; t < 4; ++t) p->strides[t][d] = 0;
  }
}
template <typename T> __device__ __forceinline__ T fe_sin(T v);
template <> __device__ __forceinline__ float fe_sin<float>(float v) { return sinf(v); }
template <> __device__ __forceinline__ double fe_sin<double>(double v) { return sin(v); }

template <typename T, int OP>
__global__ void __launch_bounds__(256)
foreach_strided_kernel(T *o, const T *x, const T *y, const T *z, ForeachParams p, T alpha) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < p.total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t rem = i, off[4] = {0, 0, 0, 0};
#pragma unroll
    for (int d = 5; d >= 0; --d) {
      if (d < p.rank) {
        const int64_t q = rem / p.shape[d], c = rem - q * p.shape[d];
#pragma unroll
        for (int t = 0; t < 4; ++t) off[t] += c * p.strides[t][d];
        rem = q;
      }
    }
    T v;
    if constexpr (OP == FE_COPY) v = x[off[1]];
    else if constexpr (OP == FE_FILL) v = alpha;
    else if constexpr (OP == FE_SCALE) v = alpha * x[off[1]];
    else if constexpr (OP == FE_ADD) v = x[off[1]] + y[off[2]];
    else if constexpr (OP == FE_SUB) v = x[off[1]] - y[off[2]];
    else if constexpr (OP == FE_MUL) v = x[off[1]] * y[off[2]];
    else if constexpr (OP == FE_FMA) v = x[off[1]] + y[off[2]] * z[off[3]];
    else if constexpr (OP == FE_AXPY) v = alpha * x[off[1]] + y[off[2]];
    else v = x[off[1]] + y[off[2]] - fe_sin<T>(z[off[3]]);
    o[off[0]] = v;
  }
}
// operands an opcode reads (bit 0: x, bit 1: y, bit 2: z)
inline int foreach_operands(int op) {
  switch (op) {
    case FE_COPY: case FE_SCALE: return 1;
    case FE_FILL: return 0;
    case FE_ADD: case FE_SUB: case FE_MUL: case FE_AXPY: return 3;
    case FE_FMA: case FE_BENCH: return 7;
    default: return -1;
  }
}

}  // namespace lb200
