// capi.cu -- host side of liblaser_b200.so: the C ABI declared in include/laser_b200.h.
//
// Mirrors the host half of the reference's gemm_strided (gemm.nim:184-247): build the
// three matrix views, pick a kernel family (the reference picks an ISA micro-kernel at
// run time, gemm.nim:228-247; here: exact SIMT vs wgmma), prepare the operands
// (the reference allocates packing Tiles per call, gemm_tiling.nim:312-341; here: TMA
// tensor maps, plus the two-piece workspace of the fp32-faithful modes) and launch.
// The wgmma kernels live in their own translation units (tc_*.cu, tc_launch.h).
// There is no CPU fallback anywhere in this file.
#include "../../include/laser_b200.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "gemm_simt.cuh"
#include "gemm_dmma.cuh"
#include "layers.cuh"
#include "split.cuh"
#include "tc_launch.h"

namespace {

using namespace lb200;

thread_local std::string g_last_error;
thread_local int g_last_path = 0;
std::atomic<int64_t> g_launches{0};
std::atomic<int64_t> g_dmma_launches{0};   // launches of the fp64 tensor-core kernel (debug counter)
std::atomic<int> g_f32_mode{-1};
constexpr int kDefaultF32Mode = LASER_B200_PATH_F16X3;
void multi_shutdown();   // capi_multi.inc

int set_error(int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      cudaGetLastError();                                                                   \
      return set_error(_e == cudaErrorMemoryAllocation ? LASER_B200_ENOMEM : LASER_B200_ECUDA, \
                       "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,   \
                       __LINE__);                                                           \
    }                                                                                       \
  } while (0)

struct Buffer {
  void *ptr = nullptr;
  size_t bytes = 0;
};

struct EventPair {
  cudaEvent_t a, b;
  int kind;  // 0 = tensor-core GEMM kernel, 1 = operand preparation kernels
  int launches;
};

// cache of encoded tensor maps (cuTensorMapEncodeTiled costs microseconds; the reference's
// analogue is re-using its Tiles object): keyed by everything the encoding depends on
struct MapKey {
  const void *base;
  int64_t inner, outer, stride;
  int esz, box_inner, box_outer, swz;
  int64_t depth, depth_stride;   // rank 3 (batched launches): matrices and their distance in elements; depth 0: rank 2
  bool operator==(const MapKey &o) const {
    return base == o.base && inner == o.inner && outer == o.outer && stride == o.stride && esz == o.esz &&
           box_inner == o.box_inner && box_outer == o.box_outer && swz == o.swz && depth == o.depth &&
           depth_stride == o.depth_stride;
  }
};
struct MapCacheEntry {
  MapKey key;
  CUtensorMap map;
  bool valid = false;
};
constexpr int kMapCacheSize = 64;

constexpr int kSchedSlots = 256;   // tile-scheduler counters: one pair of words per launch in flight, used round-robin

struct Ctx {
  MapCacheEntry map_cache[kMapCacheSize];
  int map_cache_next = 0;
  int raster_g = 0;       // env LASER_B200_RASTER (0 = default)
  bool splitk_enabled = true;  // env LASER_B200_SPLITK=0 disables split-K
  bool f64_dmma = true;        // env LASER_B200_F64_DMMA=0: fp64 problems stay on the CUDA-core kernel
  bool ring_attr_set = false, dmma_attr_set = false;
  int64_t panel_rows = 1024;  // env LASER_B200_PANEL_ROWS: row-panel height of the pipelined host-pointer entry
  bool panel_taper = false;   // env LASER_B200_PANEL_TAPER=1: cut the last row panel finer (shorter PCIe tail)
  // K extent per accumulator block of the fp32-faithful modes (env LASER_B200_KC): the tensor core's own accumulation does
  // not round to nearest, and its bias grows with the chain it accumulates; after each block the sums are added to fp32
  // running sums with round-to-nearest.  Shorter blocks cost a few register additions per k-tile.
  int kc_faithful = 128;
  bool dyn_sched = true;  // env LASER_B200_DYNSCHED=0: static round-robin tiles instead of the atomic counter
  bool pdl = true;        // env LASER_B200_PDL=0: ordinary launch of the GEMM kernel after the preparation kernels
  // env LASER_B200_BATCH_WS_MB: prepared workspace of one batched call at most; a larger batch runs in chunks of whole problems
  int64_t batch_ws_bytes = static_cast<int64_t>(1024) << 20;
  bool profiling = false;
  std::vector<EventPair> prof;
  int dev = -1;
  int sm_count = 0;
  cudaStream_t stream = nullptr;          // compute (and default) stream of the library
  cudaStream_t up = nullptr, down = nullptr;  // H2D / D2H streams of the pipelined host entry
  std::vector<cudaEvent_t> panel_ev;
  PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  Buffer ws[4];      // prepared pieces: A piece 0, A piece 1, B piece 0, B piece 1
  Buffer gather[2];  // F16X3: compact fp32 copy of a general-stride operand (A, B) before it is scaled and split
  Buffer stage[3];   // device staging of host A, B, C spans
  Buffer splitk;     // split-K partial-sum planes
  Buffer bpanels;    // row-sharded products: B prepared, panel-major (capi_multi.inc: rowshard_prepared)
  Buffer layer_ws;   // im2col workspace of the host-pointer convolution
  Buffer tfilt;      // the input gradients' rotated filters, under tfilt_mu for a whole call: W' (conv2d_input_grad_dev), W'^T
                     // (conv2d_nhwc_input_grad_dev) or W'_g of every group (conv2d_grouped_input_grad_dev, tensor-core paths)
  Buffer f16s;       // F16X3 mode: fp32 bits of max_k |a| per row of A (words [0, M)) and of max_k |b| per column of B (from
                     // f16_b_off on), written and read on the device
  Buffer sched;      // kSchedSlots x {next unit, CTAs done}: the kernel re-zeroes its slot when it ends
  int sched_next = 0;
  cudaEvent_t ws_free = nullptr;  // recorded after the last kernel that reads ws[]
  std::mutex mu;       // workspace + tensor-map construction
  std::mutex host_mu;  // staging buffers of the host-pointer entry points
  std::mutex tfilt_mu; // tfilt: written once per call of an input gradient, read by every chunk's product (each takes mu
                       // itself)
  std::atomic<bool> ready{false};
};

constexpr int kMaxDevices = 32;
Ctx g_ctx[kMaxDevices];
std::mutex g_ctx_mu;

int parse_f32_mode(const char *mode) {
  if (!mode) return kDefaultF32Mode;
  if (!strcmp(mode, "f16x3")) return LASER_B200_PATH_F16X3;
  else if (!strcmp(mode, "tf32x3")) return LASER_B200_PATH_TF32X3;
  else if (!strcmp(mode, "tf32x1")) return LASER_B200_PATH_TF32X1;
  else if (!strcmp(mode, "simt")) return LASER_B200_PATH_SIMT;
  return kDefaultF32Mode;
}

int get_ctx(Ctx **out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return set_error(LASER_B200_ENODEVICE, "no CUDA device: %s", cudaGetErrorString(e));
  }
  if (dev < 0 || dev >= kMaxDevices) return set_error(LASER_B200_ENODEVICE, "device index %d", dev);
  Ctx &c = g_ctx[dev];
  if (!c.ready) {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    if (!c.ready) {
      cudaDeviceProp prop;
      CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
      if (prop.major != 9 || prop.minor != 0)
        return set_error(LASER_B200_ENODEVICE,
                         "device %d is sm_%d%d; this library is built for sm_90a only (no fallback)",
                         dev, prop.major, prop.minor);
      c.dev = dev;
      c.sm_count = prop.multiProcessorCount;
      CUDA_TRY(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
      CUDA_TRY(cudaStreamCreateWithFlags(&c.up, cudaStreamNonBlocking));
      CUDA_TRY(cudaStreamCreateWithFlags(&c.down, cudaStreamNonBlocking));
      CUDA_TRY(cudaEventCreateWithFlags(&c.ws_free, cudaEventDisableTiming));
      void *fn = nullptr;
      cudaDriverEntryPointQueryResult qres;
      CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
      if (!fn || qres != cudaDriverEntryPointSuccess)
        return set_error(LASER_B200_ECUDA, "cuTensorMapEncodeTiled not available from the driver");
      c.encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
      CUDA_TRY(cudaMalloc(&c.sched.ptr, kSchedSlots * 2 * sizeof(unsigned int)));
      c.sched.bytes = kSchedSlots * 2 * sizeof(unsigned int);
      CUDA_TRY(cudaMemset(c.sched.ptr, 0, c.sched.bytes));
      if (const char *kc = getenv("LASER_B200_KC")) {
        const int v = atoi(kc);
        if (v >= 32) c.kc_faithful = v;
      }
      if (const char *rg = getenv("LASER_B200_RASTER")) c.raster_g = atoi(rg);
      if (const char *sk = getenv("LASER_B200_SPLITK")) c.splitk_enabled = atoi(sk) != 0;
      if (const char *dm = getenv("LASER_B200_F64_DMMA")) c.f64_dmma = atoi(dm) != 0;
      if (const char *pt = getenv("LASER_B200_PANEL_TAPER")) c.panel_taper = atoi(pt) != 0;
      if (const char *ds = getenv("LASER_B200_DYNSCHED")) c.dyn_sched = atoi(ds) != 0;
      if (const char *pd = getenv("LASER_B200_PDL")) c.pdl = atoi(pd) != 0;
      if (const char *bw = getenv("LASER_B200_BATCH_WS_MB")) {
        const int64_t v = atoll(bw);
        if (v >= 1) c.batch_ws_bytes = v << 20;
      }
      if (const char *pr = getenv("LASER_B200_PANEL_ROWS")) {
        const int64_t v = atoll(pr) / 256 * 256;   // whole multiples of 256 rows, as the option has always been read
        if (v >= 256) c.panel_rows = v;
      }
      if (g_f32_mode.load() < 0) g_f32_mode.store(parse_f32_mode(getenv("LASER_B200_F32_MODE")));
      c.ready = true;
    }
  }
  *out = &c;
  return LASER_B200_OK;
}

int ensure(Buffer &b, size_t bytes) {
  if (b.bytes >= bytes) return LASER_B200_OK;
  if (b.ptr) CUDA_TRY(cudaFree(b.ptr));
  b.ptr = nullptr;
  b.bytes = 0;
  size_t want = bytes + (bytes >> 3);  // slack: avoid re-allocation on slightly larger calls
  want = (want + 255) & ~static_cast<size_t>(255);
  CUDA_TRY(cudaMalloc(&b.ptr, want));
  b.bytes = want;
  return LASER_B200_OK;
}

// Profiling bracket around a group of launches on one stream.  launches(): how many were made since open(), counted
// whether profiling is on or not.  With profiling on, close() records the pair with that count; a bracket that is left
// without close() (an error return) releases its events unrecorded.
struct ProfBracket {
  Ctx *c = nullptr;   // set while events are held
  cudaStream_t s = nullptr;
  EventPair ep{};
  int64_t before = 0;

  int open(Ctx &ctx, cudaStream_t stream, int kind) {
    before = g_launches.load();
    if (!ctx.profiling) return LASER_B200_OK;
    c = &ctx;
    s = stream;
    ep.kind = kind;
    CUDA_TRY(cudaEventCreate(&ep.a));
    CUDA_TRY(cudaEventCreate(&ep.b));
    CUDA_TRY(cudaEventRecord(ep.a, s));
    return LASER_B200_OK;
  }
  int launches() const { return static_cast<int>(g_launches.load() - before); }
  int close() {
    if (!c) return LASER_B200_OK;
    ep.launches = launches();
    CUDA_TRY(cudaEventRecord(ep.b, s));
    c->prof.push_back(ep);
    c = nullptr;
    return LASER_B200_OK;
  }
  ~ProfBracket() {
    if (!c) return;
    if (ep.a) cudaEventDestroy(ep.a);
    if (ep.b) cudaEventDestroy(ep.b);
  }
};

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
inline int grid_for(const Ctx &c, int64_t work_items, int per_sm) {
  int64_t g = static_cast<int64_t>(c.sm_count) * per_sm;
  if (work_items < g) g = work_items > 0 ? work_items : 1;
  return static_cast<int>(g);
}
#define COUNT_LAUNCH() g_launches.fetch_add(1, std::memory_order_relaxed)
#define CHECK_LAUNCH() CUDA_TRY(cudaGetLastError())

// ---------------------------------------------------------------------------------------
//                                   exact SIMT path
// ---------------------------------------------------------------------------------------
template <typename T, int TM, int TN, int BK>
int launch_simt(Ctx &c, int64_t M, int64_t N, int64_t K, T alpha, const T *A, int64_t rsA,
                int64_t csA, const T *B, int64_t rsB, int64_t csB, T beta, T *C, int64_t rsC,
                int64_t csC, cudaStream_t s, const Epilogue &epi, int64_t batch = 1, int64_t bsA = 0, int64_t bsB = 0,
                int64_t bsC = 0) {
  SimtParams<T> p;
  const int64_t tiles = simt_plan<T, TM, TN>(p, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);
  if constexpr (std::is_same<T, float>::value) { p.bias = epi.bias; p.bias_per_row = epi.bias_per_row; p.act = epi.act; }
  if (tiles > 0x7fffffff) return set_error(LASER_B200_EINVAL, "too many tiles");
  p.batch = batch; p.bsA = bsA; p.bsB = bsB; p.bsC = bsC;
  const int grid = grid_for(c, tiles * batch, 2);
  if (batch > 1) gemm_simt_batched_kernel<T, TM, TN, BK><<<grid, 256, 0, s>>>(p);
  else gemm_simt_kernel<T, TM, TN, BK><<<grid, 256, 0, s>>>(p);
  COUNT_LAUNCH();
  CHECK_LAUNCH();
  return LASER_B200_OK;
}

template <typename T>
int gemm_simt(Ctx &c, int64_t M, int64_t N, int64_t K, T alpha, const T *A, int64_t rsA,
              int64_t csA, const T *B, int64_t rsB, int64_t csB, T beta, T *C, int64_t rsC,
              int64_t csC, cudaStream_t s, const Epilogue &epi = Epilogue(), int64_t batch = 1, int64_t bsA = 0,
              int64_t bsB = 0, int64_t bsC = 0) {
#ifndef LB200_SIMT_BK
#define LB200_SIMT_BK 16
#endif
  if constexpr (std::is_same<T, double>::value) {
    // fp64 tensor cores (mma.sync DMMA, gemm_dmma.cuh) once the 128 x 128 tiles fill at least half of the SMs: the same
    // FMA chain per element as the CUDA-core kernel, bit for bit, so the choice is a matter of speed only
    const int64_t tiles128 = ((M + DMMA_BM - 1) / DMMA_BM) * ((N + DMMA_BN - 1) / DMMA_BN) * batch;
    if (c.f64_dmma && 2 * tiles128 >= c.sm_count) {
      SimtParams<double> p;
      const int64_t tiles = dmma_plan(p, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);
      if (tiles * batch > 0x7fffffff) return set_error(LASER_B200_EINVAL, "too many tiles");
      p.batch = batch; p.bsA = bsA; p.bsB = bsB; p.bsC = bsC;
      if (!c.dmma_attr_set) {
        CUDA_TRY(cudaFuncSetAttribute(gemm_dmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(DMMA_SMEM_BYTES)));
        c.dmma_attr_set = true;
      }
      gemm_dmma_kernel<<<grid_for(c, tiles * batch, 1), 256, DMMA_SMEM_BYTES, s>>>(p);
      g_dmma_launches.fetch_add(1);
      COUNT_LAUNCH();
      CHECK_LAUNCH();
      return LASER_B200_OK;
    }
  }
  if constexpr (std::is_same<T, float>::value) {
    // few output rows, wide N (the im2col convolution's GEMM): a thread owns 4 columns of all rows, B and C stream once;
    // the same FMA chain per element as the general kernel (gemm_simt.cuh: gemm_skinny_m_kernel)
    if (M <= 32 && N >= 1024) {
      SimtParams<float> p;
      simt_plan<float, 8, 8>(p, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);
      p.bias = epi.bias; p.bias_per_row = epi.bias_per_row; p.act = epi.act;
      p.batch = batch; p.bsA = bsA; p.bsB = bsB; p.bsC = bsC;
      // B with unit column stride and 16-byte aligned rows streams through shared memory (cp.async FIFO per thread)
      const bool async_ok = csB == 1 && rsB % 4 == 0 && (batch == 1 || bsB % 4 == 0) && (reinterpret_cast<uintptr_t>(B) & 15) == 0;
      if (async_ok) {
        const int grid = grid_for(c, ((N + 1023) / 1024) * batch, 1);
#define LB200_SKA(MT)                                                                                                  \
  do {                                                                                                                 \
    static std::atomic<uint32_t> attr_set{0};                                                                          \
    if (!(attr_set.load(std::memory_order_acquire) & (1u << c.dev))) {                                                 \
      CUDA_TRY(cudaFuncSetAttribute(gemm_skinny_m_async_kernel<MT>, cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                                    static_cast<int>(ska_smem_bytes<MT>())));                                          \
      attr_set.fetch_or(1u << c.dev, std::memory_order_release);                                                       \
    }                                                                                                                  \
    gemm_skinny_m_async_kernel<MT><<<grid, 256, ska_smem_bytes<MT>(), s>>>(p);                                         \
  } while (0)
        if (M <= 8) LB200_SKA(8); else if (M <= 16) LB200_SKA(16); else if (M <= 24) LB200_SKA(24); else LB200_SKA(32);
#undef LB200_SKA
        COUNT_LAUNCH();
        CHECK_LAUNCH();
        return LASER_B200_OK;
      }
      const int nc = M <= 16 ? 4 : 2;   // columns per thread (gemm_simt.cuh)
      const int grid = grid_for(c, ((N + 256 * nc - 1) / (256 * nc)) * batch, 2);
      if (M <= 8) gemm_skinny_m_kernel<8, 4><<<grid, 256, 0, s>>>(p);
      else if (M <= 16) gemm_skinny_m_kernel<16, 4><<<grid, 256, 0, s>>>(p);
      else if (M <= 24) gemm_skinny_m_kernel<24, 2><<<grid, 256, 0, s>>>(p);
      else gemm_skinny_m_kernel<32, 2><<<grid, 256, 0, s>>>(p);
      COUNT_LAUNCH();
      CHECK_LAUNCH();
      return LASER_B200_OK;
    }
  }
  if constexpr (sizeof(T) == 4)
    return launch_simt<T, 8, 8, LB200_SIMT_BK>(c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, batch,
                                               bsA, bsB, bsC);
  else
    return launch_simt<T, 4, 4, 16>(c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, batch, bsA, bsB,
                                    bsC);
}

// ---------------------------------------------------------------------------------------
//                                  tensor-core path
// ---------------------------------------------------------------------------------------
// An operand of the contraction seen as [mn][k]: for A mn = M (s_mn = rowStrideA,
// s_k = colStrideA), for B mn = N (s_mn = colStrideB, s_k = rowStrideB).
struct Operand {
  const void *ptr;
  int64_t mn, k, s_mn, s_k;
  // batched launch: `batch` problems s_b elements apart (the aux of their op: aux_sb apart), read through rank-3 tensor maps;
  // batch 1 with a batched launch is an operand the problems share.  0: a single problem, rank-2 maps.
  int64_t batch = 0, s_b = 0, aux_sb = 0;
  // an im2col source: B of a convolution, [mn = outH * outW][k = C * kH * kW] per image, read from the `batch` NCHW images at
  // ptr, s_b floats apart (s_mn, s_k unused).  With `concat`: a concatenated im2col source, the B of a convolution's filter
  // gradient, [mn = C * kH * kW][k = outH * outW] per image, the `batch` images' k-segments end to end
  const ConvGeom *conv = nullptr;
  // a concatenated batch: the operand of a sum of products, [mn][batch * k], whose k-segment b is problem b's [mn][k] (s_b
  // apart, 0: the same matrix in every segment); prepared into compact workspace and read through rank-2 maps
  bool concat = false;
};
enum Major { K_MAJOR = 0, MN_MAJOR = 1, GENERAL = 2 };

Major classify(const Operand &o, int esz) {
  const bool aligned = (reinterpret_cast<uintptr_t>(o.ptr) & 15) == 0;
  if (!aligned) return GENERAL;
  const int64_t lim = (static_cast<int64_t>(1) << 40) / esz;
  if (o.s_k == 1 && o.s_mn > 0 && (o.s_mn * esz) % 16 == 0 && o.s_mn < lim) return K_MAJOR;
  if (o.s_mn == 1 && o.s_k > 0 && (o.s_k * esz) % 16 == 0 && o.s_k < lim) return MN_MAJOR;
  return GENERAL;
}

int encode_map(Ctx &c, CUtensorMap *map, int esz, const void *base, int64_t inner, int64_t outer,
               int64_t outer_stride_elems, int box_inner, int box_outer, CUtensorMapSwizzle swz, int64_t depth = 0,
               int64_t depth_stride = 0) {
  const MapKey key{base, inner, outer, outer_stride_elems, esz, box_inner, box_outer, static_cast<int>(swz), depth, depth_stride};
  for (int i = 0; i < kMapCacheSize; ++i)
    if (c.map_cache[i].valid && c.map_cache[i].key == key) {
      *map = c.map_cache[i].map;
      return LASER_B200_OK;
    }
  // rank 3: {inner, outer, depth} with a box depth of 1 -- one matrix of a batch per load, zero-filled at its own edges
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(outer), static_cast<cuuint64_t>(depth)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(outer_stride_elems) * esz, static_cast<cuuint64_t>(depth_stride) * esz};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_outer), 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  // 16-bit tiles travel as BFLOAT16 whatever their format (bf16 / fp16): TMA only moves the words
  const CUtensorMapDataType dt = esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = c.encode(map, dt, depth > 0 ? 3 : 2, const_cast<void *>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(LASER_B200_ECUDA,
                     "cuTensorMapEncodeTiled failed (%d): base=%p inner=%lld outer=%lld stride=%lld box=%dx%d",
                     static_cast<int>(r), base, (long long)inner, (long long)outer,
                     (long long)outer_stride_elems, box_inner, box_outer);
  MapCacheEntry &e = c.map_cache[c.map_cache_next];
  c.map_cache_next = (c.map_cache_next + 1) % kMapCacheSize;
  e.key = key;
  e.map = *map;
  e.valid = true;
  return LASER_B200_OK;
}

// tensor map for one operand given as compact/strided [mn][k] data with the stated major-ness
// (depth > 0: rank 3 over `depth` such operands depth_stride elements apart)
int operand_map(Ctx &c, CUtensorMap *map, int esz, const void *base, Major major, int64_t mn,
                int64_t k, int64_t ld, int block_mn, int64_t depth = 0, int64_t depth_stride = 0) {
  const int block_k = TC_ROW_BYTES / esz;
  const int mn_atom = TC_ROW_BYTES / esz;
  if (major == K_MAJOR)
    return encode_map(c, map, esz, base, k, mn, ld, block_k, block_mn, CU_TENSOR_MAP_SWIZZLE_128B, depth, depth_stride);
  // MN-major fp32/tf32 tiles need the 32-byte-atom flavour of the 128B swizzle (see ptx.cuh)
  return encode_map(c, map, esz, base, mn, k, ld, mn_atom, block_k,
                    esz == 4 ? CU_TENSOR_MAP_SWIZZLE_128B_ATOM_32B : CU_TENSOR_MAP_SWIZZLE_128B, depth, depth_stride);
}

// Tensor maps of one operand for the tensor-core kernel: piece 0 = the operand itself (one pass) or its high piece,
// piece 1 = its low piece (three-pass modes).
struct OperandMaps {
  CUtensorMap p0, p1;
  bool mn_major = false;
};
struct OperandWs {
  Buffer *p0, *p1, *gather;
  int64_t amax_off;   // F16X3: word offset of the operand's abs-max vector in Ctx::f16s (set by f16_scales)
};
// how an fp32 operand reaches the kernel
enum SplitMode {
  SPLIT_NONE = 0,    // as it is: TMA reads the caller's memory (TF32X1; bf16 operands)
  SPLIT_TF32 = 1,    // hi = tf32_rna(x), lo = tf32_rna(x - hi) in fp32 containers (TF32X3)
  SPLIT_F16X2 = 2,   // abs-max word per mn index + two fp16 pieces of the scaled operand (F16X3, the default)
};

// Operand ops of the fused-prologue entry.  Host side, `OperandOp` describes aux as [mn][k] like its Operand
// (aux_sr = s_mn, aux_sc = s_k); the preparation kernels see it over their [R][Cc] rows, where R runs along k when the
// prepared layout is MN-major.
inline OperandOp kernel_op(const OperandOp &op, bool rows_along_k) {
  OperandOp k = op;
  if (rows_along_k) { k.aux_sr = op.aux_sc; k.aux_sc = op.aux_sr; }
  return k;
}
// aux can be read at the operand's own offsets by the row kernels
inline bool op_same_layout(const Operand &o, const OperandOp &op) {
  return !op.aux || (op.aux_sr == o.s_mn && op.aux_sc == o.s_k && (reinterpret_cast<uintptr_t>(op.aux) & 15) == 0);
}

// ---- the preparation steps: one function, and one launch site, per kernel family of split.cuh ----
// A step takes its op as a pointer (nullptr: none) and its problems as a Batch (n == 1: one problem), and hands `launch`
// (has_op, op, batched, concat): has_op is std::true_type with *op or std::false_type with OperandOp(), batched is
// std::true_type when bt.n > 1, concat std::true_type for a concatenated batch (Operand::concat, with batched).  The kernel's
// plain, HAS_OP, BATCHED and CONCAT instantiations come from the same launch statement.
template <typename Launch>
int launch_prep(const OperandOp *op, const Batch &bt, Launch launch, bool concat = false) {
  auto with_op = [&](auto batched, auto cat) {
    if (op) launch(std::true_type(), *op, batched, cat);
    else launch(std::false_type(), OperandOp(), batched, cat);
  };
  if (concat) with_op(std::true_type(), std::true_type());
  else if (bt.n > 1) with_op(std::true_type(), std::false_type());
  else with_op(std::false_type(), std::false_type());
  COUNT_LAUNCH();
  CHECK_LAUNCH();
  return LASER_B200_OK;
}
// the problems an operand's preparation covers (an operand the batch shares: one)
inline Batch batch_of(const Operand &o) { return Batch{o.batch > 1 ? o.batch : 1, o.s_b, o.aux_sb}; }

// The gather: op(operand), or the operand itself, from any strides into compact K-major rows [mn][round_up(k, 16 / sizeof(T))]
// allocated in dst (aux read with its own strides).  MODE 1 (fp32): the tf32 hi / lo pieces into dst / *lo.  bf16 operands
// carry no op.
// A batched operand: the problems' rows stacked, [batch][mn][ld]; a concatenated one: [mn][round_up(batch * k, ..)].
template <typename T, int MODE = 0>
int gather(Ctx &c, const Operand &o, Buffer &dst, Buffer *lo, cudaStream_t s, const OperandOp *op = nullptr) {
  const Batch bt = batch_of(o);
  const int64_t ld = round_up(o.concat ? bt.n * o.k : o.k, 16 / static_cast<int64_t>(sizeof(T)));
  const size_t bytes = static_cast<size_t>((o.concat ? 1 : bt.n) * o.mn) * ld * sizeof(T);
  int rc;
  if ((rc = ensure(dst, bytes))) return rc;
  if (MODE == 1 && (rc = ensure(*lo, bytes))) return rc;
  const int64_t tiles = ((o.mn + 31) / 32) * ((o.k + 31) / 32) * bt.n;
  const int read_along_r = (llabs(o.s_mn) < llabs(o.s_k)) ? 1 : 0;
  T *d0 = static_cast<T *>(dst.ptr), *d1 = MODE == 1 ? static_cast<T *>(lo->ptr) : nullptr;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched, auto cat) {
    constexpr bool HAS_OP = decltype(has_op)::value && sizeof(T) == 4, BATCHED = decltype(batched)::value && sizeof(T) == 4,
                   CONCAT = decltype(cat)::value && sizeof(T) == 4;
    pack_general_kernel<T, MODE, HAS_OP, BATCHED, CONCAT><<<grid_for(c, tiles, 8), 256, 0, s>>>(
        static_cast<const T *>(o.ptr), o.mn, o.k, o.s_mn, o.s_k, d0, d1, ld, read_along_r, k, bt);
  }, o.concat);
}

// TF32X3 in place: tf32 hi / lo pieces [R][ld] of fp32 rows [R][Cc], src_ld apart (concat: of the batch's rows laid end to
// end, [R][bt.n * Cc])
int tf32_split(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, float *hi, float *lo, int64_t ld, cudaStream_t s,
               const OperandOp *op, const Batch &bt = Batch(), bool concat = false) {
  const int64_t items = concat ? R * ((bt.n * Cc + 3) / 4) : bt.n * R * ((Cc + 3) / 4);
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched, auto cat) {
    constexpr bool HAS_OP = decltype(has_op)::value, BATCHED = decltype(batched)::value, CONCAT = decltype(cat)::value;
    split_rows_tf32_kernel<HAS_OP, BATCHED, CONCAT><<<grid_for(c, (items + 255) / 256, 8), 256, 0, s>>>(src, R, Cc, src_ld, hi, lo,
                                                                                                       ld, k, bt);
  }, concat);
}

// F16X3, one scale per row of fp32 rows [R][Cc] (src_ld apart): the abs-max word of each row, the scale and the two fp16
// pieces [R][ld_b] in ONE pass (split.cuh).  Rows of up to 1024 floats: a warp per row.  Longer rows: prefetched into a
// shared-memory ring by the copy engine when they allow it (16-byte aligned, at most 8192 floats; the ring kernel has no op
// variant, nor a batched one), the CTA per row otherwise.  concat: the batch's rows laid end to end, rows of bt.n * Cc floats.
int f16x2_rows(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
               uint32_t *words, cudaStream_t s, const OperandOp *op = nullptr, const Batch &bt = Batch(), bool concat = false) {
  const bool ring = !op && bt.n == 1 && f16x2_rows_ring_ok(src, Cc, src_ld);
  if (ring && !c.ring_attr_set) {
    CUDA_TRY(cudaFuncSetAttribute(f16x2_rows_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(f16x2_rows_ring_smem(4 * 256 * F16ROWS_MAXV))));
    c.ring_attr_set = true;
  }
  const int64_t rows = concat ? R : bt.n * R, row_len = concat ? bt.n * Cc : Cc;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched, auto cat) {
    constexpr bool HAS_OP = decltype(has_op)::value, BATCHED = decltype(batched)::value, CONCAT = decltype(cat)::value;
    if (row_len <= 4 * 32 * F16ROWS_MAXV)
      f16x2_rows_fused_kernel<32, HAS_OP, BATCHED, CONCAT><<<grid_for(c, (rows + 7) / 8, 4), 256, 0, s>>>(src, R, Cc, src_ld, hb, lb,
                                                                                                     ld_b, words, k, bt);
    else if (ring)
      f16x2_rows_ring_kernel<<<grid_for(c, R, 2), 256, f16x2_rows_ring_smem(Cc), s>>>(src, R, Cc, src_ld, hb, lb, ld_b, words);
    else
      f16x2_rows_fused_kernel<256, HAS_OP, BATCHED, CONCAT><<<grid_for(c, rows, 4), 256, 0, s>>>(src, R, Cc, src_ld, hb, lb, ld_b,
                                                                                                words, k, bt);
  }, concat);
}

// F16X3, one scale per column of fp32 rows [R][Cc]: the abs-max word of every column (zeroed here, then strip reductions
// combined by atomicMax).  A column's scale needs the whole column, so the split is a second pass.  concat: one word per
// column over every problem of the batch.
int f16x2_col_scales(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint32_t *words, cudaStream_t s,
                     const OperandOp *op = nullptr, const Batch &bt = Batch(), bool concat = false) {
  CUDA_TRY(cudaMemsetAsync(words, 0, static_cast<size_t>((concat ? 1 : bt.n) * Cc) * sizeof(uint32_t), s));
  const int64_t items = ((Cc + 3) / 4) * ((R + ABSMAX_COL_ROWS - 1) / ABSMAX_COL_ROWS) * bt.n;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched, auto cat) {
    constexpr bool HAS_OP = decltype(has_op)::value, BATCHED = decltype(batched)::value, CONCAT = decltype(cat)::value;
    absmax_mn_kernel<true, HAS_OP, BATCHED, CONCAT><<<grid_for(c, (items + 255) / 256, 8), 256, 0, s>>>(src, R, Cc, src_ld, words, k,
                                                                                                       bt);
  }, concat);
}
// F16X3, one scale per column: the two fp16 pieces [R][ld_b] of fp32 rows [R][Cc] against the columns' scale words
int f16x2_col_split(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
                    const uint32_t *words, cudaStream_t s, const OperandOp *op = nullptr, const Batch &bt = Batch(),
                    bool concat = false) {
  const int64_t items = ((Cc + 255) / 256) * ((R + SPLIT_ROWS - 1) / SPLIT_ROWS) * bt.n;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched, auto cat) {
    constexpr bool HAS_OP = decltype(has_op)::value, BATCHED = decltype(batched)::value, CONCAT = decltype(cat)::value;
    split_rows_f16x2_kernel<true, HAS_OP, BATCHED, CONCAT><<<grid_for(c, items, 8), 256, 0, s>>>(src, R, Cc, src_ld, hb, lb, ld_b,
                                                                                                words, k, bt);
  }, concat);
}

// An im2col source (Operand::conv): every image's windows as K-major rows [batch][mn][ld] (split.cuh: im2col_rows_kernel) in
// the format of `mode` -- words and fp16 pieces into hb / lb / words (F16X2), tf32 hi / lo into dst / dst_lo (TF32), the
// values into dst (NONE: TF32X1 and the exact path).  A concatenated one (with Operand::concat): the tap rows [mn][ld] of
// every image end to end (split.cuh: im2col_tap_rows_kernel), F16X2 after an abs-max pass over the same tiles.
// A dilated source (ConvGeom::dH, dW) or an op: the transposed source of the input gradient, the rows kernel's DIL / HAS_OP
// instantiations (op applied to the values read, its aux dense like the images; not with `concat`).
// A channels-last source (ConvGeom::nhwc): the windows of NHWC images in (kh, kw, c) order, the rows kernel's NHWC
// instantiations; one problem, mn = images * outH * outW rows; dilated or op'd, the channels-last transposed source of the
// NHWC input gradient (Im2colNhwcGradSrc; vector loads only when the aux is 16-byte aligned too).  Oriented as tap rows
// (ConvGeom::taps, neither dilated nor op'd): mn = the taps, k = the
// pixels of every image end to end (split.cuh: im2col_nhwc_tap_rows_kernel), F16X2 after an abs-max pass over the same tiles.
int im2col_rows(Ctx &c, const Operand &o, SplitMode mode, float *dst, float *dst_lo, uint16_t *hb, uint16_t *lb, int64_t ld,
                uint32_t *words, cudaStream_t s, const OperandOp *op = nullptr) {
  const Im2colSrc q = im2col_src(*o.conv);
  const Batch bt = batch_of(o);
  // the images of the launch: a batch of problems of outHW rows each (the NCHW sources), or one problem whose mn rows are the
  // pixels of every image (the channels-last source, A of the NHWC forward call), or whose k columns are (the tap rows)
  const int64_t images = o.conv->taps ? o.k / q.outHW : o.concat ? bt.n : bt.n * (o.mn / q.outHW), rows = bt.n * o.mn;
  // the work items of a tap-row launch: tiles of TAP_SEG columns of one row (NCHW), of NHWC_TAPS rows x NHWC_PIX columns (NHWC)
  const int64_t tiles = o.conv->taps ? ((o.mn + NHWC_TAPS - 1) / NHWC_TAPS) * ((ld + NHWC_PIX - 1) / NHWC_PIX)
                                     : o.mn * ((ld + TAP_SEG - 1) / TAP_SEG);
  const float *in = static_cast<const float *>(o.ptr);
  const bool dil = o.conv->dH != 1 || o.conv->dW != 1;
  if (o.concat && (dil || op)) return set_error(LASER_B200_ECUDA, "internal: a concatenated im2col source has no dilation or op");
  if (o.conv->nhwc && o.concat) return set_error(LASER_B200_ECUDA, "internal: a channels-last im2col source is not concatenated");
  if (o.conv->taps && (!o.conv->nhwc || dil || op))
    return set_error(LASER_B200_ECUDA, "internal: only a channels-last source without dilation or op has tap rows");
  auto launch = [&](auto m, auto absmax) {
    constexpr int MODE = decltype(m)::value, PER_SM = MODE == IM2COL_F16X2 ? 3 : 4;   // the kernel's launch bounds
    auto rows_kernel = [&](auto d, auto has_op, const auto &src) {
      constexpr bool DIL = decltype(d)::value, HAS_OP = decltype(has_op)::value;
      constexpr bool NHWC = std::is_base_of<Im2colNhwcSrc, typename std::decay<decltype(src)>::type>::value;
      if (ld <= 4 * 32 * F16ROWS_MAXV)
        im2col_rows_kernel<MODE, 32, DIL, HAS_OP, NHWC><<<grid_for(c, (rows + 7) / 8, PER_SM), 256, 0, s>>>(in, src, images, dst,
                                                                                                         dst_lo, hb, lb, ld, words);
      else
        im2col_rows_kernel<MODE, 256, DIL, HAS_OP, NHWC><<<grid_for(c, rows, PER_SM), 256, 0, s>>>(in, src, images, dst, dst_lo, hb,
                                                                                                lb, ld, words);
    };
    if (o.conv->taps) {
      im2col_nhwc_tap_rows_kernel<MODE, decltype(absmax)::value><<<grid_for(c, tiles, NHWC_PER_SM), 256, 0, s>>>(
          in, im2col_nhwc_src(*o.conv, in), images, dst, dst_lo, hb, lb, ld, words);
    } else if (o.conv->nhwc && (dil || op)) {
      Im2colNhwcGradSrc gq{};
      static_cast<Im2colNhwcSrc &>(gq) = im2col_nhwc_src(*o.conv, in);
      gq.vec = gq.vec && (!op || !op->aux || (reinterpret_cast<uintptr_t>(op->aux) & 15) == 0);
      gq.dH = static_cast<int>(o.conv->dH);
      gq.dW = static_cast<int>(o.conv->dW);
      if (op) gq.op = *op;
      if (dil && op) rows_kernel(std::true_type(), std::true_type(), gq);
      else if (dil) rows_kernel(std::true_type(), std::false_type(), gq);
      else rows_kernel(std::false_type(), std::true_type(), gq);
    } else if (o.conv->nhwc) {
      rows_kernel(std::false_type(), std::false_type(), im2col_nhwc_src(*o.conv, in));
    } else if (o.concat) {
      im2col_tap_rows_kernel<MODE, decltype(absmax)::value><<<grid_for(c, tiles, 8), 256, 0, s>>>(in, q, images, dst, dst_lo, hb, lb,
                                                                                                 ld, words);
    } else if (dil || op) {
      Im2colGradSrc gq{};
      static_cast<Im2colSrc &>(gq) = q;
      gq.dH = static_cast<int>(o.conv->dH);
      gq.dW = static_cast<int>(o.conv->dW);
      if (op) gq.op = *op;
      if (dil && op) rows_kernel(std::true_type(), std::true_type(), gq);
      else if (dil) rows_kernel(std::true_type(), std::false_type(), gq);
      else rows_kernel(std::false_type(), std::true_type(), gq);
    } else {
      rows_kernel(std::false_type(), std::false_type(), q);
    }
    COUNT_LAUNCH();
    CHECK_LAUNCH();
    return LASER_B200_OK;
  };
  if (mode == SPLIT_F16X2 && (o.concat || o.conv->taps)) {   // one word per tap row over every image
    CUDA_TRY(cudaMemsetAsync(words, 0, static_cast<size_t>(o.mn) * sizeof(uint32_t), s));
    const int rc = launch(std::integral_constant<int, IM2COL_F16X2>(), std::true_type());
    if (rc) return rc;
  }
  if (mode == SPLIT_F16X2) return launch(std::integral_constant<int, IM2COL_F16X2>(), std::false_type());
  if (mode == SPLIT_TF32) return launch(std::integral_constant<int, IM2COL_TF32>(), std::false_type());
  return launch(std::integral_constant<int, IM2COL_F32>(), std::false_type());
}

// An fp32 operand as compact K-major rows [rows][round_up(k, 4)] (concatenated: [mn][round_up(batch * k, 4)]) in dst: gathered
// from any strides with op applied, or an im2col source's windows.  SPLIT_TF32: the tf32 hi / lo pieces into dst / *lo,
// SPLIT_NONE: the values (TF32X1 and the exact path).
int f32_rows(Ctx &c, const Operand &o, SplitMode mode, Buffer &dst, Buffer *lo, cudaStream_t s, const OperandOp *op) {
  if (!o.conv) return mode == SPLIT_TF32 ? gather<float, 1>(c, o, dst, lo, s, op) : gather<float>(c, o, dst, nullptr, s, op);
  const Batch bt = batch_of(o);
  const int64_t ld = round_up(o.concat ? bt.n * o.k : o.k, 4);
  const size_t bytes = static_cast<size_t>((o.concat ? 1 : bt.n) * o.mn) * ld * sizeof(float);
  int rc;
  if ((rc = ensure(dst, bytes))) return rc;
  if (mode == SPLIT_TF32 && (rc = ensure(*lo, bytes))) return rc;
  return im2col_rows(c, o, mode, static_cast<float *>(dst.ptr), mode == SPLIT_TF32 ? static_cast<float *>(lo->ptr) : nullptr,
                     nullptr, nullptr, ld, nullptr, s, op);
}

// One operand of a tensor-core call: first the plan, then its steps.
//   An im2col source: one pass from the images into the prepared rows, K-major like a gathered operand.
//   A concatenated im2col source: the tap rows of every image end to end, K-major [mn][batch * k] (F16X3: an abs-max pass
//     over the images first, then the split pass).
//   bf16 K- or MN-major; TF32X1 K-major without op: TMA reads the caller's memory, no workspace.
//   TF32X3 K-major; F16X3 K- or MN-major -- without op, or with aux laid out like the operand: the split reads the caller's
//     memory and applies the op on load (F16X3 MN-major: all column scales first, then the split).
//   Anything else: one gather, which applies the op, into compact K-major rows.  TMA reads those (bf16, TF32X1), the gather
//     splits them on the way (TF32X3), or the plain row kernel prepares them (F16X3).
// wgmma reads tf32 tiles K-major only, and TMA applies no op.  op: nullptr, or an operand op (fp32 operands only).
// A batched operand (o.batch > 0) is prepared in the same launches, every problem's pieces and scale words stacked; its
// maps are rank 3.  It is read in place only where every problem is: TMA needs a positive batch stride of whole 16-byte
// units, the preparation kernels 16-byte aligned rows (operand and aux) in every problem.
// A concatenated batch (o.concat) takes the same rows with the CONCAT kernels -- K-major: each row is the problems' rows laid
// end to end; MN-major (F16X3): the problems' rows stacked, one scale word per column -- into workspace read through rank-2
// maps of extent batch * k.  It is never read in place: one 2-D map cannot address the problems' segments.
template <int ESZ>
int prepare_operand(Ctx &c, const Operand &o, SplitMode mode, const OperandWs &w, int block_mn,
                    OperandMaps *m, bool *used_ws, cudaStream_t s, const OperandOp *op = nullptr) {
  const bool conv = o.conv != nullptr;   // (fp32; its op is applied by the rows kernel as it reads the source)
  const Major mj = conv ? K_MAJOR : classify(o, ESZ);
  const Batch bt = batch_of(o);
  const bool cat = o.concat;
  const int64_t kk = cat ? bt.n * o.k : o.k;                 // k extent of the operand the tensor-core kernel reads
  const bool rows_ok = bt.n == 1 || ((o.s_b * ESZ) % 16 == 0 && (!op || !op->aux || o.aux_sb % 4 == 0));
  const bool map_ok = bt.n == 1 || (o.s_b > 0 && o.s_b < (static_cast<int64_t>(1) << 40) / ESZ);
  const bool tma_layout = (mj == K_MAJOR || (mj == MN_MAJOR && (ESZ == 2 || mode == SPLIT_F16X2))) && rows_ok;
  const bool in_place = !conv && tma_layout && (mode == SPLIT_NONE ? !op && map_ok && !cat : !op || op_same_layout(o, *op));
  const Major out_mj = in_place ? mj : K_MAJOR;              // layout of the arrays the tensor-core kernel reads
  const int64_t R = (out_mj == K_MAJOR) ? o.mn : o.k;        // their rows (per problem)
  const int64_t Cc = (out_mj == K_MAJOR) ? o.k : o.mn;       // their contiguous extent (per problem)
  const int64_t src_ld = (mj == K_MAJOR) ? o.s_mn : o.s_k;   // row pitch of the operand, read in place
  // the prepared arrays: rows_p rows of row_len elements (a concatenated K-major operand: the problems' rows end to end)
  const bool cat_rows = cat && out_mj == K_MAJOR;
  const int64_t rows_p = cat_rows ? R : bt.n * R, row_len = cat_rows ? bt.n * Cc : Cc;
  const int64_t ld = round_up(row_len, 16 / ESZ);
  // rank-3 maps of a batched launch: `depth` matrices (1: shared by the batch) `d_stride(pitch)` elements apart
  const int64_t depth = o.batch > 0 && !cat ? bt.n : 0;
  auto d_stride = [&](int64_t pitch) { return bt.n > 1 ? (in_place && mode == SPLIT_NONE ? o.s_b : R * pitch) : R * pitch; };
  m->mn_major = (out_mj == MN_MAJOR);
  int rc;
  if (mode == SPLIT_NONE && in_place) {
    if ((rc = operand_map(c, &m->p0, ESZ, o.ptr, mj, o.mn, o.k, src_ld, block_mn, depth, d_stride(src_ld)))) return rc;
    m->p1 = m->p0;
    return LASER_B200_OK;
  }
  *used_ws = true;
  if constexpr (ESZ == 2) {
    if ((rc = gather<uint16_t>(c, o, *w.p0, nullptr, s))) return rc;
  } else {
    const float *src = static_cast<const float *>(o.ptr);
    const OperandOp kop = op ? kernel_op(*op, out_mj == MN_MAJOR) : OperandOp();
    const OperandOp *on_load = (in_place && op) ? &kop : nullptr;
    if (mode == SPLIT_F16X2) {
      const int64_t ld_b = round_up(row_len, 8);
      const size_t bytes_b = static_cast<size_t>(rows_p) * ld_b * 2;
      if ((rc = ensure(*w.p0, bytes_b))) return rc;
      if ((rc = ensure(*w.p1, bytes_b))) return rc;
      if (c.f16s.bytes < static_cast<size_t>(w.amax_off + (cat ? 1 : bt.n) * o.mn) * sizeof(uint32_t))
        return set_error(LASER_B200_ECUDA, "internal: F16X3 scale buffer not sized for this operand");
      uint16_t *hb = static_cast<uint16_t *>(w.p0->ptr), *lb = static_cast<uint16_t *>(w.p1->ptr);
      uint32_t *words = static_cast<uint32_t *>(c.f16s.ptr) + w.amax_off;
      if (conv) {
        rc = im2col_rows(c, o, mode, nullptr, nullptr, hb, lb, ld_b, words, s, op);
      } else if (!in_place) {   // the gathered problems are stacked (concatenated) rows: one plain row pass over all of them
        if ((rc = gather<float>(c, o, *w.gather, nullptr, s, op))) return rc;
        rc = f16x2_rows(c, static_cast<const float *>(w.gather->ptr), rows_p, row_len, ld, hb, lb, ld_b, words, s);
      } else if (out_mj == K_MAJOR) {
        rc = f16x2_rows(c, src, R, Cc, src_ld, hb, lb, ld_b, words, s, on_load, bt, cat);
      } else {
        if ((rc = f16x2_col_scales(c, src, R, Cc, src_ld, words, s, on_load, bt, cat))) return rc;
        rc = f16x2_col_split(c, src, R, Cc, src_ld, hb, lb, ld_b, words, s, on_load, bt, cat);
      }
      if (rc) return rc;
      if ((rc = operand_map(c, &m->p0, 2, w.p0->ptr, out_mj, o.mn, kk, ld_b, block_mn, depth, d_stride(ld_b)))) return rc;
      return operand_map(c, &m->p1, 2, w.p1->ptr, out_mj, o.mn, kk, ld_b, block_mn, depth, d_stride(ld_b));
    }
    if (!in_place || conv) {
      rc = f32_rows(c, o, mode, *w.p0, w.p1, s, op);
    } else {   // TF32X3 K-major: the split reads the caller's memory
      const size_t bytes = static_cast<size_t>(rows_p) * ld * sizeof(float);
      if ((rc = ensure(*w.p0, bytes))) return rc;
      if ((rc = ensure(*w.p1, bytes))) return rc;
      rc = tf32_split(c, src, R, Cc, src_ld, static_cast<float *>(w.p0->ptr), static_cast<float *>(w.p1->ptr), ld, s, on_load, bt, cat);
    }
    if (rc) return rc;
  }
  if ((rc = operand_map(c, &m->p0, ESZ, w.p0->ptr, out_mj, o.mn, kk, ld, block_mn, depth, d_stride(ld)))) return rc;
  m->p1 = m->p0;
  if (mode == SPLIT_TF32) return operand_map(c, &m->p1, ESZ, w.p1->ptr, out_mj, o.mn, kk, ld, block_mn, depth, d_stride(ld));
  return LASER_B200_OK;
}

inline OperandWs ws_of_A(Ctx &c) { return OperandWs{&c.ws[0], &c.ws[1], &c.gather[0], 0}; }
inline OperandWs ws_of_B(Ctx &c, int64_t amax_off = 0) { return OperandWs{&c.ws[2], &c.ws[3], &c.gather[1], amax_off}; }
// F16X3: room for M + N abs-max words; A's vector starts at word 0, B's at the returned offset
inline int f16_scales(Ctx &c, int64_t M, int64_t N, int64_t *b_off) {
  *b_off = round_up(M, 64);
  return ensure(c.f16s, static_cast<size_t>(*b_off + N) * sizeof(uint32_t));
}
struct F16Scales {     // where the two abs-max vectors of the current call live (device memory)
  const uint32_t *a = nullptr, *b = nullptr;
};

// kernel family of a tensor-core call
enum TcKind { TC_TF32X1, TC_TF32X3, TC_BF16, TC_F16X3 };
inline TcKind tc_kind_of_path(int path) {
  return path == LASER_B200_PATH_TF32X1 ? TC_TF32X1 : path == LASER_B200_PATH_TF32X3 ? TC_TF32X3 : TC_F16X3;
}
inline SplitMode split_mode(TcKind k) { return k == TC_TF32X3 ? SPLIT_TF32 : k == TC_F16X3 ? SPLIT_F16X2 : SPLIT_NONE; }

// a batched launch: `batch` problems, C of problem b at C + b * C_stride; a per-row bias of problem b at bias + (b % A's period)
// * bias_stride (0: one bias for the batch)
struct BatchArgs {
  int64_t batch, C, bias = 0;
};

// launch the tensor-core kernel on prepared operands (c.mu held by the caller).  bat: a batched launch (tc_params.h; the maps
// are rank 3), problem b reading slice b % period_a of A and b % period_b of B (1: an operand prepared once for the batch).
template <typename OutT>
int tc_run(Ctx &c, TcKind kind, int64_t M, int64_t N, int64_t K, float alpha, const OperandMaps &ma,
           const OperandMaps &mb, float beta, OutT *C, int64_t rsC, int64_t csC, cudaStream_t s,
           const Epilogue &epi, const F16Scales *f16 = nullptr, bool after_prep = false, const BatchArgs *bat = nullptr,
           int64_t period_a = 1, int64_t period_b = 1) {
  TcLaunch l;
  l.a0 = ma.p0; l.a1 = ma.p1; l.b0 = mb.p0; l.b1 = mb.p1;
  l.a_mn = ma.mn_major; l.b_mn = mb.mn_major;
  l.pdl = c.pdl && after_prep;   // the preceding kernel of the stream is one of ours and calls launch_dependents
  l.dev = c.dev; l.sm_count = c.sm_count; l.stream = s;
  TcParams &p = l.p;
  p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.beta = beta;
  p.C = C; p.rsC = rsC; p.csC = csC; p.epi = epi;
  if (f16) { p.amax_a = f16->a; p.amax_b = f16->b; }
  if (bat) {
    l.batched = true;
    p.batch = static_cast<int>(bat->batch);
    p.period_a = static_cast<int>(period_a);
    p.period_b = static_cast<int>(period_b);
    p.bsC = bat->C;
    p.amax_bs_a = M;
    p.amax_bs_b = N;
    p.bias_bs = bat->bias;
  }
  const int npass = (kind == TC_TF32X3 || kind == TC_F16X3) ? 3 : 1;
  const TcPlanCfg cfg{c.kc_faithful, c.raster_g, c.splitk_enabled, c.sm_count};
  if (kind == TC_BF16 || kind == TC_F16X3) tc_plan<2, std::is_same<OutT, float>::value>(p, npass, cfg);
  else tc_plan<4, std::is_same<OutT, float>::value>(p, npass, cfg);
  if (c.dyn_sched) {
    p.sched = static_cast<unsigned int *>(c.sched.ptr) + 2 * c.sched_next;
    c.sched_next = (c.sched_next + 1) % kSchedSlots;
  }
  auto launch = [&](const TcLaunch &q) -> int {
    int e;
    switch (kind) {
      case TC_TF32X1: e = launch_tc_tf32x1(q); break;
      case TC_TF32X3: e = launch_tc_tf32x3(q); break;
      case TC_BF16: e = launch_tc_bf16(q); break;
      default: e = launch_tc_f16x3(q); break;
    }
    COUNT_LAUNCH();
    if (e != 0) {
      cudaGetLastError();
      return set_error(e == static_cast<int>(cudaErrorMemoryAllocation) ? LASER_B200_ENOMEM : LASER_B200_ECUDA,
                       "tensor-core kernel launch failed: %s", cudaGetErrorString(static_cast<cudaError_t>(e)));
    }
    CHECK_LAUNCH();
    return LASER_B200_OK;
  };
  ProfBracket prof;
  int rc = prof.open(c, s, 0);
  if (rc) return rc;
  if (p.k_splits > 1) {
    if constexpr (std::is_same<OutT, float>::value) {
      // units past the direct tiles write raw partial sums to tile-local planes of the workspace (tc_params.h); a second
      // kernel adds the planes of those tiles and applies alpha / beta / epilogue
      const int64_t ws_floats = tc_split_ws_floats(p);
      if ((rc = ensure(c.splitk, static_cast<size_t>(ws_floats) * sizeof(float)))) return rc;
      p.split_ws = static_cast<float *>(c.splitk.ptr);
      if ((rc = launch(l))) return rc;
      const int n_tail = p.num_m_blocks * p.num_n_blocks * p.batch - p.n_direct;
      const int64_t items = (static_cast<int64_t>(n_tail) * TC_BLOCK_M * (TC_BLOCK_N / 4) + 255) / 256;
      auto reduce = [&](auto batched) {
        splitk_tail_reduce_kernel<decltype(batched)::value><<<grid_for(c, items, 8), 256, 0, s>>>(
            static_cast<const float *>(c.splitk.ptr), p.k_splits, n_tail, p.n_direct, p.num_m_blocks, p.num_n_blocks, p.raster_g,
            M, N, alpha, beta, C, rsC, csC, p.epi.bias, p.epi.bias_per_row, p.epi.act, p.bsC, p.period_a, p.bias_bs);
      };
      if (bat) reduce(std::true_type());
      else reduce(std::false_type());
      COUNT_LAUNCH();
      CHECK_LAUNCH();
      CUDA_TRY(cudaEventRecord(c.ws_free, s));  // the planes are workspace too
      return prof.close();
    }
  }
  if ((rc = launch(l))) return rc;
  return prof.close();
}

// An operand -- with its op -- is the same in every problem of a batch: prepared once, read by every problem
inline bool batch_shares(int64_t stride, const OperandOp *op, int64_t aux_stride) {
  return stride == 0 && (!op || !op->aux || aux_stride == 0);
}

// SRC_ESZ: element size of the caller's operands (4: fp32 in any of the three tensor-core modes, 2: bf16)
template <int SRC_ESZ, typename OutT>
int gemm_tc(Ctx &c, TcKind kind, const Operand &oa, const Operand &ob, float alpha, float beta, OutT *C, int64_t rsC, int64_t csC,
            cudaStream_t s, const Epilogue &epi, cudaEvent_t b_ready = nullptr, const OperandOp *opA = nullptr,
            const OperandOp *opB = nullptr, const BatchArgs *bat = nullptr) {
  // oa / ob: A and B as built by run_f32 (bf16: single problems)
  // b_ready: B becomes valid only when this event has fired (the row-sharded driver: B is in flight on the communication
  // stream); everything that does not read B -- the preparation of A -- is queued before the wait.
  // opA / opB: operand ops applied while the operands are prepared (fp32 only)
  // bat: a batched launch, every problem's operand in the same launches; an operand of batch_of(o).n < bat->batch problems
  // repeats with that period.  Concatenated operands (Operand::concat): one product of extent batch * K (one problem for the
  // GEMM: rank-2 maps, one scale word per row of A and column of B).
  const int64_t M = oa.mn, N = ob.mn, K = oa.k;
  const bool cat = oa.concat;
  const int64_t Kt = cat ? batch_of(oa).n * K : K;   // (the entry bounds batch * K by INT64_MAX)
  if (M > 0x7fffffffLL || N > 0x7fffffffLL || Kt > 0x7fffffffLL)
    return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: extents must fit in int32");
  std::lock_guard<std::mutex> lk(c.mu);  // workspace + descriptor construction are per context
  const SplitMode mode = split_mode(kind);
  OperandMaps ma, mb;
  bool used_ws = false;
  // the previous call may still be reading the workspace on another stream
  CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
  ProfBracket prep;
  int rc = prep.open(c, s, 1);
  if (rc) return rc;
  int64_t f16_b_off = 0;
  if (mode == SPLIT_F16X2 &&
      (rc = f16_scales(c, (cat ? 1 : batch_of(oa).n) * M, (cat ? 1 : batch_of(ob).n) * N, &f16_b_off)))
    return rc;
  if ((rc = prepare_operand<SRC_ESZ>(c, oa, mode, ws_of_A(c), TC_BLOCK_M, &ma, &used_ws, s, opA))) return rc;
  if (b_ready) CUDA_TRY(cudaStreamWaitEvent(s, b_ready, 0));
  if ((rc = prepare_operand<SRC_ESZ>(c, ob, mode, ws_of_B(c, f16_b_off), TC_BLOCK_N, &mb, &used_ws, s, opB))) return rc;
  const int prep_launches = prep.launches();
  if ((rc = prep.close())) return rc;
  const F16Scales f16{static_cast<const uint32_t *>(c.f16s.ptr), static_cast<const uint32_t *>(c.f16s.ptr) + f16_b_off};
  // (with profiling on, an event record sits between the last preparation kernel and the GEMM: no dependent launch then)
  rc = tc_run<OutT>(c, kind, M, N, Kt, alpha, ma, mb, beta, C, rsC, csC, s, epi, mode == SPLIT_F16X2 ? &f16 : nullptr,
                    prep_launches > 0 && !c.profiling, bat, batch_of(oa).n, batch_of(ob).n);
  if (rc) return rc;
  if (used_ws) CUDA_TRY(cudaEventRecord(c.ws_free, s));
  return LASER_B200_OK;
}

// ---------------------------------------------------------------------------------------
//                      pre-packed operands (gemm_prepacked.nim:63-292)
// ---------------------------------------------------------------------------------------
// Layout of a packed operand seen as [mn][k] (A: mn = M, B: mn = N), a pure function of (mn, k):
//   [h : mn x ld_b fp16][l : mn x ld_b fp16][abs-max words : mn x u32], sections 256-byte aligned,
//   ld_b = round_up(k, 8): the compact K-major pieces of the default (F16X3) mode together with the
//   per-row scale words the epilogue needs -- a repeated product skips the whole preparation pass.
int finish(Ctx &c, cudaStream_t user, cudaStream_t s);

struct PackedLayout {
  int64_t ld_b;
  size_t off_h, off_l, off_amax, bytes;
};
inline PackedLayout packed_layout(int64_t mn, int64_t k) {
  PackedLayout L;
  L.ld_b = round_up(k, 8);
  auto al = [](size_t x) { return (x + 255) & ~static_cast<size_t>(255); };
  L.off_h = 0;
  L.off_l = al(static_cast<size_t>(mn) * L.ld_b * 2);
  L.off_amax = L.off_l + al(static_cast<size_t>(mn) * L.ld_b * 2);
  L.bytes = L.off_amax + al(static_cast<size_t>(mn) * sizeof(uint32_t));
  return L;
}

int prepack_dev(int which, void *dst, int64_t mn, int64_t k, const float *src, int64_t s_mn, int64_t s_k,
                void *stream) {
  if (mn < 0 || k < 0) return set_error(LASER_B200_EINVAL, "negative extent");
  if (mn == 0 || k == 0) return LASER_B200_OK;
  if (!dst || !src) return set_error(LASER_B200_EINVAL, "null pointer");
  if (reinterpret_cast<uintptr_t>(dst) & 255) return set_error(LASER_B200_EINVAL, "packed buffer must be 256-byte aligned");
  Ctx *c;
  int rc = get_ctx(&c);
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  const PackedLayout L = packed_layout(mn, k);
  uint8_t *base = static_cast<uint8_t *>(dst);
  uint16_t *h = reinterpret_cast<uint16_t *>(base + L.off_h), *l = reinterpret_cast<uint16_t *>(base + L.off_l);
  uint32_t *amax = reinterpret_cast<uint32_t *>(base + L.off_amax);
  {
    std::lock_guard<std::mutex> lk(c->mu);   // the gather buffer is workspace
    Operand o{src, mn, k, s_mn, s_k};
    const float *rows = src;
    int64_t rows_ld = s_mn;
    if (classify(o, 4) != K_MAJOR) {
      // anything that is not K-major already (MN-major, general strides) is gathered into compact K-major rows first
      CUDA_TRY(cudaStreamWaitEvent(s, c->ws_free, 0));
      Buffer &g = c->gather[which];
      if ((rc = gather<float>(*c, o, g, nullptr, s))) return rc;
      rows = static_cast<const float *>(g.ptr);
      rows_ld = round_up(k, 4);
    }
    if ((rc = f16x2_rows(*c, rows, mn, k, rows_ld, h, l, L.ld_b, amax, s))) return rc;
    CUDA_TRY(cudaEventRecord(c->ws_free, s));
  }
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

int packed_maps(Ctx &c, const void *packed, int64_t mn, int64_t k, int block_mn, OperandMaps *m, const uint32_t **amax) {
  const PackedLayout L = packed_layout(mn, k);
  const uint8_t *base = static_cast<const uint8_t *>(packed);
  int rc;
  m->mn_major = false;
  *amax = reinterpret_cast<const uint32_t *>(base + L.off_amax);
  if ((rc = operand_map(c, &m->p0, 2, base + L.off_h, K_MAJOR, mn, k, L.ld_b, block_mn))) return rc;
  return operand_map(c, &m->p1, 2, base + L.off_l, K_MAJOR, mn, k, L.ld_b, block_mn);
}

// A: either raw (A != nullptr) or packed (packedA != nullptr); B always packed
int gemm_packed_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA,
                    int64_t csA, const void *packedA, const void *packedB, float beta, float *C,
                    int64_t rsC, int64_t csC, void *stream) {
  if (M < 0 || N < 0 || K < 0) return set_error(LASER_B200_EINVAL, "negative extent");
  if (M == 0 || N == 0 || K == 0) return LASER_B200_OK;
  if ((!A && !packedA) || !packedB || !C) return set_error(LASER_B200_EINVAL, "null pointer");
  if (M > 0x7fffffffLL || N > 0x7fffffffLL || K > 0x7fffffffLL)
    return set_error(LASER_B200_EUNSUPPORTED, "extents must fit in int32");
  Ctx *cp;
  int rc = get_ctx(&cp);
  if (rc) return rc;
  Ctx &c = *cp;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c.stream;
  {
    std::lock_guard<std::mutex> lk(c.mu);
    OperandMaps ma, mb;
    F16Scales f16;
    bool used_ws = false;
    int prep_launches = 0;
    CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
    if (packedA) {
      if ((rc = packed_maps(c, packedA, M, K, TC_BLOCK_M, &ma, &f16.a))) return rc;
    } else {
      Operand oa{A, M, K, rsA, csA};
      int64_t b_off = 0;
      if ((rc = f16_scales(c, M, 0, &b_off))) return rc;
      ProfBracket prep;
      if ((rc = prep.open(c, s, 1))) return rc;
      if ((rc = prepare_operand<4>(c, oa, SPLIT_F16X2, ws_of_A(c), TC_BLOCK_M, &ma, &used_ws, s))) return rc;
      prep_launches = prep.launches();
      if ((rc = prep.close())) return rc;
      f16.a = static_cast<const uint32_t *>(c.f16s.ptr);
    }
    if ((rc = packed_maps(c, packedB, N, K, TC_BLOCK_N, &mb, &f16.b))) return rc;
    if ((rc = tc_run<float>(c, TC_F16X3, M, N, K, alpha, ma, mb, beta, C, rsC, csC, s, Epilogue(), &f16,
                            prep_launches > 0 && !c.profiling)))
      return rc;
    if (used_ws) CUDA_TRY(cudaEventRecord(c.ws_free, s));
  }
  g_last_path = LASER_B200_PATH_F16X3;
  return finish(c, static_cast<cudaStream_t>(stream), s);
}

// ---------------------------------------------------------------------------------------
//                                      dispatch
// ---------------------------------------------------------------------------------------
int check_args(int64_t M, int64_t N, int64_t K, const void *A, const void *B, const void *C) {
  if (M < 0 || N < 0 || K < 0) return set_error(LASER_B200_EINVAL, "negative extent M=%lld N=%lld K=%lld",
                                                (long long)M, (long long)N, (long long)K);
  if (M == 0 || N == 0 || K == 0) return -1;  // nothing to do (gemm.nim:150: C untouched)
  if (!A || !B || !C) return set_error(LASER_B200_EINVAL, "null matrix pointer");
  return LASER_B200_OK;
}

int finish(Ctx &, cudaStream_t user, cudaStream_t s) {
  if (!user) CUDA_TRY(cudaStreamSynchronize(s));
  return LASER_B200_OK;
}

inline bool is_tc_mode(int mode) {
  return mode == LASER_B200_PATH_F16X3 || mode == LASER_B200_PATH_TF32X3 || mode == LASER_B200_PATH_TF32X1;
}
// What PATH_AUTO resolves to -- ONE predicate for the device-pointer and the host-pointer entry points:
//   work <= 128^3 (the reference's own switch, gemm.nim:140-141): exact kernel -- a 128 x 256 tensor-core tile would be
//       mostly padding;
//   mode SIMT: exact kernel for every shape (the mode documented as bit-identical to the CPU reference), before any shortcut;
//   N <= 4 tall problems without a fused epilogue or operand op: warp-shuffle GEMV (-1);
//   otherwise the fp32 mode in force.
int resolve_auto(int64_t M, int64_t N, int64_t K, const Epilogue &epi, bool operand_op = false) {
  const double work = static_cast<double>(M) * N * K;
  if (work <= 128.0 * 128.0 * 128.0) return LASER_B200_PATH_SIMT;
  const int mode = g_f32_mode.load();
  if (mode == LASER_B200_PATH_SIMT) return LASER_B200_PATH_SIMT;
  if (N <= 4 && M >= 1024 && !epi.bias && !epi.act && !operand_op) return -1;
  // few output rows, wide N (the im2col convolution's product): the exact few-rows kernel streams B once; a tensor-core
  // call would first spend three passes over B preparing it and then compute 84+ % padding (20 x 788544 x 27: 0.08 ms
  // against 0.28 ms, profiles/r02_large_shapes.txt) -- and exact is at least as accurate as any tensor-core mode
  if (M <= 32 && N >= 1024) return LASER_B200_PATH_SIMT;
  return mode < 0 ? kDefaultF32Mode : mode;
}

// the paths of the fp32 entries: PATH_AUTO, the exact kernel or a tensor-core mode
int check_f32_path(int path) {
  if (path == LASER_B200_PATH_AUTO || path == LASER_B200_PATH_SIMT || is_tc_mode(path)) return LASER_B200_OK;
  return set_error(LASER_B200_EINVAL, "unknown path %d for float32", path);
}

// The exact path: each operand with an op, concatenated or an im2col source is written once into compact K-major rows of
// the gather workspace (f32_rows, op applied), each other one is read in place; then one exact-kernel launch over the batch
// (`batch` problems, C bsC apart), so the path stays bit-identical to the CPU reference on the operands as prepared.
int simt_run(Ctx &c, const Operand &oa, const Operand &ob, float alpha, float beta, float *C, int64_t rsC, int64_t csC,
             cudaStream_t s, const Epilogue &epi, const OperandOp *opA, const OperandOp *opB, int64_t batch, int64_t bsC) {
  struct Rows {
    const float *p;
    int64_t s_mn, s_k, s_b;
  };
  const bool copy_a = opA || oa.concat || oa.conv, copy_b = opB || ob.concat || ob.conv;
  std::unique_lock<std::mutex> lk(c.mu, std::defer_lock);   // the gather buffers are workspace
  if (copy_a || copy_b) {
    lk.lock();
    CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
  }
  auto rows = [&](const Operand &o, const OperandOp *op, bool copy, Buffer &g, Rows *r) {
    *r = Rows{static_cast<const float *>(o.ptr), o.s_mn, o.s_k, o.s_b};
    if (!copy) return LASER_B200_OK;
    const int rc = f32_rows(c, o, SPLIT_NONE, g, nullptr, s, op);
    const int64_t ld = round_up(o.concat ? batch_of(o).n * o.k : o.k, 4);
    *r = Rows{static_cast<const float *>(g.ptr), ld, 1, !o.concat && !batch_shares(o.s_b, op, o.aux_sb) ? o.mn * ld : 0};
    return rc;
  };
  Rows a, b;
  int rc;
  if ((rc = rows(oa, opA, copy_a, c.gather[0], &a))) return rc;
  if ((rc = rows(ob, opB, copy_b, c.gather[1], &b))) return rc;
  const int64_t K = oa.concat ? batch_of(oa).n * oa.k : oa.k;
  if ((rc = gemm_simt<float>(c, oa.mn, ob.mn, K, alpha, a.p, a.s_mn, a.s_k, b.p, b.s_k, b.s_mn, beta, C, rsC, csC, s, epi, batch,
                             a.s_b, b.s_b, bsC)))
    return rc;
  if (copy_a || copy_b) CUDA_TRY(cudaEventRecord(c.ws_free, s));
  return LASER_B200_OK;
}

// One fp32 product on a resolved path, the exact kernel or the tensor cores.  Its operands as [mn][k] (B: [n][k]):
//   batch > 0: a batched call, operand X of problem b at X + b * bs->X and the aux of its op bs->auxX apart; an operand the
//     batch shares, op included, is one problem, prepared once.  The problems' C bs->C apart.
//   concat: the sum of the batch's products into one C, one product over the operands concatenated along k
//     (Operand::concat; bs->C unused).
//   convB: B is an im2col source, the images at B bs->B floats apart (rsB, csB unused).  A channels-last one as tap rows
//     (ConvGeom::taps): N = the taps, K = images * outH * outW pixels of the images at B (a single problem).
//   convA: A is a channels-last im2col source (ConvGeom::nhwc), M = images * outH * outW rows of the images at A (rsA, csA
//     unused; a single problem).
//   periodA > 0 (batched, tensor cores): A is periodA problems bs->A apart and problem b reads A_{b % periodA} -- the filters of
//     a grouped convolution --, a per-row bias periodA blocks of M, problem b reading block b % periodA.
int run_f32(Ctx &c, int path, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA, const float *B,
            int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC, cudaStream_t s, const Epilogue &epi,
            const OperandOp *opA, const OperandOp *opB, int64_t batch = 0, const laser_b200_batch_strides *bs = nullptr,
            bool concat = false, const ConvGeom *convB = nullptr, cudaEvent_t b_ready = nullptr, const ConvGeom *convA = nullptr,
            int64_t periodA = 0) {
  Operand oa{A, M, K, rsA, csA}, ob{B, N, K, csB, rsB};
  if (batch > 0) {
    oa.batch = periodA > 0 ? periodA : !concat && batch_shares(bs->A, opA, bs->auxA) ? 1 : batch; oa.s_b = bs->A; oa.aux_sb = bs->auxA; oa.concat = concat;
    ob.batch = !concat && batch_shares(bs->B, opB, bs->auxB) ? 1 : batch; ob.s_b = bs->B; ob.aux_sb = bs->auxB; ob.concat = concat;
  }
  oa.conv = convA;
  ob.conv = convB;
  const bool batched = batch > 0 && !concat;
  if (periodA > 0 && (!batched || opA || path == LASER_B200_PATH_SIMT))
    return set_error(LASER_B200_ECUDA, "internal: a periodic A is a batched tensor-core operand without op");
  if (path == LASER_B200_PATH_SIMT)
    return simt_run(c, oa, ob, alpha, beta, C, rsC, csC, s, epi, opA, opB, batched ? batch : 1, batched ? bs->C : 0);
  const BatchArgs bat{batch, batched ? bs->C : 0, periodA > 0 ? M : 0};
  return gemm_tc<4, float>(c, tc_kind_of_path(path), oa, ob, alpha, beta, C, rsC, csC, s, epi, b_ready, opA, opB,
                           batched ? &bat : nullptr);
}

// opA / opB: operand ops of the fused-prologue entry (nullptr: none)
int f32_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
            const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
            int path, void *stream, const Epilogue &epi = Epilogue(), cudaEvent_t b_ready = nullptr,
            const OperandOp *opA = nullptr, const OperandOp *opB = nullptr) {
  int rc = check_args(M, N, K, A, B, C);
  if (rc == -1) return LASER_B200_OK;
  if (rc) return rc;
  const bool has_op = opA || opB;
  if ((has_op || path != -1) && (rc = check_f32_path(path))) return rc;   // (-1: the GEMV, for calls without an op)
  Ctx *c;
  rc = get_ctx(&c);
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_AUTO) path = resolve_auto(M, N, K, epi, has_op);
  if (b_ready && !is_tc_mode(path)) CUDA_TRY(cudaStreamWaitEvent(s, b_ready, 0));   // no separate preparation of A to overlap
  switch (path) {
    case -1: {
      const int grid = grid_for(*c, (M + 7) / 8, 8);
      const bool vec = (csA == 1) && (rsA % 4 == 0) && (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
      const size_t bsmem = static_cast<size_t>(N) * K * sizeof(float);
      const bool use_smem = vec && bsmem <= 96 * 1024;
#define LB200_GEMV(NV)                                                                                         \
  do {                                                                                                         \
    if (use_smem) {                                                                                            \
      static std::atomic<uint32_t> attr_set{0};                                                                \
      if (!(attr_set.load(std::memory_order_acquire) & (1u << c->dev))) {                                      \
        CUDA_TRY(cudaFuncSetAttribute(gemv_warp_smem_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)); \
        attr_set.fetch_or(1u << c->dev, std::memory_order_release);                                            \
      }                                                                                                        \
      gemv_warp_smem_kernel<NV><<<grid_for(*c, (M + 7) / 8, 2), 256, bsmem, s>>>(M, K, alpha, A, rsA, B, rsB, csB, beta, C, rsC, csC); \
    } else if (vec) gemv_warp_kernel<NV, true><<<grid, 256, 0, s>>>(M, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);  \
    else gemv_warp_kernel<NV, false><<<grid, 256, 0, s>>>(M, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC);     \
  } while (0)
      if (N == 1) LB200_GEMV(1); else if (N == 2) LB200_GEMV(2); else if (N == 3) LB200_GEMV(3); else LB200_GEMV(4);
#undef LB200_GEMV
      COUNT_LAUNCH();
      CHECK_LAUNCH();
      g_last_path = LASER_B200_PATH_SIMT;
      break;
    }
    default:
      // SIMT: the exact kernel.  F16X3 (default): two fp16 pieces of each operand scaled by a power of two per row of A /
      // column of B (device-side abs-max), three passes, the epilogue undoes the scales.  TF32X3: hi/lo tf32 pieces, three
      // passes.  TF32X1: one pass.
      rc = run_f32(*c, path, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, opA, opB, 0, nullptr, false,
                   nullptr, b_ready);
      if (rc) return rc;
      g_last_path = path;
      break;
  }
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

template <typename T>
int simt_dev(int64_t M, int64_t N, int64_t K, T alpha, const T *A, int64_t rsA, int64_t csA,
             const T *B, int64_t rsB, int64_t csB, T beta, T *C, int64_t rsC, int64_t csC,
             void *stream) {
  int rc = check_args(M, N, K, A, B, C);
  if (rc == -1) return LASER_B200_OK;
  if (rc) return rc;
  Ctx *c;
  rc = get_ctx(&c);
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  rc = gemm_simt<T>(*c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s);
  if (rc) return rc;
  g_last_path = LASER_B200_PATH_SIMT;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

int bf16_dev(int64_t M, int64_t N, int64_t K, float alpha, const uint16_t *A, int64_t rsA,
             int64_t csA, const uint16_t *B, int64_t rsB, int64_t csB, float beta, uint16_t *C,
             int64_t rsC, int64_t csC, void *stream) {
  int rc = check_args(M, N, K, A, B, C);
  if (rc == -1) return LASER_B200_OK;
  if (rc) return rc;
  Ctx *c;
  rc = get_ctx(&c);
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  rc = gemm_tc<2, uint16_t>(*c, TC_BF16, Operand{A, M, K, rsA, csA}, Operand{B, N, K, csB, rsB}, alpha, beta, C, rsC, csC, s,
                            Epilogue());
  if (rc) return rc;
  g_last_path = LASER_B200_PATH_BF16;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// arguments of the fused entries -> their internal form; nothing is launched before both are validated
int epilogue_of(const laser_b200_epilogue *epi, Epilogue *e) {
  if (!epi) return LASER_B200_OK;
  if (epi->activation < 0 || epi->activation > 3) return set_error(LASER_B200_EINVAL, "unknown activation %d", epi->activation);
  e->bias = epi->bias;
  e->bias_per_row = epi->bias_per_row ? 1 : 0;
  e->act = epi->activation;
  return LASER_B200_OK;
}
// *out = nullptr for no op; aux strides become [mn][k] ones (B is seen as [n][k])
int operand_op_of(const laser_b200_operand_op *in, bool is_b, OperandOp *op, const OperandOp **out) {
  *out = nullptr;
  if (!in || in->op == LASER_B200_OP_NONE) return LASER_B200_OK;
  if (in->op < LASER_B200_OP_NONE || in->op > LASER_B200_OP_SIGMOID_GRAD)
    return set_error(LASER_B200_EINVAL, "unknown operand op %d", in->op);
  const bool derivative = in->op >= LASER_B200_OP_RELU_GRAD;
  if (derivative && !in->aux) return set_error(LASER_B200_EINVAL, "operand op %d needs an aux tensor", in->op);
  op->op = in->op;
  op->aux = derivative ? in->aux : nullptr;
  op->aux_sr = is_b ? in->auxColStride : in->auxRowStride;
  op->aux_sc = is_b ? in->auxRowStride : in->auxColStride;
  *out = op;
  return LASER_B200_OK;
}
// epilogue and operand ops of a fused GEMM entry, all checked before anything is launched (opA / opB: nullptr, or they point
// into a / b -- a FusedArgs is used where it was decoded, never copied)
struct FusedArgs {
  Epilogue epi;
  OperandOp a, b;
  const OperandOp *opA = nullptr, *opB = nullptr;
};
int fused_args_of(const laser_b200_epilogue *epi, const laser_b200_operand_op *opA, const laser_b200_operand_op *opB, FusedArgs *f) {
  int rc;
  if ((rc = epilogue_of(epi, &f->epi))) return rc;
  if ((rc = operand_op_of(opA, false, &f->a, &f->opA))) return rc;
  return operand_op_of(opB, true, &f->b, &f->opB);
}

// ---------------------------------------------------------------------------------------
//              batched fused product: the problems of a batch in one GEMM launch
// ---------------------------------------------------------------------------------------
// workspace one problem of a batched call prepares on `path` (bytes, an upper bound): the pieces, gather copy and scale words
// of each operand the problems do not share
int64_t batch_ws_per_problem(int path, int64_t M, int64_t N, int64_t K, bool a_own, bool b_own, bool opA, bool opB) {
  auto one = [&](int64_t mn, bool has_op) -> int64_t {
    const int64_t g = mn * round_up(K, 4) * 4;   // a compact fp32 copy, or one tf32 piece
    if (path == LASER_B200_PATH_F16X3) return 2 * mn * round_up(K, 8) * 2 + g + mn * 4;
    if (path == LASER_B200_PATH_TF32X3) return 2 * g;
    if (path == LASER_B200_PATH_TF32X1) return g;
    return has_op ? g : 0;   // exact path: the op'd operand
  };
  return (a_own ? one(M, opA) : 0) + (b_own ? one(N, opB) : 0);
}

// convB: B is an im2col source (a convolution, run_f32): even one image takes the batched launch.  periodA > 0: A and a
// per-row bias repeat with that period (run_f32), every chunk a whole number of periods.
int batched_fused_dev(int64_t batch, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
                      const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                      const laser_b200_batch_strides *bs, const OperandOp *opA, const OperandOp *opB, const Epilogue &epi,
                      int path, void *stream, const ConvGeom *convB = nullptr, int64_t periodA = 0) {
  if (batch < 0) return set_error(LASER_B200_EINVAL, "negative batch %lld", (long long)batch);
  if (batch > 0 && !bs) return set_error(LASER_B200_EINVAL, "batchStrides is NULL");
  if (batch > 1 && bs->C == 0) return set_error(LASER_B200_EINVAL, "batchStrides->C is 0: the problems' outputs would overlap");
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  rc = check_args(M, N, K, A, B, C);
  if (rc == -1 || batch == 0) return LASER_B200_OK;
  if (rc) return rc;
  if (batch == 1 && !convB)
    return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, epi, nullptr, opA, opB);
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_AUTO) path = resolve_auto(M, N, K, epi, /*operand_op=*/true);
  // chunks of whole problems: the prepared workspace stays under the cap, and the launch's tile counts -- batch x tiles x
  // up to 16 K-splits -- fit in int32 (an im2col source counts as an op'd B: the exact path writes its rows)
  // (a periodic A is prepared once, its periodA slices are not workspace per problem)
  const int64_t per = batch_ws_per_problem(path, M, N, K, periodA == 0 && !batch_shares(bs->A, opA, bs->auxA),
                                           !batch_shares(bs->B, opB, bs->auxB), opA != nullptr, opB != nullptr || convB);
  int64_t chunk = per > 0 ? c->batch_ws_bytes / per : batch;
  const int64_t tiles = ((M + TC_BLOCK_M - 1) / TC_BLOCK_M) * ((N + TC_BLOCK_N - 1) / TC_BLOCK_N);
  if (chunk > 0x7fffffffLL / (16 * tiles)) chunk = 0x7fffffffLL / (16 * tiles);
  if (periodA > 0) {
    if (periodA > 0x7fffffffLL / (16 * tiles))
      return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: %lld problems of %lld tiles do not fit in int32",
                       (long long)periodA, (long long)tiles);
    chunk -= chunk % periodA;
    if (chunk < periodA) chunk = periodA;
  }
  if (chunk < 1) chunk = 1;
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    OperandOp ca, cb;
    if (opA) { ca = *opA; if (ca.aux) ca.aux += b0 * bs->auxA; }
    if (opB) { cb = *opB; if (cb.aux) cb.aux += b0 * bs->auxB; }
    // (a chunk of a periodic batch starts at a whole period: problem b0 reads A's first slice)
    if ((rc = run_f32(*c, path, M, N, K, alpha, periodA > 0 ? A : A + b0 * bs->A, rsA, csA, B + b0 * bs->B, rsB, csB, beta,
                      C + b0 * bs->C, rsC, csC, s, epi, opA ? &ca : nullptr, opB ? &cb : nullptr, batch - b0 < chunk ? batch - b0 : chunk,
                      bs, false, convB, nullptr, nullptr, periodA)))
      return rc;
  }
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}
// laser_b200_gemm_strided_batched_f32_fused_dev (defined with the other batched entries in capi_layers.inc)
int batched_fused_entry(int64_t batch, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
                        const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                        const laser_b200_batch_strides *bs, const laser_b200_operand_op *opA, const laser_b200_operand_op *opB,
                        const laser_b200_epilogue *epi, int path, void *stream) {
  FusedArgs f;
  const int rc = fused_args_of(epi, opA, opB, &f);
  if (rc) return rc;
  return batched_fused_dev(batch, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, bs, f.opA, f.opB, f.epi, path, stream);
}

// ---------------------------------------------------------------------------------------
//   batch-reduced fused product: the sum of a batch's products, one product over the operands concatenated along k
// ---------------------------------------------------------------------------------------
// laser_b200_gemm_strided_batch_reduce_f32_fused_dev: C <- act(alpha * sum_b opA(A_b) * opB(B_b) + beta * C + bias), the fused
// call over A^ = [opA(A_0) | .. | opA(A_{n-1})] (M x nK) and B^ = [opB(B_0); ..; opB(B_{n-1})] (nK x N).  One chunk always:
// chunking a sum would round C between chunks and apply the activation too early.  convB: B is a concatenated im2col source
// (a convolution's filter gradient, run_f32): even one image takes the concatenated preparation.
int batch_reduce_dev(int64_t batch, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
                     const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                     const laser_b200_batch_strides *bs, const OperandOp *opA, const OperandOp *opB, const Epilogue &epi, int path,
                     void *stream, const ConvGeom *convB = nullptr) {
  if (batch < 0) return set_error(LASER_B200_EINVAL, "negative batch %lld", (long long)batch);
  if (batch > 0 && !bs) return set_error(LASER_B200_EINVAL, "batchStrides is NULL");
  if (batch > 0 && bs->C != 0)
    return set_error(LASER_B200_EINVAL, "batchStrides->C is %lld: the batch sums into one C", (long long)bs->C);
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  rc = check_args(M, N, K, A, B, C);
  if (rc == -1 || batch == 0) return LASER_B200_OK;
  if (rc) return rc;
  if (batch == 1 && !convB)
    return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, epi, nullptr, opA, opB);
  if (K > INT64_MAX / batch) return set_error(LASER_B200_EUNSUPPORTED, "batch * K overflows int64");
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_AUTO) path = resolve_auto(M, N, batch * K, epi, /*operand_op=*/true);
  if ((rc = run_f32(*c, path, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, opA, opB, batch, bs, true, convB)))
    return rc;
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// ---------------------------------------------------------------------------------------
//     fused convolution: im2col folded into the preparation of B, the images of a chunk in one GEMM launch
// ---------------------------------------------------------------------------------------
// The product of both fused convolution entries, image by image: output_n = epi(alpha * A * B_n + beta * output_n), A [Cout][K]
// (rsA, csA; K-major with 16-byte rows unless the kernel is 1 x 1), shared by the images; B_n image n of `input` as an im2col
// source of geometry g (dilated: ConvGeom::dH, dW), opB applied to its values (aux dense like `input`).  The batched fused
// product over the images, in its chunks of whole images under LASER_B200_BATCH_WS_MB: the images do not sum into each other.
// PATH_AUTO of a convolution of geometry g, in either layout: as conv2d_im2col_f32_dev decides, the exact kernel for a batch of
// short M = c_out or K (batched_f32_dev), else resolve_auto over one NCHW image's product with this call's epilogue (never
// the GEMV: N is a pixel count and the batch needs one launch)
int conv_auto_path(const ConvGeom &g, const Epilogue &epi) {
  const int64_t M = g.Cout, K = g.K();
  return (g.B > 1 && (M < 64 || K < 64)) ? LASER_B200_PATH_SIMT : resolve_auto(M, g.outHW(), K, epi, /*operand_op=*/true);
}

int conv_windows_dev(const ConvGeom &g, float alpha, const float *A, int64_t rsA, int64_t csA, const float *input, float beta,
                     float *output, const OperandOp *opB, const Epilogue &epi, int path, void *stream) {
  const int64_t M = g.Cout, K = g.K(), N = g.outHW(), image = g.C * g.H * g.W;
  if (path == LASER_B200_PATH_AUTO) path = conv_auto_path(g, epi);
  // a 1 x 1 kernel with unit strides, no padding and no dilation: the image already is B_n, the [C][H*W] matrix
  const bool in_place = g.kH * g.kW == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0 && g.dH == 1 && g.dW == 1;
  const laser_b200_batch_strides bs{0, image, M * N, 0, image};
  return batched_fused_dev(g.B, M, N, K, alpha, A, rsA, csA, input, N, 1, beta, output, N, 1, &bs, nullptr, opB, epi, path, stream,
                           in_place ? nullptr : &g);
}

// laser_b200_conv2d_f32_fused_dev (capi_layers.inc checks the geometry): output_n = act(F * im2col(input_n) + bias) for every
// image n.  A = the filters F [Cout][K], shared by the images (prepared once per launch); B = the images as an im2col source.
int conv2d_fused_dev(float *output, const float *input, const ConvGeom &g, const float *kernel, const laser_b200_epilogue *epi_in,
                     int path, void *stream) {
  Epilogue epi;
  int rc;
  if ((rc = epilogue_of(epi_in, &epi))) return rc;
  if ((rc = check_f32_path(path))) return rc;
  if (g.B == 0) return LASER_B200_OK;
  if (!output || !input || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  return conv_windows_dev(g, 1.0f, kernel, g.K(), 1, input, 0.0f, output, nullptr, epi, path, stream);
}

// laser_b200_conv2d_grouped_f32_fused_dev (capi_layers.inc checks the geometry and the groups; groups == 1 never comes here):
// G groups of Cg = C / G input and Mg = Cout / G output channels.  Per group, the per-group geometry gp -- n * G images of Cg
// channels, Cout = Mg -- is a batch of convolutions whose problem b = i * G + g reads image i's channel slice of group g (one
// image of gp, the NCHW slices are Cg * H * W apart), writes output channels g * Mg .. (one output image of gp) and reads the
// filters and bias of group b % G.
//   PATH_AUTO: conv_auto_path over gp.  The exact path is the direct kernel (gemm_simt.cuh: conv_grouped_direct_kernel), one launch; the tensor-core
//   paths are the batched fused product over gp with A = the filters as G problems of Mg x Kg, periodic with period G
//   (batched_fused_dev), in chunks of whole images.
int conv2d_grouped_fused_dev(float *output, const float *input, const ConvGeom &g, int64_t groups, const float *kernel,
                             const laser_b200_epilogue *epi_in, int path, void *stream) {
  Epilogue epi;
  int rc;
  if ((rc = epilogue_of(epi_in, &epi))) return rc;
  if ((rc = check_f32_path(path))) return rc;
  if (epi.bias && !epi.bias_per_row)
    return set_error(LASER_B200_EINVAL, "a convolution's bias is one per output channel: bias_per_row must be 1");
  if (g.B == 0) return LASER_B200_OK;
  if (!output || !input || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  ConvGeom gp = g;
  gp.B = g.B * groups;
  gp.C = g.C / groups;
  gp.Cout = g.Cout / groups;
  if (path == LASER_B200_PATH_AUTO) path = conv_auto_path(gp, epi);
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_SIMT) {
    ConvGroupedParams p;
    int mc;
    size_t smem;
    const int threads = conv_grouped_plan(g, groups, epi.bias, epi.act, &p, &mc, &smem);
    if (threads == 0)
      return set_error(LASER_B200_EUNSUPPORTED, "grouped convolution: a %lld x %lld kernel window does not fit in shared memory",
                       (long long)g.kH, (long long)g.kW);
    const int grid = grid_for(*c, p.tiles, 2048 / threads);
    if (mc == 4) conv_grouped_direct_kernel<4><<<grid, threads, smem, s>>>(output, input, kernel, p);
    else if (mc == 2) conv_grouped_direct_kernel<2><<<grid, threads, smem, s>>>(output, input, kernel, p);
    else conv_grouped_direct_kernel<1><<<grid, threads, smem, s>>>(output, input, kernel, p);
    COUNT_LAUNCH();
    CHECK_LAUNCH();
  } else {
    const int64_t M = gp.Cout, K = gp.K(), N = gp.outHW(), image = gp.C * gp.H * gp.W;
    const bool in_place = g.kH * g.kW == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0;
    const laser_b200_batch_strides bs{M * K, image, M * N, 0, 0};
    if ((rc = batched_fused_dev(gp.B, M, N, K, 1.0f, kernel, K, 1, input, N, 1, 0.0f, output, N, 1, &bs, nullptr, nullptr, epi, path,
                                s, in_place ? nullptr : &gp, groups)))
      return rc;
  }
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// The product of both channels-last convolution entries, over the NHWC images `src` (a geometry with nhwc set) at A:
//   C[n * P + p][j] <- epi(alpha * sum_k A(n * P + p, k) * B[k][j] + beta * C[n * P + p][j]),  P = src.outHW(), K = src.K()
// A the images' windows (split.cuh: Im2colNhwcSrc, dilated or op'd Im2colNhwcGradSrc), or with in_place the images themselves
// read as [n * P][K]; opA applied to the values read, its aux laid out like the images.  B [K][N] through (rsB, csB); C dense
// [n * P][N].  Chunks of whole images under LASER_B200_BATCH_WS_MB, the tile count of each in int32, one preparation and one
// GEMM launch sequence each; the images do not sum into each other, so chunks give the bits of one.
int conv_nhwc_chunks(Ctx &c, int path, const ConvGeom &src, int64_t N, float alpha, const float *A, const float *B, int64_t rsB,
                     int64_t csB, float beta, float *C, cudaStream_t s, const Epilogue &epi, const OperandOp *opA, bool in_place) {
  const int64_t K = src.K(), P = src.outHW(), image = src.H * src.W * src.C;
  const int64_t per = batch_ws_per_problem(path, P, N, K, true, false, !in_place || opA, false);
  int64_t chunk = per > 0 ? c.batch_ws_bytes / per : src.B;
  const int64_t max_m_blocks = 0x7fffffffLL / (16 * ((N + TC_BLOCK_N - 1) / TC_BLOCK_N));
  if (chunk > max_m_blocks * TC_BLOCK_M / P) chunk = max_m_blocks * TC_BLOCK_M / P;
  if (chunk < 1) chunk = 1;
  ConvGeom gc = src;
  int rc;
  for (int64_t b0 = 0; b0 < src.B; b0 += chunk) {
    const int64_t imgs = src.B - b0 < chunk ? src.B - b0 : chunk;
    gc.B = imgs;
    OperandOp ca;
    if (opA) { ca = *opA; if (ca.aux) ca.aux += b0 * image; }
    if ((rc = run_f32(c, path, imgs * P, N, K, alpha, A + b0 * image, src.C, 1, B, rsB, csB, beta, C + b0 * P * N, N, 1, s, epi,
                      opA ? &ca : nullptr, nullptr, 0, nullptr, false, nullptr, nullptr, in_place ? nullptr : &gc)))
      return rc;
  }
  return LASER_B200_OK;
}

// laser_b200_conv2d_nhwc_f32_fused_dev (capi_layers.inc checks the geometry): NHWC images, one product for the images of a chunk,
//   output[n * P + p][co] = act(sum_k rows[n * P + p][k] * Wmat[k][co] + bias[co]),  P = outH * outW
// A = the images as a channels-last im2col source (one row per output pixel, K-major), B = the filter matrix [K][c_out] read
// with its strides (kernelStrides[0] over k, [1] over co), C = the NHWC output, the bias one per column.  1 x 1 kernels with unit strides
// and no padding: A is the images read in place as [n * H * W][C].  Chunks of whole images (conv_nhwc_chunks).
int conv2d_nhwc_fused_dev(float *output, const float *input, const ConvGeom &g, const float *kernel, const int64_t kernelStrides[2],
                          const laser_b200_epilogue *epi_in, int path, void *stream) {
  Epilogue epi;
  int rc;
  if ((rc = epilogue_of(epi_in, &epi))) return rc;
  if ((rc = check_f32_path(path))) return rc;
  if (!kernelStrides) return set_error(LASER_B200_EINVAL, "kernelStrides is NULL");
  if (epi.bias && !epi.bias_per_row)
    return set_error(LASER_B200_EINVAL, "a convolution's bias is one per output channel: bias_per_row must be 1");
  if (g.B == 0) return LASER_B200_OK;
  if (!output || !input || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  if (path == LASER_B200_PATH_AUTO) path = conv_auto_path(g, epi);
  if (is_tc_mode(path) && g.outHW() > 0x7fffffffLL / g.B)
    return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: images * outH * outW must fit in int32");
  epi.bias_per_row = 0;   // the output channels are the columns of C
  const bool in_place = g.kH * g.kW == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0;
  ConvGeom gn = g;
  gn.nhwc = true;
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if ((rc = conv_nhwc_chunks(*c, path, gn, g.Cout, 1.0f, input, kernel, kernelStrides[0], kernelStrides[1], 0.0f, output, s, epi,
                             nullptr, in_place)))
    return rc;
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

template <typename T>
int launch_copy(Ctx &c, void *dst, const void *src, const CopyParams &p, cudaStream_t s);   // capi_layers.inc

// ---------------------------------------------------------------------------------------
//   convolution input gradient: the forward product over the output gradients as a transposed, dilated im2col source
// ---------------------------------------------------------------------------------------
// The transposed geometry of the input gradients: the output gradients (Cout channels of outH x outW) as the source, zero-dilated
// by the forward strides and padded by kH - 1 - pH, stride 1, windows at the input's H x W pixels and C output channels
ConvGeom transposed_geom(const ConvGeom &g) {
  ConvGeom gt = g;
  gt.C = g.Cout; gt.H = g.outH; gt.W = g.outW; gt.Cout = g.C;
  gt.pH = g.kH - 1 - g.pH; gt.pW = g.kW - 1 - g.pW;
  gt.sH = gt.sW = 1;
  gt.dH = g.sH; gt.dW = g.sW;
  gt.outH = g.H; gt.outW = g.W;
  return gt;
}

// laser_b200_conv2d_input_grad_f32_fused_dev (capi_layers.inc checks the geometry):
//   grad_input_n <- alpha * W' * B_n + beta * grad_input_n,  W'[ci][(co, kh', kw')] = W[co][ci][kH-1-kh'][kW-1-kw']
// B_n: grad_output_n (op applied) as the im2col source of the transposed geometry gt -- C = Cout, H x W = outH x outW,
// padding kH - 1 - pH, stride 1, dilated by the forward strides, windows at the input's H x W pixels (split.cuh:
// Im2colGradSrc).  M = C, N = H * W, K' = Cout * kH * kW; conv_windows_dev runs it as it runs the forward call.
int conv2d_input_grad_dev(float *grad_input, const ConvGeom &g, const float *grad_output, const float *kernel, float alpha, float beta,
                          const laser_b200_operand_op *op_in, int path, void *stream) {
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  OperandOp op;
  const OperandOp *opB;
  if ((rc = operand_op_of(op_in, true, &op, &opB))) return rc;
  const int64_t P = g.outHW(), khw = g.kH * g.kW;
  // (B seen as [mn = pixel][k = channel]: a dense NCHW aux has aux_sr = 1, aux_sc = outH * outW)
  if (opB && opB->aux && (opB->aux_sr != 1 || opB->aux_sc != P))
    return set_error(LASER_B200_EINVAL, "the aux tensor of op %d must be dense like grad_output: strides (%lld, 1), not (%lld, %lld)",
                     opB->op, (long long)P, (long long)opB->aux_sc, (long long)opB->aux_sr);
  if (g.B == 0) return LASER_B200_OK;
  if (!grad_input || !grad_output || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  if (g.Cout > INT32_MAX / khw) return set_error(LASER_B200_EUNSUPPORTED, "c_out * kH * kW beyond 2^31");
  ConvGeom gt = transposed_geom(g);
  const int64_t K = gt.K();
  // dX_n = W^T * dY_n for a 1 x 1 kernel with unit strides and no padding: W read transposed, no copy
  if (khw == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0)
    return conv_windows_dev(gt, alpha, kernel, 1, g.C, grad_output, beta, grad_input, opB, Epilogue(), path, stream);
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  // W' once per call into library workspace, K-major rows 16 bytes apart, read in place by every chunk's product.  The buffer
  // (tfilt, shared with the channels-last input gradient) is held for the whole call; the copy waits for the last kernel that
  // read it (ws_free).
  std::lock_guard<std::mutex> lk(c->tfilt_mu);
  const int64_t lda = round_up(K, 4);
  if ((rc = ensure(c->tfilt, static_cast<size_t>(g.C * lda) * sizeof(float)))) return rc;
  CUDA_TRY(cudaStreamWaitEvent(s, c->ws_free, 0));
  const int64_t shape[4] = {g.C, g.Cout, g.kH, g.kW}, dst_st[4] = {lda, khw, g.kW, 1}, src_st[4] = {khw, g.C * khw, -g.kW, -1};
  CopyParams cp;
  copy_plan(4, shape, dst_st, src_st, &cp);
  float *wt = static_cast<float *>(c->tfilt.ptr);
  if ((rc = launch_copy<uint32_t>(*c, wt, kernel + khw - 1, cp, s))) return rc;
  return conv_windows_dev(gt, alpha, wt, lda, 1, grad_output, beta, grad_input, opB, Epilogue(), path, stream);
}

// laser_b200_conv2d_grouped_input_grad_f32_fused_dev (capi_layers.inc checks the geometry and the groups; groups == 1 never
// comes here): conv2d_input_grad_dev per group, G groups of Cg = C / G input and Mg = Cout / G output channels, T = kH * kW,
// K' = Mg * T.  gt is the transposed geometry of the whole layer (Cout source channels, C output channels), gtp that of one
// group -- n * G images of Mg channels, Cout = Cg --: problem b = i * G + g reads image i's dY channel slice of group g (one
// image of gtp, the NCHW slices are Mg * outH * outW apart; the aux likewise), writes dX channels g * Cg .. (one output image
// of gtp) and reads the rotated filters W'_g of group b % G.
//   PATH_AUTO: conv_auto_path over gtp.  The exact path is the direct kernel over gt (gemm_simt.cuh: conv_grouped_direct_kernel
//   with GRAD), one launch, the filters read rotated in place.  The tensor-core paths are the batched fused product over gtp
//   with A = W' copied once per call into tfilt as G problems of [Cg][round_up(K', 4)], periodic with period G
//   (batched_fused_dev), and B the dilated, op'd windows of dY (split.cuh: Im2colGradSrc); a 1 x 1 kernel with unit strides
//   and no padding reads dY in place and the filters transposed, no copy.
int conv2d_grouped_input_grad_dev(float *grad_input, const ConvGeom &g, int64_t groups, const float *grad_output, const float *kernel,
                                  float alpha, float beta, const laser_b200_operand_op *op_in, int path, void *stream) {
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  OperandOp op;
  const OperandOp *opB;
  if ((rc = operand_op_of(op_in, true, &op, &opB))) return rc;
  const int64_t P = g.outHW(), khw = g.kH * g.kW;
  if (opB && opB->aux && (opB->aux_sr != 1 || opB->aux_sc != P))
    return set_error(LASER_B200_EINVAL, "the aux tensor of op %d must be dense like grad_output: strides (%lld, 1), not (%lld, %lld)",
                     opB->op, (long long)P, (long long)opB->aux_sc, (long long)opB->aux_sr);
  if (g.B == 0) return LASER_B200_OK;
  if (!grad_input || !grad_output || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  const int64_t Cg = g.C / groups, Mg = g.Cout / groups;
  if (Mg > INT32_MAX / khw) return set_error(LASER_B200_EUNSUPPORTED, "c_out / groups * kH * kW beyond 2^31");
  ConvGeom gt = transposed_geom(g);
  ConvGeom gtp = gt;
  gtp.B = g.B * groups;
  gtp.C = Mg;
  gtp.Cout = Cg;
  if (path == LASER_B200_PATH_AUTO) path = conv_auto_path(gtp, Epilogue());
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_SIMT) {
    ConvGroupedGradParams p;
    int mc;
    size_t smem;
    const int threads = conv_grouped_plan(gt, groups, nullptr, 0, &p, &mc, &smem);
    if (threads == 0)
      return set_error(LASER_B200_EUNSUPPORTED, "grouped convolution input gradient: a %lld x %lld kernel window does not fit in "
                       "shared memory", (long long)g.kH, (long long)g.kW);
    p.dH = static_cast<int>(g.sH);
    p.dW = static_cast<int>(g.sW);
    p.alpha = alpha;
    p.beta = beta;
    p.op = opB ? opB->op : 0;
    p.aux = opB ? opB->aux : nullptr;
    const int grid = grid_for(*c, p.tiles, 2048 / threads);
    if (mc == 4) conv_grouped_direct_kernel<4, true><<<grid, threads, smem, s>>>(grad_input, grad_output, kernel, p);
    else if (mc == 2) conv_grouped_direct_kernel<2, true><<<grid, threads, smem, s>>>(grad_input, grad_output, kernel, p);
    else conv_grouped_direct_kernel<1, true><<<grid, threads, smem, s>>>(grad_input, grad_output, kernel, p);
    COUNT_LAUNCH();
    CHECK_LAUNCH();
  } else {
    const int64_t M = Cg, N = gtp.outHW(), K = gtp.K(), image = Mg * g.outH * g.outW;
    if (khw == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0) {
      // dX_{n,g} = W_g^T * dY_{n,g}: group g's filters [Mg][Cg] read transposed, dY in place
      const laser_b200_batch_strides bs{Mg * Cg, image, M * N, 0, image};
      if ((rc = batched_fused_dev(gtp.B, M, N, K, alpha, kernel, 1, Cg, grad_output, N, 1, beta, grad_input, N, 1, &bs, nullptr, opB,
                                  Epilogue(), path, s, nullptr, groups)))
        return rc;
    } else {
      // W' of every group once per call into tfilt (held for the whole call), K-major rows 16 bytes apart, read in place by
      // every chunk's product; the copy waits for the last kernel that read the buffer (ws_free)
      std::lock_guard<std::mutex> lk(c->tfilt_mu);
      const int64_t lda = round_up(K, 4);
      if ((rc = ensure(c->tfilt, static_cast<size_t>(g.C * lda) * sizeof(float)))) return rc;
      CUDA_TRY(cudaStreamWaitEvent(s, c->ws_free, 0));
      const int64_t shape[4] = {groups, Cg, Mg, khw}, dst_st[4] = {Cg * lda, lda, khw, 1}, src_st[4] = {Mg * Cg * khw, khw, Cg * khw, -1};
      CopyParams cp;
      copy_plan(4, shape, dst_st, src_st, &cp);
      float *wt = static_cast<float *>(c->tfilt.ptr);
      if ((rc = launch_copy<uint32_t>(*c, wt, kernel + khw - 1, cp, s))) return rc;
      const laser_b200_batch_strides bs{Cg * lda, image, M * N, 0, image};
      if ((rc = batched_fused_dev(gtp.B, M, N, K, alpha, wt, lda, 1, grad_output, N, 1, beta, grad_input, N, 1, &bs, nullptr, opB,
                                  Epilogue(), path, s, &gtp, groups)))
        return rc;
    }
  }
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// laser_b200_conv2d_nhwc_input_grad_f32_fused_dev (capi_layers.inc checks the geometry): NHWC output gradients and input
// gradient, ONE product for the images of a chunk,
//   dX[n * H * W + q][ci] <- alpha * sum_k' R[n * H * W + q][k'] * W'^T[ci][k'] + beta * dX[n * H * W + q][ci]
// with k' = (kh' * kW + kw') * Cout + co, T = kH * kW, W'^T[ci][k'] = Wmat[(T - 1 - (kh' * kW + kw')) * C + ci][co]: M = n * H * W,
// N = C, K' = T * Cout.  A = R, the input pixels' windows over op(dY) zero-dilated by the forward strides -- the transposed
// geometry of conv2d_input_grad_dev, channels-last (split.cuh: Im2colNhwcGradSrc); B = W'^T, copied once per call into tfilt as
// K-major rows [C][round_up(K', 4)]: no rank-2 view of the caller's filters has k' in (tap, co) order, and ordering A by (co,
// tap) instead would lose its channel-contiguous loads.  1 x 1 kernels with unit strides and no padding: the plain product
// op(dY) * Wmat^T, dY read in place as [n * P][Cout] and Wmat through its strides, no copy.  Chunks of whole images
// (conv_nhwc_chunks).  PATH_AUTO: the path of conv2d_input_grad_dev for the same geometry.
int conv2d_nhwc_input_grad_dev(float *grad_input, const ConvGeom &g, const float *grad_output, const float *kernel,
                               const int64_t kernelStrides[2], float alpha, float beta, const laser_b200_operand_op *op_in, int path,
                               void *stream) {
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  if (!kernelStrides) return set_error(LASER_B200_EINVAL, "kernelStrides is NULL");
  OperandOp op;
  const OperandOp *opA;
  if ((rc = operand_op_of(op_in, false, &op, &opA))) return rc;
  const int64_t khw = g.kH * g.kW;
  if (opA && opA->aux && (opA->aux_sr != g.Cout || opA->aux_sc != 1))
    return set_error(LASER_B200_EINVAL, "the aux tensor of op %d must be dense NHWC like grad_output: strides (%lld, 1), not (%lld, %lld)",
                     opA->op, (long long)g.Cout, (long long)opA->aux_sr, (long long)opA->aux_sc);
  if (g.B == 0) return LASER_B200_OK;
  if (!grad_input || !grad_output || !kernel) return set_error(LASER_B200_EINVAL, "null pointer");
  if (g.Cout > INT32_MAX / khw) return set_error(LASER_B200_EUNSUPPORTED, "c_out * kH * kW beyond 2^31");
  ConvGeom gt = transposed_geom(g);
  gt.nhwc = true;
  if (path == LASER_B200_PATH_AUTO) path = conv_auto_path(gt, Epilogue());
  if (is_tc_mode(path) && gt.outHW() > 0x7fffffffLL / g.B)
    return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: images * H * W must fit in int32");
  const int64_t K = gt.K(), ks0 = kernelStrides[0], ks1 = kernelStrides[1];
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (khw == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0) {
    rc = conv_nhwc_chunks(*c, path, gt, g.C, alpha, grad_output, kernel, ks1, ks0, beta, grad_input, s, Epilogue(), opA, true);
  } else {
    // W'^T once per call into tfilt (held for the whole call), K-major rows 16 bytes apart, read in place by every chunk's
    // product; the copy waits for the last kernel that read the buffer (ws_free)
    std::lock_guard<std::mutex> lk(c->tfilt_mu);
    const int64_t lda = round_up(K, 4);
    if ((rc = ensure(c->tfilt, static_cast<size_t>(g.C * lda) * sizeof(float)))) return rc;
    CUDA_TRY(cudaStreamWaitEvent(s, c->ws_free, 0));
    const int64_t shape[3] = {g.C, khw, g.Cout}, dst_st[3] = {lda, g.Cout, 1}, src_st[3] = {ks0, -g.C * ks0, ks1};
    CopyParams cp;
    copy_plan(3, shape, dst_st, src_st, &cp);
    float *wt = static_cast<float *>(c->tfilt.ptr);
    if ((rc = launch_copy<uint32_t>(*c, wt, kernel + (khw - 1) * g.C * ks0, cp, s))) return rc;
    rc = conv_nhwc_chunks(*c, path, gt, g.C, alpha, grad_output, wt, 1, lda, beta, grad_input, s, Epilogue(), opA, false);
  }
  if (rc) return rc;
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// ---------------------------------------------------------------------------------------
//   convolution filter gradient: one batch-reduced product whose B is prepared straight from the images
// ---------------------------------------------------------------------------------------
// laser_b200_conv2d_filter_grad_f32_fused_dev (capi_layers.inc checks the geometry):
//   grad_kernel <- alpha * sum_n op(grad_output_n) * im2col(input_n)^T + beta * grad_kernel
// the batch-reduced product with M = Cout, N = Kc = C * kH * kW, K = P = outH * outW per image: A = grad_output ([Cout][P] per
// image, the op's aux laid out the same way), B = the images as a concatenated im2col source.  One chunk always, as for
// batch_reduce_dev: chunks would round dW between them.
int conv2d_filter_grad_dev(float *grad_kernel, const float *input, const ConvGeom &g, const float *grad_output, float alpha,
                           float beta, const laser_b200_operand_op *op_in, int path, void *stream) {
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  OperandOp op;
  const OperandOp *opA;
  if ((rc = operand_op_of(op_in, false, &op, &opA))) return rc;
  const int64_t M = g.Cout, N = g.K(), P = g.outHW(), image = g.C * g.H * g.W;
  if (opA && opA->aux && (opA->aux_sr != P || opA->aux_sc != 1))
    return set_error(LASER_B200_EINVAL, "the aux tensor of op %d must be dense like grad_output: strides (%lld, 1), not (%lld, %lld)",
                     opA->op, (long long)P, (long long)opA->aux_sr, (long long)opA->aux_sc);
  if (g.B == 0) return LASER_B200_OK;
  if (!grad_kernel || !input || !grad_output) return set_error(LASER_B200_EINVAL, "null pointer");
  // B of a 1 x 1 kernel with unit strides and no padding is the images read in place: B_n[p][c] = input_n[c][p]
  const bool in_place = g.kH * g.kW == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0;
  if (!in_place && P > INT64_MAX / g.B) return set_error(LASER_B200_EUNSUPPORTED, "images * outH * outW overflows int64");
  const laser_b200_batch_strides bs{M * P, image, 0, M * P, 0};
  return batch_reduce_dev(g.B, M, N, P, alpha, grad_output, P, 1, input, 1, P, beta, grad_kernel, N, 1, &bs, opA, nullptr, Epilogue(),
                          path, stream, in_place ? nullptr : &g);
}

// laser_b200_conv2d_nhwc_filter_grad_f32_fused_dev (capi_layers.inc checks the geometry): NHWC images and gradients, ONE product
//   dWmat[k][co] <- alpha * sum_j rows[j][k] * op(dY)[j][co] + beta * dWmat[k][co],  j = n * P + p over every image
// with M = Cout, N = K = kH * kW * C, K' = n * P: A = op(dY)^T, the [Cout][n * P] view of the NHWC gradients (strides (1, Cout),
// MN-major; the op's aux laid out the same way), B = the images as channels-last tap rows (ConvGeom::taps), C = the filter matrix
// through kernelStrides (C[co][k] at co * kernelStrides[1] + k * kernelStrides[0]).  NHWC stores the images end to end along j,
// so no batch is reduced.  1 x 1 kernels with unit strides and no padding: B is the images read in place as [C][n * H * W].
// One chunk always: chunks would round dW between them.
int conv2d_nhwc_filter_grad_dev(float *grad_kernel, const float *input, const ConvGeom &g, const float *grad_output,
                                const int64_t kernelStrides[2], float alpha, float beta, const laser_b200_operand_op *op_in, int path,
                                void *stream) {
  int rc;
  if ((rc = check_f32_path(path))) return rc;
  if (!kernelStrides) return set_error(LASER_B200_EINVAL, "kernelStrides is NULL");
  OperandOp op;
  const OperandOp *opA;
  if ((rc = operand_op_of(op_in, false, &op, &opA))) return rc;
  const int64_t M = g.Cout, N = g.K(), P = g.outHW();
  if (opA && opA->aux && (opA->aux_sr != 1 || opA->aux_sc != M))
    return set_error(LASER_B200_EINVAL, "the aux tensor of op %d must be dense NHWC like grad_output: strides (1, %lld), not (%lld, %lld)",
                     opA->op, (long long)M, (long long)opA->aux_sr, (long long)opA->aux_sc);
  if (g.B == 0) return LASER_B200_OK;
  if (!grad_kernel || !input || !grad_output) return set_error(LASER_B200_EINVAL, "null pointer");
  if (P > INT64_MAX / g.B) return set_error(LASER_B200_EUNSUPPORTED, "images * outH * outW overflows int64");
  const int64_t Kr = g.B * P;
  // PATH_AUTO: as the NCHW filter gradient decides for the same geometry (batch_reduce_dev over K' = n * P)
  if (path == LASER_B200_PATH_AUTO) path = resolve_auto(M, N, Kr, Epilogue(), /*operand_op=*/true);
  if (is_tc_mode(path) && Kr > 0x7fffffffLL)
    return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: images * outH * outW must fit in int32");
  const bool in_place = g.kH * g.kW == 1 && g.sH == 1 && g.sW == 1 && g.pH == 0 && g.pW == 0;
  ConvGeom gt = g;
  gt.nhwc = gt.taps = true;
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if ((rc = run_f32(*c, path, M, N, Kr, alpha, grad_output, 1, M, input, g.C, 1, beta, grad_kernel, kernelStrides[1], kernelStrides[0],
                    s, Epilogue(), opA, nullptr, 0, nullptr, false, in_place ? nullptr : &gt)))
    return rc;
  g_last_path = path;
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

// ---------------------------------------------------------------------------------------
//                         host-pointer (drop-in) variants
// ---------------------------------------------------------------------------------------
struct Span {
  int64_t lo, hi;   // element offsets relative to the base pointer, inclusive
  bool dense;       // every element of [lo, hi] belongs to the view
};
Span span_of(int64_t rows, int64_t cols, int64_t rs, int64_t cs) {
  Span sp;
  const int64_t r = (rows - 1) * rs, q = (cols - 1) * cs;
  sp.lo = (r < 0 ? r : 0) + (q < 0 ? q : 0);
  sp.hi = (r > 0 ? r : 0) + (q > 0 ? q : 0);
  const int64_t ars = llabs(rs), acs = llabs(cs);
  sp.dense = (acs == 1 && (ars == cols || rows == 1)) || (ars == 1 && (acs == rows || cols == 1)) ||
             (rows == 1 && cols == 1);
  return sp;
}

// Host-pointer fp32 GEMM, pipelined over row panels (the drop-in call's fast path).
// PCIe is the bound of a host-resident GEMM (805 MB cross the bus for 1.1 TFLOP at 8192^3), so
// the three phases run on three streams: B is uploaded and prepared once; then row panel p+1 of
// A is in flight H2D while panel p is split + multiplied and panel p-1 of C returns D2H.
// Preconditions (checked by the caller): tensor-core path, row panels of A and of C are
// (nearly) disjoint address ranges, C dense inside each panel span (with beta != 0 the old panel of
// C travels to the device next to its panel of A).
struct PanelPlan {
  int64_t rows;   // rows per panel
  int panels;
};
inline bool panel_separable(int64_t rows, int64_t cols, int64_t rs, int64_t cs) {
  // a panel of `rows` consecutive rows must cover an address span not much larger than its data
  const Span sp = span_of(rows, cols, rs, cs);
  const double span = static_cast<double>(sp.hi - sp.lo + 1);
  return llabs(rs) >= llabs(cs) && span <= 1.25 * static_cast<double>(rows) * static_cast<double>(cols);
}

int host_gemm_f32_pipelined(Ctx &c, int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                            int64_t rsA, int64_t csA, const float *B, int64_t rsB, int64_t csB,
                            float beta, float *C, int64_t rsC, int64_t csC, int path) {
  const TcKind kind = tc_kind_of_path(path);
  const bool f16x3 = (kind == TC_F16X3);
  std::lock_guard<std::mutex> host_lk(c.host_mu);
  std::lock_guard<std::mutex> lk(c.mu);
  int rc;
  // Once the first copy is queued the caller's A, B, C are in use by the device: no return -- error or not -- before the
  // three streams have drained (the caller may free or reuse the buffers as soon as this function returns).
  struct Drain {
    Ctx &c;
    bool armed = false;
    ~Drain() {
      if (!armed) return;
      cudaStreamSynchronize(c.up);
      cudaStreamSynchronize(c.stream);
      cudaStreamSynchronize(c.down);
      cudaEventRecord(c.ws_free, c.stream);
    }
  } drain{c};
  const int64_t panel_rows = c.panel_rows;
  // row panels (first row, rows).  The time after the last byte of A has crossed the bus is one
  // panel's split + GEMM + D2H: optionally the last panel is cut finer (halves down to 256 rows).
  std::vector<std::pair<int64_t, int64_t>> plist;
  for (int64_t m0 = 0; m0 < M; m0 += panel_rows) plist.emplace_back(m0, (M - m0 < panel_rows) ? (M - m0) : panel_rows);
  if (c.panel_taper && plist.size() >= 2) {
    int64_t m0 = plist.back().first, rows = plist.back().second;
    plist.pop_back();
    while (rows > 256) {
      const int64_t h = (rows / 2 + 255) / 256 * 256;
      if (h >= rows) break;
      plist.emplace_back(m0, h);
      m0 += h;
      rows -= h;
    }
    plist.emplace_back(m0, rows);
  }
  const int panels = static_cast<int>(plist.size());
  const Span sa = span_of(M, K, rsA, csA), sb = span_of(K, N, rsB, csB), sc = span_of(M, N, rsC, csC);
  const size_t na = static_cast<size_t>(sa.hi - sa.lo + 1) * 4, nb = static_cast<size_t>(sb.hi - sb.lo + 1) * 4;
  const size_t nc = static_cast<size_t>(sc.hi - sc.lo + 1) * 4;
  if ((rc = ensure(c.stage[0], na + 256))) return rc;
  if ((rc = ensure(c.stage[1], nb + 256))) return rc;
  if ((rc = ensure(c.stage[2], nc + 256))) return rc;
  float *dA = static_cast<float *>(c.stage[0].ptr) - sa.lo;   // device address of element A[0,0]
  float *dB = static_cast<float *>(c.stage[1].ptr) - sb.lo;
  float *dC = static_cast<float *>(c.stage[2].ptr) - sc.lo;
  if (static_cast<int>(c.panel_ev.size()) < 2 * panels + 1) {
    const size_t old = c.panel_ev.size();
    c.panel_ev.resize(2 * panels + 1);
    for (size_t i = old; i < c.panel_ev.size(); ++i)
      CUDA_TRY(cudaEventCreateWithFlags(&c.panel_ev[i], cudaEventDisableTiming));
  }
  cudaStream_t up = c.up, cmp = c.stream, down = c.down;
  // f16x3: B's abs-max words are written once, A's (one per row of the panel) are rewritten by every panel's preparation --
  // after the previous panel's GEMM, whose epilogue reads them, because everything of a panel runs on the compute stream
  const SplitMode mode = split_mode(kind);
  // staging buffers / workspace may still be in use by an earlier call
  CUDA_TRY(cudaStreamWaitEvent(up, c.ws_free, 0));
  CUDA_TRY(cudaStreamWaitEvent(cmp, c.ws_free, 0));
  // ---- B: upload once, prepare once ----
  drain.armed = true;
  CUDA_TRY(cudaMemcpyAsync(dB + sb.lo, B + sb.lo, nb, cudaMemcpyHostToDevice, up));
  CUDA_TRY(cudaEventRecord(c.panel_ev[2 * panels], up));
  CUDA_TRY(cudaStreamWaitEvent(cmp, c.panel_ev[2 * panels], 0));
  OperandMaps mb;
  bool used_ws = false;
  Operand ob{dB, N, K, csB, rsB};
  int64_t f16_b_off = 0;       // f16x3: room for the longest panel's rows of A + the columns of B
  if (f16x3 && (rc = f16_scales(c, panel_rows < M ? panel_rows : M, N, &f16_b_off))) return rc;
  if ((rc = prepare_operand<4>(c, ob, mode, ws_of_B(c, f16_b_off), TC_BLOCK_N, &mb, &used_ws, cmp)))
    return rc;
  const F16Scales f16{static_cast<const uint32_t *>(c.f16s.ptr), static_cast<const uint32_t *>(c.f16s.ptr) + f16_b_off};
  // ---- row panels ----
  for (int pnl = 0; pnl < panels; ++pnl) {
    const int64_t m0 = plist[pnl].first;
    const int64_t mp = plist[pnl].second;
    const float *Ap = A + m0 * rsA;
    float *Cp = C + m0 * rsC;
    const Span pa = span_of(mp, K, rsA, csA), pc = span_of(mp, N, rsC, csC);
    CUDA_TRY(cudaMemcpyAsync(dA + m0 * rsA + pa.lo, Ap + pa.lo, static_cast<size_t>(pa.hi - pa.lo + 1) * 4,
                             cudaMemcpyHostToDevice, up));
    if (beta != 0.0f)   // the old values of this panel of C are read by the epilogue
      CUDA_TRY(cudaMemcpyAsync(dC + m0 * rsC + pc.lo, Cp + pc.lo, static_cast<size_t>(pc.hi - pc.lo + 1) * 4,
                               cudaMemcpyHostToDevice, up));
    CUDA_TRY(cudaEventRecord(c.panel_ev[pnl], up));
    CUDA_TRY(cudaStreamWaitEvent(cmp, c.panel_ev[pnl], 0));
    OperandMaps ma;
    Operand oa{dA + m0 * rsA, mp, K, rsA, csA};
    if ((rc = prepare_operand<4>(c, oa, mode, ws_of_A(c), TC_BLOCK_M, &ma, &used_ws, cmp))) return rc;
    rc = tc_run<float>(c, kind, mp, N, K, alpha, ma, mb, beta, dC + m0 * rsC, rsC, csC, cmp, Epilogue(),
                       f16x3 ? &f16 : nullptr, mode != SPLIT_NONE && !c.profiling);
    if (rc) return rc;
    CUDA_TRY(cudaEventRecord(c.panel_ev[panels + pnl], cmp));
    CUDA_TRY(cudaStreamWaitEvent(down, c.panel_ev[panels + pnl], 0));
    CUDA_TRY(cudaMemcpyAsync(Cp + pc.lo, dC + m0 * rsC + pc.lo, static_cast<size_t>(pc.hi - pc.lo + 1) * 4,
                             cudaMemcpyDeviceToHost, down));
  }
  CUDA_TRY(cudaEventRecord(c.ws_free, cmp));
  CUDA_TRY(cudaStreamSynchronize(down));
  CUDA_TRY(cudaStreamSynchronize(cmp));
  drain.armed = false;
  g_last_path = path;
  return LASER_B200_OK;
}

template <typename T, typename Fn>
int host_gemm(int64_t M, int64_t N, int64_t K, const T *A, int64_t rsA, int64_t csA, const T *B,
              int64_t rsB, int64_t csB, bool beta_zero, T *C, int64_t rsC, int64_t csC, Fn run) {
  int rc = check_args(M, N, K, A, B, C);
  if (rc == -1) return LASER_B200_OK;
  if (rc) return rc;
  Ctx *c;
  rc = get_ctx(&c);
  if (rc) return rc;
  const Span sa = span_of(M, K, rsA, csA), sb = span_of(K, N, rsB, csB), sc = span_of(M, N, rsC, csC);
  const size_t na = static_cast<size_t>(sa.hi - sa.lo + 1) * sizeof(T);
  const size_t nb = static_cast<size_t>(sb.hi - sb.lo + 1) * sizeof(T);
  const size_t nc = static_cast<size_t>(sc.hi - sc.lo + 1) * sizeof(T);
  std::lock_guard<std::mutex> host_lk(c->host_mu);  // one host-pointer call at a time per device
  if ((rc = ensure(c->stage[0], na + 256))) return rc;
  if ((rc = ensure(c->stage[1], nb + 256))) return rc;
  if ((rc = ensure(c->stage[2], nc + 256))) return rc;
  T *dA = static_cast<T *>(c->stage[0].ptr);
  T *dB = static_cast<T *>(c->stage[1].ptr);
  T *dC = static_cast<T *>(c->stage[2].ptr);
  cudaStream_t s = c->stream;
  CUDA_TRY(cudaMemcpyAsync(dA, A + sa.lo, na, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(dB, B + sb.lo, nb, cudaMemcpyHostToDevice, s));
  // C travels to the device only if it is read (beta != 0) or if the span holds
  // elements outside the view that must survive the round trip
  if (!beta_zero || !sc.dense) CUDA_TRY(cudaMemcpyAsync(dC, C + sc.lo, nc, cudaMemcpyHostToDevice, s));
  rc = run(dA - sa.lo, dB - sb.lo, dC - sc.lo, static_cast<void *>(s));
  if (rc) {   // copies from the caller's buffers may still be in flight
    cudaStreamSynchronize(s);
    return rc;
  }
  CUDA_TRY(cudaMemcpyAsync(C + sc.lo, dC, nc, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  return LASER_B200_OK;
}

}  // namespace

// =======================================================================================
//                                     extern "C"
// =======================================================================================
extern "C" {

int laser_b200_init(void) {
  Ctx *c;
  return get_ctx(&c);
}

void laser_b200_shutdown(void) {
  multi_shutdown();
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  int cur = 0;
  cudaGetDevice(&cur);
  for (int d = 0; d < kMaxDevices; ++d) {
    Ctx &c = g_ctx[d];
    if (!c.ready) continue;
    cudaSetDevice(d);
    cudaStreamSynchronize(c.stream);
    for (auto &b : c.ws) { if (b.ptr) cudaFree(b.ptr); b = Buffer(); }
    for (auto &b : c.stage) { if (b.ptr) cudaFree(b.ptr); b = Buffer(); }
    if (c.splitk.ptr) { cudaFree(c.splitk.ptr); c.splitk = Buffer(); }
    if (c.bpanels.ptr) { cudaFree(c.bpanels.ptr); c.bpanels = Buffer(); }
    if (c.layer_ws.ptr) { cudaFree(c.layer_ws.ptr); c.layer_ws = Buffer(); }
    if (c.tfilt.ptr) { cudaFree(c.tfilt.ptr); c.tfilt = Buffer(); }
    if (c.f16s.ptr) { cudaFree(c.f16s.ptr); c.f16s = Buffer(); }
    for (auto &b : c.gather) { if (b.ptr) cudaFree(b.ptr); b = Buffer(); }
    if (c.sched.ptr) { cudaFree(c.sched.ptr); c.sched = Buffer(); }
    c.sched_next = 0;
    for (auto &e : c.map_cache) e.valid = false;
    cudaEventDestroy(c.ws_free);
    for (auto e : c.panel_ev) cudaEventDestroy(e);
    c.panel_ev.clear();
    cudaStreamDestroy(c.stream);
    cudaStreamDestroy(c.up);
    cudaStreamDestroy(c.down);
    c.ready = false;
  }
  cudaSetDevice(cur);
}

int laser_b200_profile_begin(void) {
  Ctx *c;
  int rc = get_ctx(&c);
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  for (auto &e : c->prof) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  c->prof.clear();
  c->profiling = true;
  return LASER_B200_OK;
}
int laser_b200_profile_end(double *gemm_ms, int64_t *gemm_launches, double *prep_ms,
                           int64_t *prep_launches) {
  Ctx *c;
  int rc = get_ctx(&c);
  if (rc) return rc;
  CUDA_TRY(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(c->mu);
  double ms[2] = {0.0, 0.0};
  int64_t n[2] = {0, 0};
  for (auto &e : c->prof) {
    float t = 0.0f;
    if (e.launches > 0) {
      CUDA_TRY(cudaEventElapsedTime(&t, e.a, e.b));
      ms[e.kind] += t;
      n[e.kind] += e.launches;
    }
    cudaEventDestroy(e.a);
    cudaEventDestroy(e.b);
  }
  c->prof.clear();
  c->profiling = false;
  if (gemm_ms) *gemm_ms = ms[0];
  if (gemm_launches) *gemm_launches = n[0];
  if (prep_ms) *prep_ms = ms[1];
  if (prep_launches) *prep_launches = n[1];
  return LASER_B200_OK;
}

const char *laser_b200_last_error(void) { return g_last_error.c_str(); }
int laser_b200_version(void) { return 200; }
int64_t laser_b200_launch_count(void) { return g_launches.load(); }
int laser_b200_last_path(void) { return g_last_path; }
int laser_b200_set_f32_mode(int path) {
  if (path != LASER_B200_PATH_SIMT && path != LASER_B200_PATH_TF32X1 && path != LASER_B200_PATH_TF32X3 &&
      path != LASER_B200_PATH_F16X3)
    return set_error(LASER_B200_EINVAL, "f32 mode must be F16X3, TF32X3, TF32X1 or SIMT");
  g_f32_mode.store(path);
  return LASER_B200_OK;
}
int laser_b200_get_f32_mode(void) {
  const int m = g_f32_mode.load();
  return m < 0 ? parse_f32_mode(getenv("LASER_B200_F32_MODE")) : m;
}

// ---- device-resident -----------------------------------------------------------------
int laser_b200_gemm_strided_f32_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                    int64_t rsA, int64_t csA, const float *B, int64_t rsB,
                                    int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                                    int path, void *stream) {
  return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream);
}
int laser_b200_gemm_strided_f32_epi_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                        int64_t rsA, int64_t csA, const float *B, int64_t rsB,
                                        int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                                        const laser_b200_epilogue *epi, int path, void *stream) {
  Epilogue e;
  const int rc = epilogue_of(epi, &e);
  if (rc) return rc;
  return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, e);
}
int laser_b200_gemm_strided_f32_fused_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                          int64_t rsA, int64_t csA, const float *B, int64_t rsB,
                                          int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                                          const laser_b200_operand_op *opA, const laser_b200_operand_op *opB,
                                          const laser_b200_epilogue *epi, int path, void *stream) {
  FusedArgs f;
  const int rc = fused_args_of(epi, opA, opB, &f);
  if (rc) return rc;
  return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, f.epi, nullptr, f.opA, f.opB);
}
int laser_b200_gemm_strided_batch_reduce_f32_fused_dev(int64_t batch, int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                                       int64_t rsA, int64_t csA, const float *B, int64_t rsB, int64_t csB, float beta,
                                                       float *C, int64_t rsC, int64_t csC, const laser_b200_batch_strides *batchStrides,
                                                       const laser_b200_operand_op *opA, const laser_b200_operand_op *opB,
                                                       const laser_b200_epilogue *epi, int path, void *stream) {
  FusedArgs f;
  const int rc = fused_args_of(epi, opA, opB, &f);
  if (rc) return rc;
  return batch_reduce_dev(batch, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, batchStrides, f.opA, f.opB, f.epi, path,
                          stream);
}
int laser_b200_gemm_strided_f64_dev(int64_t M, int64_t N, int64_t K, double alpha, const double *A,
                                    int64_t rsA, int64_t csA, const double *B, int64_t rsB,
                                    int64_t csB, double beta, double *C, int64_t rsC, int64_t csC,
                                    void *stream) {
  return simt_dev<double>(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, stream);
}
int laser_b200_gemm_strided_i32_dev(int64_t M, int64_t N, int64_t K, int32_t alpha, const int32_t *A,
                                    int64_t rsA, int64_t csA, const int32_t *B, int64_t rsB,
                                    int64_t csB, int32_t beta, int32_t *C, int64_t rsC, int64_t csC,
                                    void *stream) {
  return simt_dev<int32_t>(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, stream);
}
int laser_b200_gemm_strided_i64_dev(int64_t M, int64_t N, int64_t K, int64_t alpha, const int64_t *A,
                                    int64_t rsA, int64_t csA, const int64_t *B, int64_t rsB,
                                    int64_t csB, int64_t beta, int64_t *C, int64_t rsC, int64_t csC,
                                    void *stream) {
  return simt_dev<int64_t>(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, stream);
}
int laser_b200_gemm_strided_bf16_dev(int64_t M, int64_t N, int64_t K, float alpha, const uint16_t *A,
                                     int64_t rsA, int64_t csA, const uint16_t *B, int64_t rsB,
                                     int64_t csB, float beta, uint16_t *C, int64_t rsC, int64_t csC,
                                     void *stream) {
  return bf16_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, stream);
}

// ---- host pointers (the drop-in signature, gemm.nim:184-193) ---------------------------
int laser_b200_gemm_strided_f32(int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                int64_t rsA, int64_t csA, const float *B, int64_t rsB, int64_t csB,
                                float beta, float *C, int64_t rsC, int64_t csC) {
  // large tensor-core problems whose row panels are separate address ranges: overlap the
  // PCIe transfers with the compute, panel by panel
  if (M >= 2048 && K > 0 && A && B && C &&
      M <= 0x7fffffffLL && N <= 0x7fffffffLL && K <= 0x7fffffffLL) {
    Ctx *c;
    int rc = get_ctx(&c);
    if (rc) return rc;
    const int mode = resolve_auto(M, N, K, Epilogue());   // the kernel family the device entry would pick
    if (is_tc_mode(mode) && panel_separable(c->panel_rows, K, rsA, csA) && panel_separable(c->panel_rows, N, rsC, csC) &&
        span_of(c->panel_rows, N, rsC, csC).dense && rsA > 0 && rsC > 0)
      return host_gemm_f32_pipelined(*c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, mode);
  }
  return host_gemm<float>(M, N, K, A, rsA, csA, B, rsB, csB, beta == 0.0f, C, rsC, csC,
                          [&](const float *a, const float *b, float *c, void *s) {
                            return f32_dev(M, N, K, alpha, a, rsA, csA, b, rsB, csB, beta, c, rsC, csC,
                                           LASER_B200_PATH_AUTO, s);
                          });
}
int laser_b200_gemm_strided_f64(int64_t M, int64_t N, int64_t K, double alpha, const double *A,
                                int64_t rsA, int64_t csA, const double *B, int64_t rsB, int64_t csB,
                                double beta, double *C, int64_t rsC, int64_t csC) {
  return host_gemm<double>(M, N, K, A, rsA, csA, B, rsB, csB, beta == 0.0, C, rsC, csC,
                           [&](const double *a, const double *b, double *c, void *s) {
                             return simt_dev<double>(M, N, K, alpha, a, rsA, csA, b, rsB, csB, beta, c,
                                                     rsC, csC, s);
                           });
}
int laser_b200_gemm_strided_i32(int64_t M, int64_t N, int64_t K, int32_t alpha, const int32_t *A,
                                int64_t rsA, int64_t csA, const int32_t *B, int64_t rsB, int64_t csB,
                                int32_t beta, int32_t *C, int64_t rsC, int64_t csC) {
  return host_gemm<int32_t>(M, N, K, A, rsA, csA, B, rsB, csB, beta == 0, C, rsC, csC,
                            [&](const int32_t *a, const int32_t *b, int32_t *c, void *s) {
                              return simt_dev<int32_t>(M, N, K, alpha, a, rsA, csA, b, rsB, csB, beta, c,
                                                       rsC, csC, s);
                            });
}
int laser_b200_gemm_strided_i64(int64_t M, int64_t N, int64_t K, int64_t alpha, const int64_t *A,
                                int64_t rsA, int64_t csA, const int64_t *B, int64_t rsB, int64_t csB,
                                int64_t beta, int64_t *C, int64_t rsC, int64_t csC) {
  return host_gemm<int64_t>(M, N, K, A, rsA, csA, B, rsB, csB, beta == 0, C, rsC, csC,
                            [&](const int64_t *a, const int64_t *b, int64_t *c, void *s) {
                              return simt_dev<int64_t>(M, N, K, alpha, a, rsA, csA, b, rsB, csB, beta, c,
                                                       rsC, csC, s);
                            });
}
int laser_b200_gemm_strided_bf16(int64_t M, int64_t N, int64_t K, float alpha, const uint16_t *A,
                                 int64_t rsA, int64_t csA, const uint16_t *B, int64_t rsB,
                                 int64_t csB, float beta, uint16_t *C, int64_t rsC, int64_t csC) {
  return host_gemm<uint16_t>(M, N, K, A, rsA, csA, B, rsB, csB, beta == 0.0f, C, rsC, csC,
                             [&](const uint16_t *a, const uint16_t *b, uint16_t *c, void *s) {
                               return bf16_dev(M, N, K, alpha, a, rsA, csA, b, rsB, csB, beta, c, rsC,
                                               csC, s);
                             });
}

// ---- pre-packed operands (gemm_prepacked.nim:63-292) --------------------------------------
size_t laser_b200_gemm_prepackA_mem_required_f32(int64_t M, int64_t N, int64_t K) {
  (void)N;
  return (M > 0 && K > 0) ? packed_layout(M, K).bytes : 0;
}
size_t laser_b200_gemm_prepackB_mem_required_f32(int64_t M, int64_t N, int64_t K) {
  (void)M;
  return (N > 0 && K > 0) ? packed_layout(N, K).bytes : 0;
}
int laser_b200_gemm_prepackA_f32_dev(void *dst, int64_t M, int64_t N, int64_t K, const float *A,
                                     int64_t rsA, int64_t csA, void *stream) {
  (void)N;
  return prepack_dev(0, dst, M, K, A, rsA, csA, stream);
}
int laser_b200_gemm_prepackB_f32_dev(void *dst, int64_t M, int64_t N, int64_t K, const float *B,
                                     int64_t rsB, int64_t csB, void *stream) {
  (void)M;
  return prepack_dev(1, dst, N, K, B, csB, rsB, stream);   // B seen as [n][k]
}
int laser_b200_gemm_packed_f32_dev(int64_t M, int64_t N, int64_t K, float alpha, const void *packedA,
                                   const void *packedB, float beta, float *C, int64_t rsC, int64_t csC,
                                   void *stream) {
  return gemm_packed_dev(M, N, K, alpha, nullptr, 0, 0, packedA, packedB, beta, C, rsC, csC, stream);
}
int laser_b200_gemm_packedB_f32_dev(int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                                    int64_t rsA, int64_t csA, const void *packedB, float beta, float *C,
                                    int64_t rsC, int64_t csC, void *stream) {
  if (!A) return set_error(LASER_B200_EINVAL, "null pointer");
  return gemm_packed_dev(M, N, K, alpha, A, rsA, csA, nullptr, packedB, beta, C, rsC, csC, stream);
}

// ---- storage -----------------------------------------------------------------------------
int laser_b200_malloc(void **dev_ptr, size_t bytes) {
  if (!dev_ptr) return set_error(LASER_B200_EINVAL, "null out pointer");
  Ctx *c;
  int rc = get_ctx(&c);
  if (rc) return rc;
  *dev_ptr = nullptr;
  CUDA_TRY(cudaMalloc(dev_ptr, bytes ? bytes : 1));
  return LASER_B200_OK;
}
int laser_b200_free(void *dev_ptr) {
  if (dev_ptr) CUDA_TRY(cudaFree(dev_ptr));
  return LASER_B200_OK;
}
int laser_b200_memcpy_h2d(void *dst_dev, const void *src_host, size_t bytes) {
  CUDA_TRY(cudaMemcpy(dst_dev, src_host, bytes, cudaMemcpyHostToDevice));
  return LASER_B200_OK;
}
int laser_b200_memcpy_d2h(void *dst_host, const void *src_dev, size_t bytes) {
  CUDA_TRY(cudaMemcpy(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost));
  return LASER_B200_OK;
}
int laser_b200_memset_zero(void *dst_dev, size_t bytes) {
  CUDA_TRY(cudaMemset(dst_dev, 0, bytes));
  return LASER_B200_OK;
}
int laser_b200_synchronize(void) {
  CUDA_TRY(cudaDeviceSynchronize());
  return LASER_B200_OK;
}

int laser_b200_matmul_views(const laser_b200_tensor_view *A, const laser_b200_tensor_view *B,
                            laser_b200_tensor_view *C, double alpha, double beta, int path,
                            void *stream) {
  if (!A || !B || !C) return set_error(LASER_B200_EINVAL, "null view");
  if (A->rank != 2 || B->rank != 2 || C->rank != 2)
    return set_error(LASER_B200_EINVAL, "matmul needs rank-2 views (got %d, %d, %d)", A->rank, B->rank, C->rank);
  if (A->dtype != B->dtype || A->dtype != C->dtype) return set_error(LASER_B200_EINVAL, "dtype mismatch");
  const int64_t M = A->shape[0], K = A->shape[1], N = B->shape[1];
  if (B->shape[0] != K || C->shape[0] != M || C->shape[1] != N)
    return set_error(LASER_B200_EINVAL, "shape mismatch: A %lldx%lld B %lldx%lld C %lldx%lld", (long long)M,
                     (long long)K, (long long)B->shape[0], (long long)N, (long long)C->shape[0],
                     (long long)C->shape[1]);
#define LB200_RAW(T, v) (static_cast<T *>((v)->storage) + (v)->offset)
  switch (A->dtype) {
    case 0:
      return f32_dev(M, N, K, (float)alpha, LB200_RAW(float, A), A->strides[0], A->strides[1],
                     LB200_RAW(float, B), B->strides[0], B->strides[1], (float)beta, LB200_RAW(float, C),
                     C->strides[0], C->strides[1], path, stream);
    case 1:
      return simt_dev<double>(M, N, K, alpha, LB200_RAW(double, A), A->strides[0], A->strides[1],
                              LB200_RAW(double, B), B->strides[0], B->strides[1], beta,
                              LB200_RAW(double, C), C->strides[0], C->strides[1], stream);
    case 2:
      return simt_dev<int32_t>(M, N, K, (int32_t)alpha, LB200_RAW(int32_t, A), A->strides[0],
                               A->strides[1], LB200_RAW(int32_t, B), B->strides[0], B->strides[1],
                               (int32_t)beta, LB200_RAW(int32_t, C), C->strides[0], C->strides[1], stream);
    case 3:
      return simt_dev<int64_t>(M, N, K, (int64_t)alpha, LB200_RAW(int64_t, A), A->strides[0],
                               A->strides[1], LB200_RAW(int64_t, B), B->strides[0], B->strides[1],
                               (int64_t)beta, LB200_RAW(int64_t, C), C->strides[0], C->strides[1], stream);
    case 4:
      return bf16_dev(M, N, K, (float)alpha, LB200_RAW(uint16_t, A), A->strides[0], A->strides[1],
                      LB200_RAW(uint16_t, B), B->strides[0], B->strides[1], (float)beta,
                      LB200_RAW(uint16_t, C), C->strides[0], C->strides[1], stream);
    default:
      return set_error(LASER_B200_EINVAL, "unknown dtype %d", A->dtype);
  }
#undef LB200_RAW
}

int64_t laser_b200_debug_f64_dmma_launches(void) { return g_dmma_launches.load(); }

int laser_b200_debug_classify(int elem_size, const void *base, int64_t s_mn, int64_t s_k) {
  if (elem_size != 2 && elem_size != 4) return -1;
  Operand o{base, 1, 1, s_mn, s_k};
  return static_cast<int>(classify(o, elem_size));
}
int laser_b200_debug_span(int64_t rows, int64_t cols, int64_t row_stride, int64_t col_stride, int64_t *lo,
                          int64_t *hi, int *dense) {
  if (rows <= 0 || cols <= 0 || !lo || !hi || !dense) return LASER_B200_EINVAL;
  const Span sp = span_of(rows, cols, row_stride, col_stride);
  *lo = sp.lo; *hi = sp.hi; *dense = sp.dense ? 1 : 0;
  return LASER_B200_OK;
}

int laser_b200_fill_uniform_f32_dev(float *dst_dev, int64_t n, uint64_t seed, float lo, float hi,
                                    void *stream) {
  if (n <= 0) return LASER_B200_OK;
  if (!dst_dev) return set_error(LASER_B200_EINVAL, "null pointer");
  Ctx *c;
  int rc = get_ctx(&c);
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  fill_uniform_f32_kernel<<<grid_for(*c, (n + 255) / 256, 8), 256, 0, s>>>(dst_dev, n, seed, lo, hi);
  COUNT_LAUNCH();
  CHECK_LAUNCH();
  return finish(*c, static_cast<cudaStream_t>(stream), s);
}

}  // extern "C"

#define LB200_BATCHED_FUSED_F32 batched_fused_entry
#define LB200_CONV2D_FUSED_F32 conv2d_fused_dev
#define LB200_CONV2D_NHWC_FUSED_F32 conv2d_nhwc_fused_dev
#define LB200_CONV2D_GROUPED_FUSED_F32 conv2d_grouped_fused_dev
#define LB200_CONV2D_FILTER_GRAD_F32 conv2d_filter_grad_dev
#define LB200_CONV2D_NHWC_FILTER_GRAD_F32 conv2d_nhwc_filter_grad_dev
#define LB200_CONV2D_INPUT_GRAD_F32 conv2d_input_grad_dev
#define LB200_CONV2D_GROUPED_INPUT_GRAD_F32 conv2d_grouped_input_grad_dev
#define LB200_CONV2D_NHWC_INPUT_GRAD_F32 conv2d_nhwc_input_grad_dev
#include "capi_layers.inc"
#include "capi_multi.inc"
