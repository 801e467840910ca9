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
  Buffer f16s;       // F16X3 mode: fp32 bits of max_k |a| per row of A (words [0, M)) and of max_k |b| per column of B (from
                     // f16_b_off on), written and read on the device
  Buffer sched;      // kSchedSlots x {next unit, CTAs done}: the kernel re-zeroes its slot when it ends
  int sched_next = 0;
  cudaEvent_t ws_free = nullptr;  // recorded after the last kernel that reads ws[]
  std::mutex mu;       // workspace + tensor-map construction
  std::mutex host_mu;  // staging buffers of the host-pointer entry points
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
// (has_op, op, batched): has_op is std::true_type with *op or std::false_type with OperandOp(), batched is std::true_type
// when bt.n > 1.  The kernel's plain, HAS_OP and BATCHED instantiations come from the same launch statement.
template <typename Launch>
int launch_prep(const OperandOp *op, const Batch &bt, Launch launch) {
  auto with_op = [&](auto batched) {
    if (op) launch(std::true_type(), *op, batched);
    else launch(std::false_type(), OperandOp(), batched);
  };
  if (bt.n > 1) with_op(std::true_type());
  else with_op(std::false_type());
  COUNT_LAUNCH();
  CHECK_LAUNCH();
  return LASER_B200_OK;
}
// the problems an operand's preparation covers (an operand the batch shares: one)
inline Batch batch_of(const Operand &o) { return Batch{o.batch > 1 ? o.batch : 1, o.s_b, o.aux_sb}; }

// The gather: op(operand), or the operand itself, from any strides into compact K-major rows [mn][round_up(k, 16 / sizeof(T))]
// allocated in dst (aux read with its own strides).  MODE 1 (fp32): the tf32 hi / lo pieces into dst / *lo.  bf16 operands
// carry no op.
// A batched operand: the problems' rows stacked, [batch][mn][ld].
template <typename T, int MODE = 0>
int gather(Ctx &c, const Operand &o, Buffer &dst, Buffer *lo, cudaStream_t s, const OperandOp *op = nullptr) {
  const Batch bt = batch_of(o);
  const int64_t ld = round_up(o.k, 16 / static_cast<int64_t>(sizeof(T)));
  const size_t bytes = static_cast<size_t>(bt.n * o.mn) * ld * sizeof(T);
  int rc;
  if ((rc = ensure(dst, bytes))) return rc;
  if (MODE == 1 && (rc = ensure(*lo, bytes))) return rc;
  const int64_t tiles = ((o.mn + 31) / 32) * ((o.k + 31) / 32) * bt.n;
  const int read_along_r = (llabs(o.s_mn) < llabs(o.s_k)) ? 1 : 0;
  T *d0 = static_cast<T *>(dst.ptr), *d1 = MODE == 1 ? static_cast<T *>(lo->ptr) : nullptr;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched) {
    constexpr bool HAS_OP = decltype(has_op)::value && sizeof(T) == 4, BATCHED = decltype(batched)::value && sizeof(T) == 4;
    pack_general_kernel<T, MODE, HAS_OP, BATCHED><<<grid_for(c, tiles, 8), 256, 0, s>>>(
        static_cast<const T *>(o.ptr), o.mn, o.k, o.s_mn, o.s_k, d0, d1, ld, read_along_r, k, bt);
  });
}

// TF32X3 in place: tf32 hi / lo pieces [R][ld] of fp32 rows [R][Cc], src_ld apart
int tf32_split(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, float *hi, float *lo, int64_t ld, cudaStream_t s,
               const OperandOp *op, const Batch &bt = Batch()) {
  const int64_t items = bt.n * R * ((Cc + 3) / 4);
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched) {
    split_rows_tf32_kernel<decltype(has_op)::value, decltype(batched)::value><<<grid_for(c, (items + 255) / 256, 8), 256, 0, s>>>(
        src, R, Cc, src_ld, hi, lo, ld, k, bt);
  });
}

// F16X3, one scale per row of fp32 rows [R][Cc] (src_ld apart): the abs-max word of each row, the scale and the two fp16
// pieces [R][ld_b] in ONE pass (split.cuh).  Rows of up to 1024 floats: a warp per row.  Longer rows: prefetched into a
// shared-memory ring by the copy engine when they allow it (16-byte aligned, at most 8192 floats; the ring kernel has no op
// variant, nor a batched one), the CTA per row otherwise.
int f16x2_rows(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
               uint32_t *words, cudaStream_t s, const OperandOp *op = nullptr, const Batch &bt = Batch()) {
  const bool ring = !op && bt.n == 1 && f16x2_rows_ring_ok(src, Cc, src_ld);
  if (ring && !c.ring_attr_set) {
    CUDA_TRY(cudaFuncSetAttribute(f16x2_rows_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(f16x2_rows_ring_smem(4 * 256 * F16ROWS_MAXV))));
    c.ring_attr_set = true;
  }
  const int64_t rows = bt.n * R;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched) {
    constexpr bool HAS_OP = decltype(has_op)::value, BATCHED = decltype(batched)::value;
    if (Cc <= 4 * 32 * F16ROWS_MAXV)
      f16x2_rows_fused_kernel<32, HAS_OP, BATCHED><<<grid_for(c, (rows + 7) / 8, 4), 256, 0, s>>>(src, R, Cc, src_ld, hb, lb, ld_b,
                                                                                             words, k, bt);
    else if (ring)
      f16x2_rows_ring_kernel<<<grid_for(c, R, 2), 256, f16x2_rows_ring_smem(Cc), s>>>(src, R, Cc, src_ld, hb, lb, ld_b, words);
    else
      f16x2_rows_fused_kernel<256, HAS_OP, BATCHED><<<grid_for(c, rows, 4), 256, 0, s>>>(src, R, Cc, src_ld, hb, lb, ld_b, words, k,
                                                                                        bt);
  });
}

// F16X3, one scale per column of fp32 rows [R][Cc]: the abs-max word of every column (zeroed here, then strip reductions
// combined by atomicMax).  A column's scale needs the whole column, so the split is a second pass.
int f16x2_col_scales(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint32_t *words, cudaStream_t s,
                     const OperandOp *op = nullptr, const Batch &bt = Batch()) {
  CUDA_TRY(cudaMemsetAsync(words, 0, static_cast<size_t>(bt.n * Cc) * sizeof(uint32_t), s));
  const int64_t items = ((Cc + 3) / 4) * ((R + ABSMAX_COL_ROWS - 1) / ABSMAX_COL_ROWS) * bt.n;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched) {
    absmax_mn_kernel<true, decltype(has_op)::value, decltype(batched)::value><<<grid_for(c, (items + 255) / 256, 8), 256, 0, s>>>(
        src, R, Cc, src_ld, words, k, bt);
  });
}
// F16X3, one scale per column: the two fp16 pieces [R][ld_b] of fp32 rows [R][Cc] against the columns' scale words
int f16x2_col_split(Ctx &c, const float *src, int64_t R, int64_t Cc, int64_t src_ld, uint16_t *hb, uint16_t *lb, int64_t ld_b,
                    const uint32_t *words, cudaStream_t s, const OperandOp *op = nullptr, const Batch &bt = Batch()) {
  const int64_t items = ((Cc + 255) / 256) * ((R + SPLIT_ROWS - 1) / SPLIT_ROWS) * bt.n;
  return launch_prep(op, bt, [&](auto has_op, const OperandOp &k, auto batched) {
    split_rows_f16x2_kernel<true, decltype(has_op)::value, decltype(batched)::value><<<grid_for(c, items, 8), 256, 0, s>>>(
        src, R, Cc, src_ld, hb, lb, ld_b, words, k, bt);
  });
}

// One operand of a tensor-core call: first the plan, then its steps.
//   bf16 K- or MN-major; TF32X1 K-major without op: TMA reads the caller's memory, no workspace.
//   TF32X3 K-major; F16X3 K- or MN-major -- without op, or with aux laid out like the operand: the split reads the caller's
//     memory and applies the op on load (F16X3 MN-major: all column scales first, then the split).
//   Anything else: one gather, which applies the op, into compact K-major rows.  TMA reads those (bf16, TF32X1), the gather
//     splits them on the way (TF32X3), or the plain row kernel prepares them (F16X3).
// wgmma reads tf32 tiles K-major only, and TMA applies no op.  op: nullptr, or an operand op (fp32 operands only).
// A batched operand (o.batch > 0) is prepared in the same launches, every problem's pieces and scale words stacked; its
// maps are rank 3.  It is read in place only where every problem is: TMA needs a positive batch stride of whole 16-byte
// units, the preparation kernels 16-byte aligned rows (operand and aux) in every problem.
template <int ESZ>
int prepare_operand(Ctx &c, const Operand &o, SplitMode mode, const OperandWs &w, int block_mn,
                    OperandMaps *m, bool *used_ws, cudaStream_t s, const OperandOp *op = nullptr) {
  const Major mj = classify(o, ESZ);
  const Batch bt = batch_of(o);
  const bool rows_ok = bt.n == 1 || ((o.s_b * ESZ) % 16 == 0 && (!op || !op->aux || o.aux_sb % 4 == 0));
  const bool map_ok = bt.n == 1 || (o.s_b > 0 && o.s_b < (static_cast<int64_t>(1) << 40) / ESZ);
  const bool tma_layout = (mj == K_MAJOR || (mj == MN_MAJOR && (ESZ == 2 || mode == SPLIT_F16X2))) && rows_ok;
  const bool in_place = tma_layout && (mode == SPLIT_NONE ? !op && map_ok : !op || op_same_layout(o, *op));
  const Major out_mj = in_place ? mj : K_MAJOR;              // layout of the arrays the tensor-core kernel reads
  const int64_t R = (out_mj == K_MAJOR) ? o.mn : o.k;        // their rows
  const int64_t Cc = (out_mj == K_MAJOR) ? o.k : o.mn;       // their contiguous extent
  const int64_t src_ld = (mj == K_MAJOR) ? o.s_mn : o.s_k;   // row pitch of the operand, read in place
  const int64_t ld = round_up(Cc, 16 / ESZ);
  // rank-3 maps of a batched launch: `depth` matrices (1: shared by the batch) `d_stride(pitch)` elements apart
  const int64_t depth = o.batch > 0 ? bt.n : 0;
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
      const int64_t ld_b = round_up(Cc, 8);
      const size_t bytes_b = static_cast<size_t>(bt.n * R) * ld_b * 2;
      if ((rc = ensure(*w.p0, bytes_b))) return rc;
      if ((rc = ensure(*w.p1, bytes_b))) return rc;
      if (c.f16s.bytes < static_cast<size_t>(w.amax_off + bt.n * o.mn) * sizeof(uint32_t))
        return set_error(LASER_B200_ECUDA, "internal: F16X3 scale buffer not sized for this operand");
      uint16_t *hb = static_cast<uint16_t *>(w.p0->ptr), *lb = static_cast<uint16_t *>(w.p1->ptr);
      uint32_t *words = static_cast<uint32_t *>(c.f16s.ptr) + w.amax_off;
      if (!in_place) {   // the gathered problems are stacked rows: one plain row pass over all of them
        if ((rc = gather<float>(c, o, *w.gather, nullptr, s, op))) return rc;
        rc = f16x2_rows(c, static_cast<const float *>(w.gather->ptr), bt.n * R, Cc, ld, hb, lb, ld_b, words, s);
      } else if (out_mj == K_MAJOR) {
        rc = f16x2_rows(c, src, R, Cc, src_ld, hb, lb, ld_b, words, s, on_load, bt);
      } else {
        if ((rc = f16x2_col_scales(c, src, R, Cc, src_ld, words, s, on_load, bt))) return rc;
        rc = f16x2_col_split(c, src, R, Cc, src_ld, hb, lb, ld_b, words, s, on_load, bt);
      }
      if (rc) return rc;
      if ((rc = operand_map(c, &m->p0, 2, w.p0->ptr, out_mj, o.mn, o.k, ld_b, block_mn, depth, d_stride(ld_b)))) return rc;
      return operand_map(c, &m->p1, 2, w.p1->ptr, out_mj, o.mn, o.k, ld_b, block_mn, depth, d_stride(ld_b));
    }
    if (!in_place) {
      rc = (mode == SPLIT_TF32) ? gather<float, 1>(c, o, *w.p0, w.p1, s, op) : gather<float>(c, o, *w.p0, nullptr, s, op);
    } else {   // TF32X3, K-major
      const size_t bytes = static_cast<size_t>(bt.n * R) * ld * sizeof(float);
      if ((rc = ensure(*w.p0, bytes))) return rc;
      if ((rc = ensure(*w.p1, bytes))) return rc;
      rc = tf32_split(c, src, R, Cc, src_ld, static_cast<float *>(w.p0->ptr), static_cast<float *>(w.p1->ptr), ld, s, on_load, bt);
    }
    if (rc) return rc;
  }
  if ((rc = operand_map(c, &m->p0, ESZ, w.p0->ptr, out_mj, o.mn, o.k, ld, block_mn, depth, d_stride(ld)))) return rc;
  m->p1 = m->p0;
  if (mode == SPLIT_TF32) return operand_map(c, &m->p1, ESZ, w.p1->ptr, out_mj, o.mn, o.k, ld, block_mn, depth, d_stride(ld));
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

// a batched call: `batch` problems, operand X of problem b at X + b * X_stride (0: the batch shares it)
struct BatchArgs {
  int64_t batch;
  int64_t A, B, C, auxA, auxB;
};

// launch the tensor-core kernel on prepared operands (c.mu held by the caller).  bat: a batched launch (tc_params.h; the maps
// are rank 3), with a_shared / b_shared for operands prepared once for the whole batch.
template <typename OutT>
int tc_run(Ctx &c, TcKind kind, int64_t M, int64_t N, int64_t K, float alpha, const OperandMaps &ma,
           const OperandMaps &mb, float beta, OutT *C, int64_t rsC, int64_t csC, cudaStream_t s,
           const Epilogue &epi, const F16Scales *f16 = nullptr, bool after_prep = false, const BatchArgs *bat = nullptr,
           bool a_shared = false, bool b_shared = false) {
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
    p.map_b_a = a_shared ? 0 : 1;
    p.map_b_b = b_shared ? 0 : 1;
    p.bsC = bat->C;
    p.amax_bs_a = a_shared ? 0 : M;
    p.amax_bs_b = b_shared ? 0 : N;
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
            M, N, alpha, beta, C, rsC, csC, p.epi.bias, p.epi.bias_per_row, p.epi.act, p.bsC);
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

// SRC_ESZ: element size of the caller's operands (4: fp32 in any of the three tensor-core modes, 2: bf16)
template <int SRC_ESZ, typename OutT>
int gemm_tc(Ctx &c, TcKind kind, int64_t M, int64_t N, int64_t K, float alpha, const void *A, int64_t rsA,
            int64_t csA, const void *B, int64_t rsB, int64_t csB, float beta, OutT *C, int64_t rsC,
            int64_t csC, cudaStream_t s, const Epilogue &epi, cudaEvent_t b_ready = nullptr, const OperandOp *opA = nullptr,
            const OperandOp *opB = nullptr, const BatchArgs *bat = nullptr) {
  // b_ready: B becomes valid only when this event has fired (the row-sharded driver: B is in flight on the communication
  // stream); everything that does not read B -- the preparation of A -- is queued before the wait.
  // opA / opB: operand ops applied while the operands are prepared (fp32 only)
  if (M > 0x7fffffffLL || N > 0x7fffffffLL || K > 0x7fffffffLL)
    return set_error(LASER_B200_EUNSUPPORTED, "tensor-core path: extents must fit in int32");
  std::lock_guard<std::mutex> lk(c.mu);  // workspace + descriptor construction are per context
  const SplitMode mode = split_mode(kind);
  Operand oa{A, M, K, rsA, csA};
  Operand ob{B, N, K, csB, rsB};
  // bat: every problem's operand in the same launches (an operand -- op included -- that the batch shares: prepared once)
  const bool a_shared = bat && bat->A == 0 && (!opA || !opA->aux || bat->auxA == 0);
  const bool b_shared = bat && bat->B == 0 && (!opB || !opB->aux || bat->auxB == 0);
  if (bat) {
    oa.batch = a_shared ? 1 : bat->batch; oa.s_b = bat->A; oa.aux_sb = bat->auxA;
    ob.batch = b_shared ? 1 : bat->batch; ob.s_b = bat->B; ob.aux_sb = bat->auxB;
  }
  OperandMaps ma, mb;
  bool used_ws = false;
  // the previous call may still be reading the workspace on another stream
  CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
  ProfBracket prep;
  int rc = prep.open(c, s, 1);
  if (rc) return rc;
  int64_t f16_b_off = 0;
  if (mode == SPLIT_F16X2 &&
      (rc = f16_scales(c, batch_of(oa).n * M, batch_of(ob).n * N, &f16_b_off)))
    return rc;
  if ((rc = prepare_operand<SRC_ESZ>(c, oa, mode, ws_of_A(c), TC_BLOCK_M, &ma, &used_ws, s, opA))) return rc;
  if (b_ready) CUDA_TRY(cudaStreamWaitEvent(s, b_ready, 0));
  if ((rc = prepare_operand<SRC_ESZ>(c, ob, mode, ws_of_B(c, f16_b_off), TC_BLOCK_N, &mb, &used_ws, s, opB))) return rc;
  const int prep_launches = prep.launches();
  if ((rc = prep.close())) return rc;
  const F16Scales f16{static_cast<const uint32_t *>(c.f16s.ptr), static_cast<const uint32_t *>(c.f16s.ptr) + f16_b_off};
  // (with profiling on, an event record sits between the last preparation kernel and the GEMM: no dependent launch then)
  rc = tc_run<OutT>(c, kind, M, N, K, alpha, ma, mb, beta, C, rsC, csC, s, epi, mode == SPLIT_F16X2 ? &f16 : nullptr,
                    prep_launches > 0 && !c.profiling, bat, a_shared, b_shared);
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

// Exact path with operand ops: each op'd operand is materialised once by the gather (compact [mn][k] workspace) and the
// unchanged exact kernel multiplies that, so the path stays bit-identical to the CPU reference on the op'd operands.
int gemm_simt_ops(Ctx &c, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
                  const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC, cudaStream_t s,
                  const Epilogue &epi, const OperandOp *opA, const OperandOp *opB) {
  std::lock_guard<std::mutex> lk(c.mu);   // the gather buffers are workspace
  CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
  int rc;
  if (opA) {
    if ((rc = gather<float>(c, Operand{A, M, K, rsA, csA}, c.gather[0], nullptr, s, opA))) return rc;
    A = static_cast<const float *>(c.gather[0].ptr); rsA = round_up(K, 4); csA = 1;
  }
  if (opB) {
    if ((rc = gather<float>(c, Operand{B, N, K, csB, rsB}, c.gather[1], nullptr, s, opB))) return rc;
    B = static_cast<const float *>(c.gather[1].ptr); rsB = 1; csB = round_up(K, 4);
  }
  if ((rc = gemm_simt<float>(c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi))) return rc;
  CUDA_TRY(cudaEventRecord(c.ws_free, s));
  return LASER_B200_OK;
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
  if (has_op && path == -1) return set_error(LASER_B200_EINVAL, "unknown path %d for float32", path);
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
    case LASER_B200_PATH_SIMT:
      if (has_op) rc = gemm_simt_ops(*c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, opA, opB);
      else rc = gemm_simt<float>(*c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi);
      if (rc) return rc;
      g_last_path = LASER_B200_PATH_SIMT;
      break;
    case LASER_B200_PATH_TF32X1:
    case LASER_B200_PATH_TF32X3:
    case LASER_B200_PATH_F16X3:
      // F16X3 (default): two fp16 pieces of each operand scaled by a power of two per row of A / column of B (device-side
      // abs-max), three passes, the epilogue undoes the scales.  TF32X3: hi/lo tf32 pieces, three passes.  TF32X1: one pass.
      rc = gemm_tc<4, float>(*c, tc_kind_of_path(path), M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, b_ready,
                             opA, opB);
      if (rc) return rc;
      g_last_path = path;
      break;
    default:
      return set_error(LASER_B200_EINVAL, "unknown path %d for float32", path);
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
  rc = gemm_tc<2, uint16_t>(*c, TC_BF16, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, Epilogue());
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

// ---------------------------------------------------------------------------------------
//              batched fused product: the problems of a batch in one GEMM launch
// ---------------------------------------------------------------------------------------
// An operand -- with its op -- is the same in every problem: prepared once, read by every problem
inline bool batch_shares(int64_t stride, const OperandOp *op, int64_t aux_stride) {
  return stride == 0 && (!op || !op->aux || aux_stride == 0);
}

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

// problems [0, bat.batch) of a batched call on the resolved path: one preparation launch per step and operand, one GEMM launch
int batched_run(Ctx &c, int path, const BatchArgs &bat, int64_t M, int64_t N, int64_t K, float alpha, const float *A,
                int64_t rsA, int64_t csA, const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC,
                int64_t csC, cudaStream_t s, const Epilogue &epi, const OperandOp *opA, const OperandOp *opB) {
  if (path != LASER_B200_PATH_SIMT)
    return gemm_tc<4, float>(c, tc_kind_of_path(path), M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, nullptr,
                             opA, opB, &bat);
  int64_t bsA = bat.A, bsB = bat.B;
  if (!opA && !opB)
    return gemm_simt<float>(c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, bat.batch, bsA, bsB, bat.C);
  // exact path with ops: the batched gather materialises every problem's op'd operand (gemm_simt_ops, batched)
  std::lock_guard<std::mutex> lk(c.mu);
  CUDA_TRY(cudaStreamWaitEvent(s, c.ws_free, 0));
  int rc;
  if (opA) {
    const bool shared = batch_shares(bat.A, opA, bat.auxA);
    if ((rc = gather<float>(c, Operand{A, M, K, rsA, csA, shared ? 1 : bat.batch, bat.A, bat.auxA}, c.gather[0], nullptr, s, opA)))
      return rc;
    A = static_cast<const float *>(c.gather[0].ptr); rsA = round_up(K, 4); csA = 1; bsA = shared ? 0 : M * rsA;
  }
  if (opB) {
    const bool shared = batch_shares(bat.B, opB, bat.auxB);
    if ((rc = gather<float>(c, Operand{B, N, K, csB, rsB, shared ? 1 : bat.batch, bat.B, bat.auxB}, c.gather[1], nullptr, s, opB)))
      return rc;
    B = static_cast<const float *>(c.gather[1].ptr); rsB = 1; csB = round_up(K, 4); bsB = shared ? 0 : N * csB;
  }
  if ((rc = gemm_simt<float>(c, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, s, epi, bat.batch, bsA, bsB, bat.C)))
    return rc;
  CUDA_TRY(cudaEventRecord(c.ws_free, s));
  return LASER_B200_OK;
}

int batched_fused_dev(int64_t batch, int64_t M, int64_t N, int64_t K, float alpha, const float *A, int64_t rsA, int64_t csA,
                      const float *B, int64_t rsB, int64_t csB, float beta, float *C, int64_t rsC, int64_t csC,
                      const laser_b200_batch_strides *bs, const OperandOp *opA, const OperandOp *opB, const Epilogue &epi,
                      int path, void *stream) {
  if (batch < 0) return set_error(LASER_B200_EINVAL, "negative batch %lld", (long long)batch);
  if (batch > 0 && !bs) return set_error(LASER_B200_EINVAL, "batchStrides is NULL");
  if (batch > 1 && bs->C == 0) return set_error(LASER_B200_EINVAL, "batchStrides->C is 0: the problems' outputs would overlap");
  if (path != LASER_B200_PATH_AUTO && path != LASER_B200_PATH_SIMT && !is_tc_mode(path))
    return set_error(LASER_B200_EINVAL, "unknown path %d for float32", path);
  int rc = check_args(M, N, K, A, B, C);
  if (rc == -1 || batch == 0) return LASER_B200_OK;
  if (rc) return rc;
  if (batch == 1) return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, epi, nullptr, opA, opB);
  Ctx *c;
  if ((rc = get_ctx(&c))) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
  if (path == LASER_B200_PATH_AUTO) path = resolve_auto(M, N, K, epi, /*operand_op=*/true);
  // chunks of whole problems: the prepared workspace stays under the cap, and the launch's tile counts -- batch x tiles x
  // up to 16 K-splits -- fit in int32
  const int64_t per = batch_ws_per_problem(path, M, N, K, !batch_shares(bs->A, opA, bs->auxA), !batch_shares(bs->B, opB, bs->auxB),
                                           opA != nullptr, opB != nullptr);
  int64_t chunk = per > 0 ? c->batch_ws_bytes / per : batch;
  const int64_t tiles = ((M + TC_BLOCK_M - 1) / TC_BLOCK_M) * ((N + TC_BLOCK_N - 1) / TC_BLOCK_N);
  if (chunk > 0x7fffffffLL / (16 * tiles)) chunk = 0x7fffffffLL / (16 * tiles);
  if (chunk < 1) chunk = 1;
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const BatchArgs bat{batch - b0 < chunk ? batch - b0 : chunk, bs->A, bs->B, bs->C, bs->auxA, bs->auxB};
    OperandOp ca, cb;
    if (opA) { ca = *opA; if (ca.aux) ca.aux += b0 * bs->auxA; }
    if (opB) { cb = *opB; if (cb.aux) cb.aux += b0 * bs->auxB; }
    if ((rc = batched_run(*c, path, bat, M, N, K, alpha, A + b0 * bs->A, rsA, csA, B + b0 * bs->B, rsB, csB, beta, C + b0 * bs->C, rsC,
                          csC, s, epi, opA ? &ca : nullptr, opB ? &cb : nullptr)))
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
  Epilogue e;
  OperandOp oa, ob;
  const OperandOp *pa, *pb;
  int rc;
  if ((rc = epilogue_of(epi, &e))) return rc;
  if ((rc = operand_op_of(opA, false, &oa, &pa))) return rc;
  if ((rc = operand_op_of(opB, true, &ob, &pb))) return rc;
  return batched_fused_dev(batch, M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, bs, pa, pb, e, path, stream);
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
  Epilogue e;
  OperandOp oa, ob;
  const OperandOp *pa, *pb;
  int rc;
  if ((rc = epilogue_of(epi, &e))) return rc;
  if ((rc = operand_op_of(opA, false, &oa, &pa))) return rc;
  if ((rc = operand_op_of(opB, true, &ob, &pb))) return rc;
  return f32_dev(M, N, K, alpha, A, rsA, csA, B, rsB, csB, beta, C, rsC, csC, path, stream, e, nullptr, pa, pb);
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
#include "capi_layers.inc"
#include "capi_multi.inc"
