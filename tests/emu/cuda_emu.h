// cuda_emu.h -- TEST INFRASTRUCTURE: runs a __global__ function of the product on host threads so
// that the CPU test suite can execute the kernels' index arithmetic, bounds handling, shared-memory
// choreography and synchronisation protocols without a GPU: one std::thread per CUDA thread, a
// pthread barrier for __syncthreads, clusters of CTAs running side by side, clusters one after the
// other.  Kernels written in plain CUDA C++ run as they are (layers.cuh, gemm_simt.cuh, split.cuh
// with a software tf32 rounding; of the warp intrinsics only full-mask __shfl_xor_sync and
// __syncwarp are modelled); the wgmma kernel runs on top of ptx_emu.h, a functional model of
// the PTX it uses.  It is a test of the product's source, not a fallback: nothing under laser_b200/
// can reach it.
#pragma once

#include <cuda_runtime.h>  // host-side definitions of float4 / make_float4
#include <pthread.h>
#include <stdint.h>

#include <cmath>
#include <sched.h>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#undef __global__
#define __global__
#undef __device__
#define __device__
#undef __host__
#define __host__
#undef __forceinline__
#define __forceinline__ inline
#undef __launch_bounds__
#define __launch_bounds__(...)
#undef __shared__
#define __shared__ static  // one cluster at a time: a function-local static is the block's shared memory
                           // (kernels launched as clusters of 2 must use dynamic shared memory only)
#undef __grid_constant__
#define __grid_constant__

namespace emu {
constexpr unsigned kMaxCluster = 2;                 // CTAs running side by side
constexpr size_t kDynSmemBytes = 232448;            // 227 KB, the sm_90 limit per CTA
struct Idx {
  unsigned x, y, z;
};
inline thread_local Idx t_idx{0, 0, 0};
inline thread_local Idx b_idx{0, 0, 0};
inline thread_local unsigned cta_rank = 0;          // rank of this thread's CTA inside its cluster
inline Idx b_dim{1, 1, 1}, g_dim{1, 1, 1};
inline unsigned cluster_size = 1;
inline pthread_barrier_t cta_barrier[kMaxCluster];  // __syncthreads
inline pthread_barrier_t cluster_barrier;           // barrier.cluster / end of a cluster's run
inline pthread_barrier_t warp_barrier[kMaxCluster][32];   // one per warp (shuffles, __syncwarp)
inline float warp_scratch[kMaxCluster][1024];
inline int warp_scratch_i[kMaxCluster][1024];
inline double warp_scratch_d[kMaxCluster][2][1024];
alignas(1024) inline unsigned char dyn_smem[kMaxCluster][kDynSmemBytes];   // dynamic shared memory
inline unsigned char *dyn_smem_ptr() { return dyn_smem[cta_rank]; }
// ONE emulated device: everything above is global, so kernels launched by concurrent host threads (the library's
// thread-safety test, tests/c_harness/threads_harness.c) run one after the other -- the host code around the launches
// (workspace, tensor-map cache, dispatch state) still runs concurrently, which is what that test is about
inline std::recursive_mutex launch_mu;

// grid = number of CTAs (a multiple of `cluster`); block a multiple of 32 (or < 32 without warp ops).
// Every thread of a CTA must reach every __syncthreads of the kernel (true for the product's kernels).
template <typename Body>
void launch(unsigned grid, unsigned block, Body body, unsigned cluster = 1) {
  std::lock_guard<std::recursive_mutex> device_lk(launch_mu);
  g_dim = Idx{grid, 1, 1};
  b_dim = Idx{block, 1, 1};
  cluster_size = cluster;
  const unsigned warps = (block + 31) / 32;
  for (unsigned r = 0; r < cluster; ++r) {
    pthread_barrier_init(&cta_barrier[r], nullptr, block);
    for (unsigned w = 0; w < warps; ++w) {
      const unsigned lanes = (w + 1) * 32 <= block ? 32 : block - w * 32;
      pthread_barrier_init(&warp_barrier[r][w], nullptr, lanes);
    }
  }
  pthread_barrier_init(&cluster_barrier, nullptr, block * cluster);
  std::vector<std::thread> threads;
  threads.reserve(static_cast<size_t>(block) * cluster);
  for (unsigned r = 0; r < cluster; ++r)
    for (unsigned t = 0; t < block; ++t)
      threads.emplace_back([=]() {
        t_idx = Idx{t, 0, 0};
        cta_rank = r;
        for (unsigned c = 0; c < grid / cluster; ++c) {
          b_idx = Idx{c * cluster + r, 0, 0};
          body();
          pthread_barrier_wait(&cluster_barrier);  // next cluster only when this one is done
        }
      });
  for (auto &th : threads) th.join();
  pthread_barrier_destroy(&cluster_barrier);
  for (unsigned r = 0; r < cluster; ++r) {
    pthread_barrier_destroy(&cta_barrier[r]);
    for (unsigned w = 0; w < warps; ++w) pthread_barrier_destroy(&warp_barrier[r][w]);
  }
}
}  // namespace emu

// correctly rounded single operations (compile with -ffp-contract=off so that a * b + c stays unfused)
inline float __fmaf_rn(float a, float b, float c) { return std::fma(a, b, c); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline double __fma_rn(double a, double b, double c) { return std::fma(a, b, c); }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
template <typename T>
inline T __ldg(const T *p) { return *p; }
inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
inline uint32_t atomicMax(uint32_t *p, uint32_t v) {   // shared or global word; returns the old value
  uint32_t old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
  }
  return old;
}
inline unsigned int atomicAdd(unsigned int *p, unsigned int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T>
inline T __ldcg(const T *p) { return *reinterpret_cast<const volatile T *>(p); }
inline void __nanosleep(unsigned) { sched_yield(); }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }

#define threadIdx (emu::t_idx)
#define blockIdx (emu::b_idx)
inline emu::Idx &blockDim = emu::b_dim;   // plain references, not macros: `cfg.gridDim` must stay a member access
inline emu::Idx &gridDim = emu::g_dim;
inline void __syncthreads() { pthread_barrier_wait(&emu::cta_barrier[emu::cta_rank]); }
inline void __syncwarp() { pthread_barrier_wait(&emu::warp_barrier[emu::cta_rank][emu::t_idx.x >> 5]); }
// full-mask broadcast of `v` from lane `src`: every lane of the warp must call it
inline int __shfl_sync(unsigned, int v, int src) {
  const unsigned t = emu::t_idx.x, w = t >> 5, r = emu::cta_rank;
  emu::warp_scratch_i[r][t] = v;
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  const int out = emu::warp_scratch_i[r][(t & ~31u) + static_cast<unsigned>(src)];
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  return out;
}
inline float __shfl_sync(unsigned, float v, int src) {
  const unsigned t = emu::t_idx.x, w = t >> 5, r = emu::cta_rank;
  emu::warp_scratch[r][t] = v;
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  const float out = emu::warp_scratch[r][(t & ~31u) + static_cast<unsigned>(src)];
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  return out;
}
// full-mask butterfly shuffle: every lane of the warp must call it (true for the reductions it is used in)
inline float __shfl_xor_sync(unsigned, float v, int lane_mask) {
  const unsigned t = emu::t_idx.x, w = t >> 5, r = emu::cta_rank;
  emu::warp_scratch[r][t] = v;
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  const float out = emu::warp_scratch[r][t ^ static_cast<unsigned>(lane_mask)];
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  return out;
}
