// ptx_emu.h -- TEST INFRASTRUCTURE: a functional model of the PTX that laser_b200/csrc/ptx.cuh
// wraps (mbarrier, cp.async.bulk.tensor, wgmma, clusters of two CTAs), under the same names, so
// that gemm_tc.cuh -- the wgmma kernel -- can be compiled by g++ and run on host threads
// (cuda_emu.h).  What the model checks: the producer / consumer protocol (barrier counts, phases,
// stage rings: a protocol error shows up as a deadlock or as a wrong sum), the tile scheduler,
// raster and split-K ranges, the k-block bookkeeping of every mode, operand addressing through the
// descriptors' start / LBO / SBO fields, the accumulator fragment layout the epilogue assumes,
// out-of-bounds zero fill, the cluster's ownership of rows, and every epilogue path.  What it
// cannot check: anything that is a property of the silicon -- the 128-byte swizzle patterns (tiles
// are kept unswizzled here, on both the TMA and the MMA side), instruction encodings, the
// asynchrony of wgmma (an instruction completes when it is issued here), memory-proxy fences,
// register limits, the accumulator's rounding (modelled: tf32 operands truncated, exact products,
// one rounding per instruction).  Those are covered by the -m gpu tests only.
#pragma once

#include <cuda.h>
#include <stdint.h>

#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

// dynamic shared memory of the kernel: this CTA's buffer
#define LB200_DYN_SMEM(T, name) T *name = reinterpret_cast<T *>(emu::dyn_smem_ptr())

namespace emu {

// what the host side of the harness puts inside the 128 opaque bytes of a CUtensorMap: the
// arguments of cuTensorMapEncodeTiled for a 2-d tensor
struct TensorMap2D {
  uint64_t magic;
  const unsigned char *base;
  int64_t dim0, dim1;        // extents in elements, dim0 innermost
  int64_t stride1_bytes;     // pitch of dim1
  int32_t esz, box0, box1;   // element size, box extents in elements
  int64_t dim2 = 1, stride2_bytes = 0;   // rank 3: dim2 matrices, stride2 apart (box depth 1)
};
constexpr uint64_t kMapMagic = 0x4c42323030544d41ull;
static_assert(sizeof(TensorMap2D) <= sizeof(CUtensorMap), "fits in the opaque struct");

struct MBarrier {
  int init_count = 0, pending = 0;
  long tx = 0;
  unsigned phase = 0;
};
inline std::mutex mb_mu;
inline std::condition_variable mb_cv;
inline std::map<const void *, MBarrier> mbars;

inline void reset_state() {
  std::lock_guard<std::mutex> lk(mb_mu);
  mbars.clear();
}
inline void mb_check(MBarrier &b) {
  if (b.pending == 0 && b.tx == 0) {
    b.phase ^= 1u;
    b.pending = b.init_count;
    mb_cv.notify_all();
  }
}
inline MBarrier &mb_get(const void *bar) {
  auto it = mbars.find(bar);
  if (it == mbars.end()) { std::fprintf(stderr, "emu: mbarrier %p used before init\n", bar); std::abort(); }
  return it->second;
}
inline void mb_arrive(const void *bar, long expect_tx) {
  std::lock_guard<std::mutex> lk(mb_mu);
  MBarrier &b = mb_get(bar);
  b.tx += expect_tx;
  if (--b.pending < 0) { std::fprintf(stderr, "emu: mbarrier %p over-arrived\n", bar); std::abort(); }
  mb_check(b);
}
inline void mb_complete_tx(const void *bar, long bytes) {
  std::lock_guard<std::mutex> lk(mb_mu);
  MBarrier &b = mb_get(bar);
  b.tx -= bytes;
  mb_check(b);
}
// the same offset in the shared memory of CTA `rank` of the cluster
template <typename T>
inline T *peer_ptr(T *p, unsigned rank) {
  const unsigned char *q = reinterpret_cast<const unsigned char *>(p);
  for (unsigned r = 0; r < kMaxCluster; ++r)
    if (q >= dyn_smem[r] && q < dyn_smem[r] + kDynSmemBytes)
      return reinterpret_cast<T *>(dyn_smem[rank] + (q - dyn_smem[r]));
  std::fprintf(stderr, "emu: pointer %p is not in shared memory\n", static_cast<const void *>(p));
  std::abort();
}
}  // namespace emu

namespace lb200 {
namespace ptx {

// shared-window address: offset inside the CTA's shared memory, CTA rank in bit 24
inline uint32_t smem_u32(const void *p) {
  const unsigned char *q = static_cast<const unsigned char *>(p);
  for (unsigned r = 0; r < emu::kMaxCluster; ++r)
    if (q >= emu::dyn_smem[r] && q < emu::dyn_smem[r] + emu::kDynSmemBytes)
      return static_cast<uint32_t>(q - emu::dyn_smem[r]) | (r << 24);
  std::fprintf(stderr, "emu: smem_u32 of a pointer outside shared memory\n");
  std::abort();
}
inline bool elect_one() { return (emu::t_idx.x & 31) == 0; }

// ------------------------------------------------------------------ mbarrier
inline void mbar_init(uint64_t *bar, uint32_t count) {
  std::lock_guard<std::mutex> lk(emu::mb_mu);
  emu::MBarrier b;
  b.init_count = b.pending = static_cast<int>(count);
  emu::mbars[bar] = b;
}
inline void fence_barrier_init() {}
inline void fence_proxy_async_smem() {}
inline void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) { emu::mb_arrive(bar, bytes); }
inline void mbar_arrive(uint64_t *bar) { emu::mb_arrive(bar, 0); }
inline bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  std::lock_guard<std::mutex> lk(emu::mb_mu);
  return emu::mb_get(bar).phase != parity;
}
// seconds one thread may wait on one mbarrier before the wait is reported as a deadlock: env LASER_B200_EMU_WAIT_S
// (default 120), ten times that in a sanitizer build, where everything runs several times slower
inline int mbar_wait_limit_s() {
  static const int limit = []() {
    const char *e = std::getenv("LASER_B200_EMU_WAIT_S");
    int v = e ? std::atoi(e) : 0;
    if (v <= 0) v = 120;
#if defined(__SANITIZE_ADDRESS__) || defined(__SANITIZE_THREAD__)
    v *= 10;
#endif
    return v;
  }();
  return limit;
}
inline void mbar_wait(uint64_t *bar, uint32_t parity) {   // blocking (hundreds of waiters on a few cores)
  std::unique_lock<std::mutex> lk(emu::mb_mu);
  emu::MBarrier &b = emu::mb_get(bar);
  // a protocol error is a deadlock: past the limit, report the barrier and the waiting thread instead of hanging
  if (!emu::mb_cv.wait_for(lk, std::chrono::seconds(mbar_wait_limit_s()), [&]() { return b.phase != parity; })) {
    std::fprintf(stderr, "emu: deadlock: thread %u of CTA rank %u waits for parity %u of the mbarrier at shared offset %u "
                 "(pending %d of %d arrivals, tx %ld)\n", emu::t_idx.x, emu::cta_rank, parity,
                 static_cast<unsigned>(smem_u32(bar) & 0xFFFFFF), b.pending, b.init_count, b.tx);
    emu::mb_cv.wait_for(lk, std::chrono::seconds(5));   // the other blocked threads report too
    std::abort();
  }
}

// ----------------------------------------------------------------------- TMA
inline void prefetch_tensormap(const CUtensorMap *) {}
inline void prefetch_l2(const void *) {}
template <int N> inline void setmaxnreg_inc() {}
template <int N> inline void setmaxnreg_dec() {}
inline void tma_copy_box(void *smem_dst, const CUtensorMap *map, int32_t c0, int32_t c1, long *bytes, int32_t c2 = 0) {
  emu::TensorMap2D m;
  std::memcpy(&m, map, sizeof m);
  if (m.magic != emu::kMapMagic) { std::fprintf(stderr, "emu: not an emulated tensor map\n"); std::abort(); }
  unsigned char *dst = static_cast<unsigned char *>(smem_dst);
  {   // the destination must be this CTA's shared memory, whole box inside it, swizzle-atom (1024 B) aligned
    const unsigned char *lo = emu::dyn_smem[emu::cta_rank];
    const size_t box_bytes = static_cast<size_t>(m.box0) * m.box1 * m.esz;
    if (dst < lo || dst + box_bytes > lo + emu::kDynSmemBytes || ((dst - lo) & 1023)) {
      std::fprintf(stderr, "emu: TMA destination outside this CTA's shared memory or not 1024-byte aligned\n");
      std::abort();
    }
  }
  const bool z_inside = c2 >= 0 && c2 < m.dim2;
  m.base += static_cast<int64_t>(z_inside ? c2 : 0) * m.stride2_bytes;
  if (!z_inside) m.dim1 = 0;   // a matrix outside the batch reads as zeros
  for (int r = 0; r < m.box1; ++r)
    for (int e = 0; e < m.box0; ++e) {
      const int64_t i0 = static_cast<int64_t>(c0) + e, i1 = static_cast<int64_t>(c1) + r;
      unsigned char *d = dst + (static_cast<size_t>(r) * m.box0 + e) * m.esz;
      if (i0 >= 0 && i0 < m.dim0 && i1 >= 0 && i1 < m.dim1) std::memcpy(d, m.base + i1 * m.stride1_bytes + i0 * m.esz, m.esz);
      else std::memset(d, 0, m.esz);   // out-of-bounds elements are zero-filled (and still counted)
    }
  *bytes = static_cast<long>(m.box0) * m.box1 * m.esz;
}
inline void cp_async_8(void *smem_dst, const void *gsrc, bool valid) {   // completes at once: wait_group has nothing to wait for
  if (valid) std::memcpy(smem_dst, gsrc, 8);
  else std::memset(smem_dst, 0, 8);
}
inline void cp_async_16(void *smem_dst, const void *gsrc, uint32_t src_bytes) {
  if ((reinterpret_cast<uintptr_t>(smem_dst) | reinterpret_cast<uintptr_t>(gsrc)) & 15u) std::abort();   // the hardware faults
  std::memset(smem_dst, 0, 16);
  if (src_bytes) std::memcpy(smem_dst, gsrc, src_bytes);
}
inline void cp_async_commit() {}
template <int N> inline void cp_async_wait() {}
inline void bulk_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  if ((reinterpret_cast<uintptr_t>(smem_dst) | reinterpret_cast<uintptr_t>(gsrc) | bytes) & 15u) std::abort();   // the hardware faults
  std::memcpy(smem_dst, gsrc, bytes);
  emu::mb_complete_tx(bar, bytes);
}
inline void tma_load_2d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1) {
  long bytes;
  tma_copy_box(smem_dst, map, c0, c1, &bytes);
  emu::mb_complete_tx(bar, bytes);
}

inline void tma_load_3d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1, int32_t c2) {
  long bytes;
  tma_copy_box(smem_dst, map, c0, c1, &bytes, c2);
  emu::mb_complete_tx(bar, bytes);
}

constexpr uint64_t kEvictNormal = 0x1000000000000000ull, kEvictFirst = 0x12F0000000000000ull, kEvictLast = 0x14F0000000000000ull;
inline void tma_load_2d_hint(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1, uint64_t) {
  tma_load_2d(smem_dst, map, bar, c0, c1);   // cache policies have no functional effect
}

// ------------------------------------------------------------------- wgmma
inline void wgmma_fence() {}
inline void wgmma_commit() {}
// .sync.aligned: every lane of the warp has issued (and, in this model, completed) its MMAs before any lane goes on -- lane 0
// then releases the stage for the whole warp
template <int N> inline void wgmma_wait() { pthread_barrier_wait(&emu::warp_barrier[emu::cta_rank][emu::t_idx.x >> 5]); }
inline void wgmma_hold(float (&)[64]) {}

constexpr uint32_t kLayoutSw128 = 1;
inline uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
constexpr uint32_t kFmtF16 = 0, kFmtBF16 = 1, kFmtTF32 = 2;

// one operand element as fp32: tile kept UNSWIZZLED in shared memory, addressed through the
// descriptor fields the way the canonical layouts define them:
//   K-major : row i at (i / 8) * SBO + (i % 8) * 128, k inside the 128-byte row
//   MN-major: 128-byte chunk c of the mn extent at c * LBO, k-row kk at (kk / 8) * SBO + (kk % 8) * 128
inline float operand_elem(const unsigned char *cta_smem, uint64_t desc, bool mn_major, int E, uint32_t fmt, int i, int kk) {
  const uint32_t start = static_cast<uint32_t>(desc & 0x3FFF) << 4;
  const uint32_t lbo = static_cast<uint32_t>((desc >> 16) & 0x3FFF) << 4;
  const uint32_t sbo = static_cast<uint32_t>((desc >> 32) & 0x3FFF) << 4;
  if (static_cast<uint32_t>(desc >> 62) != kLayoutSw128) { std::fprintf(stderr, "emu: descriptor without the 128B swizzle\n"); std::abort(); }
  size_t off;
  if (!mn_major) {
    off = start + static_cast<size_t>(i / 8) * sbo + static_cast<size_t>(i % 8) * 128 + static_cast<size_t>(kk) * E;
  } else {
    const int per_chunk = 128 / E;
    off = start + static_cast<size_t>(i / per_chunk) * lbo + static_cast<size_t>(kk / 8) * sbo +
          static_cast<size_t>(kk % 8) * 128 + static_cast<size_t>(i % per_chunk) * E;
  }
  if (off + E > emu::kDynSmemBytes) { std::fprintf(stderr, "emu: operand read outside shared memory\n"); std::abort(); }
  if (E == 4) {
    uint32_t u;
    std::memcpy(&u, cta_smem + off, 4);
    if (fmt == kFmtTF32) u &= 0xffffe000u;   // tf32 ignores the low 13 mantissa bits
    return __uint_as_float(u);
  }
  uint16_t h;
  std::memcpy(&h, cta_smem + off, 2);
  if (fmt == kFmtF16) {   // IEEE binary16 (subnormals included), exactly representable in fp32
    const int e = (h >> 10) & 31, m = h & 1023;
    float v;
    if (e == 0) v = std::ldexp(static_cast<float>(m), -24);
    else if (e == 31) v = m ? std::nanf("") : HUGE_VALF;
    else v = std::ldexp(static_cast<float>(1024 + m), e - 25);
    return (h & 0x8000) ? -v : v;
  }
  if (fmt != kFmtBF16) { std::fprintf(stderr, "emu: unknown 16-bit operand format\n"); std::abort(); }
  return __uint_as_float(static_cast<uint32_t>(h) << 16);
}

// D (64 x 128) (+)= A (64 x K) * B (K x 128) for one instruction (K = 32 bytes per operand row), operands from THIS CTA's
// shared memory.  Every thread of the warpgroup computes its own fragment: thread t holds rows 16 (t / 32) + (t % 32) / 4
// (+ 8) and columns 8 i + 2 (t % 4) + {0, 1}, d[4 i + 2 h + e] (ptx.cuh).
inline void wgmma_model(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d, int E, uint32_t fmt, bool a_mn, bool b_mn) {
  if (E == 4 && (a_mn || b_mn)) { std::fprintf(stderr, "emu: tf32 operands must be K-major\n"); std::abort(); }
  const unsigned t = emu::t_idx.x & 127u, w = t >> 5, lane = t & 31u;
  const unsigned char *sm = emu::dyn_smem[emu::cta_rank];
  const int KI = 32 / E;
  float a[2][16], b[32][16];
  for (int h = 0; h < 2; ++h)
    for (int kk = 0; kk < KI; ++kk) a[h][kk] = operand_elem(sm, a_desc, a_mn, E, fmt, static_cast<int>(16 * w + lane / 4 + 8 * h), kk);
  for (int i = 0; i < 16; ++i)
    for (int e = 0; e < 2; ++e)
      for (int kk = 0; kk < KI; ++kk) b[2 * i + e][kk] = operand_elem(sm, b_desc, b_mn, E, fmt, static_cast<int>(8 * i + 2 * (lane & 3) + e), kk);
  for (int i = 0; i < 16; ++i)
    for (int h = 0; h < 2; ++h)
      for (int e = 0; e < 2; ++e) {
        float &out = d[4 * i + 2 * h + e];
        double s = scale_d ? static_cast<double>(out) : 0.0;
        for (int kk = 0; kk < KI; ++kk) s += static_cast<double>(a[h][kk]) * static_cast<double>(b[2 * i + e][kk]);
        out = static_cast<float>(s);
      }
}
template <int TA, int TB>
inline void wgmma_m64n128k16_f16(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t scale_d) { wgmma_model(d, ad, bd, scale_d, 2, kFmtF16, TA, TB); }
template <int TA, int TB>
inline void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t scale_d) { wgmma_model(d, ad, bd, scale_d, 2, kFmtBF16, TA, TB); }
inline void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t scale_d) { wgmma_model(d, ad, bd, scale_d, 4, kFmtTF32, false, false); }

// ------------------------------------------------------------ clusters of two CTAs
constexpr uint32_t kPeerBitMask = 0xFEFFFFFFu;
inline uint32_t cluster_ctarank() { return emu::cta_rank; }
inline void cluster_sync() { pthread_barrier_wait(&emu::cluster_barrier); }
inline void mbar_arrive_leader(uint64_t *bar) { emu::mb_arrive(emu::peer_ptr(bar, 0), 0); }
inline void mbar_arrive_cluster(uint64_t *bar, uint32_t rank) { emu::mb_arrive(emu::peer_ptr(bar, rank), 0); }
inline void mbar_arrive_cluster_relaxed(uint64_t *bar, uint32_t rank, uint32_t count) {
  for (uint32_t i = 0; i < count; ++i) emu::mb_arrive(emu::peer_ptr(bar, rank), 0);
}
inline void mbar_wait_cluster(uint64_t *bar, uint32_t parity) { mbar_wait(bar, parity); }
inline void st_shared_cluster_s32(int *p, uint32_t rank, int v) { *reinterpret_cast<volatile int *>(emu::peer_ptr(p, rank)) = v; }
inline void griddep_wait() {}
inline void griddep_launch_dependents() {}

}  // namespace ptx
// mma.sync.aligned.m8n8k4.row.col.f64 (gemm_dmma.cuh): lane l holds A[l / 4][l % 4], B[l % 4][l / 4] and the two accumulators
// D[l / 4][2 * (l % 4) + {0, 1}]; per output element the four steps of the FMA chain in k order
inline void dmma_m8n8k4(double &d0, double &d1, double a, double b) {
  const unsigned t = emu::t_idx.x, w = t >> 5, r = emu::cta_rank, base = t & ~31u, lane = t & 31u;
  emu::warp_scratch_d[r][0][t] = a;
  emu::warp_scratch_d[r][1][t] = b;
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
  const unsigned row = lane >> 2, c0 = 2 * (lane & 3);
  for (unsigned k = 0; k < 4; ++k) {
    const double ak = emu::warp_scratch_d[r][0][base + row * 4 + k];
    d0 = std::fma(ak, emu::warp_scratch_d[r][1][base + c0 * 4 + k], d0);
    d1 = std::fma(ak, emu::warp_scratch_d[r][1][base + (c0 + 1) * 4 + k], d1);
  }
  pthread_barrier_wait(&emu::warp_barrier[r][w]);
}
}  // namespace lb200
