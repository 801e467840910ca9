// capi_host_prelude.h -- TEST INFRASTRUCTURE: what lets laser_b200/csrc/capi.cu -- the WHOLE host side of
// the library -- compile with g++ and run on the CPU: stand-ins for the CUDA runtime calls it makes
// ("device" memory is host memory, streams and events are no-ops because everything runs in program
// order), for cuTensorMapEncodeTiled (the arguments are kept in the opaque struct, see ptx_emu.h) and for
// kernel launches (host threads, cuda_emu.h).  tests/emu_build.py generates the translation unit: this
// prelude + capi.cu with every `kernel<<<grid, block, smem, stream>>>(args)` rewritten textually into
// `emu_launch_kernel(kernel, grid, block, smem, stream, args)`; nothing else of the source is changed.
#pragma once
#define LB200_HOST_EMULATION 1
#include "cuda_emu.h"

#include <cuda.h>
#include <cudaTypedefs.h>

#include <cstdlib>

#include "ptx_emu.h"

// ---- kernel launches ------------------------------------------------------------------------------
template <typename... KArgs, typename... Args>
inline void emu_launch_kernel(void (*kernel)(KArgs...), unsigned grid, unsigned block, size_t, cudaStream_t, Args &&...args) {
  emu::launch(grid, block, [=]() { kernel(static_cast<KArgs>(args)...); });
}
// capi_layers.inc's spelling
template <typename... KArgs, typename... Args>
inline void launch_kernel(void (*kernel)(KArgs...), unsigned grid, unsigned block, cudaStream_t s, Args &&...args) {
  emu_launch_kernel(kernel, grid, block, 0, s, static_cast<Args &&>(args)...);
}
// cudaLaunchKernelEx (the wgmma kernel; its launch attributes have no functional effect here)
template <typename... KArgs, typename... Args>
inline cudaError_t emu_launch_ex(const cudaLaunchConfig_t *cfg, void (*kernel)(KArgs...), Args &&...args) {
  if (cfg->dynamicSmemBytes > emu::kDynSmemBytes) return cudaErrorInvalidValue;
  std::lock_guard<std::recursive_mutex> device_lk(emu::launch_mu);   // reset + launch are one step of the one emulated device
  emu::reset_state();
  emu::launch(cfg->gridDim.x, cfg->blockDim.x, [=]() { kernel(static_cast<KArgs>(args)...); });
  return cudaSuccess;
}

#define LB200_LAUNCH_EX emu_launch_ex   // tc_launch_impl.cuh

// the C++ overload of cuda_runtime.h (function pointer instead of const void *) exists under nvcc only
template <typename... KArgs>
inline cudaError_t cudaFuncSetAttribute(void (*)(KArgs...), cudaFuncAttribute, int) { return cudaSuccess; }

// ---- cuTensorMapEncodeTiled ---------------------------------------------------------------------------
static CUresult emu_encode_tiled(CUtensorMap *map, CUtensorMapDataType dt, cuuint32_t rank, void *base, const cuuint64_t *dims,
                                 const cuuint64_t *strides, const cuuint32_t *box, const cuuint32_t *, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
  if (rank != 2 && rank != 3) return CUDA_ERROR_INVALID_VALUE;
  emu::TensorMap2D m;
  if (rank == 3) {
    if (box[2] != 1 || (strides[1] & 15) || dims[2] == 0) return CUDA_ERROR_INVALID_VALUE;
    m.dim2 = static_cast<int64_t>(dims[2]);
    m.stride2_bytes = static_cast<int64_t>(strides[1]);
  }
  m.magic = emu::kMapMagic;
  m.base = static_cast<const unsigned char *>(base);
  m.esz = dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
  m.dim0 = static_cast<int64_t>(dims[0]); m.dim1 = static_cast<int64_t>(dims[1]);
  m.stride1_bytes = static_cast<int64_t>(strides[0]);
  m.box0 = static_cast<int32_t>(box[0]); m.box1 = static_cast<int32_t>(box[1]);
  // the constraints the driver enforces (a violation there is CUDA_ERROR_INVALID_VALUE at run time)
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (m.stride1_bytes & 15) || m.box0 * m.esz > 128 || m.box0 > 256 || m.box1 > 256 ||
      m.dim0 <= 0 || m.dim1 <= 0)
    return CUDA_ERROR_INVALID_VALUE;
  std::memset(map, 0, sizeof *map);
  std::memcpy(map, &m, sizeof m);
  return CUDA_SUCCESS;
}

// ---- CUDA runtime ---------------------------------------------------------------------------------------
extern "C" {
// marks this build: the Python mirror refuses to load a library exporting it unless LASER_B200_EMU=1
int laser_b200_is_host_emulation(void) { return 1; }
inline int emu_device_count_sms() { const char *e = getenv("LASER_B200_EMU_SMS"); return e ? atoi(e) : 8; }
// "devices": an index per thread (one context of the library each, like real devices); how many there are comes from the test
static thread_local int emu_current_device = 0;
inline int emu_device_count() { const char *e = getenv("LASER_B200_EMU_DEVICES"); return e ? atoi(e) : 1; }
cudaError_t cudaGetDevice(int *d) { *d = emu_current_device; return cudaSuccess; }
cudaError_t cudaSetDevice(int d) {
  if (d < 0 || d >= emu_device_count()) return cudaErrorInvalidDevice;
  emu_current_device = d;
  return cudaSuccess;
}
cudaError_t cudaGetDeviceCount(int *n) { *n = emu_device_count(); return cudaSuccess; }
cudaError_t cudaGetDeviceProperties_v2(cudaDeviceProp *p, int) {
  std::memset(p, 0, sizeof *p);
  p->major = 9; p->minor = 0; p->multiProcessorCount = emu_device_count_sms();
  return cudaSuccess;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { static long n = 0x100; *s = reinterpret_cast<cudaStream_t>(n += 0x10); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void) { return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = reinterpret_cast<cudaEvent_t>(0x1); return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = reinterpret_cast<cudaEvent_t>(0x1); return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
cudaError_t cudaMalloc(void **p, size_t n) { *p = std::aligned_alloc(256, (n + 255) / 256 * 256 + 256); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFree(void *p) { std::free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { std::memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { std::memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemset(void *d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t) { return "emulated"; }
cudaError_t cudaFuncSetAttribute(const void *, cudaFuncAttribute, int) { return cudaSuccess; }
cudaError_t cudaGetDriverEntryPoint(const char *, void **fn, unsigned long long, cudaDriverEntryPointQueryResult *q) {
  *fn = reinterpret_cast<void *>(&emu_encode_tiled);
  if (q) *q = cudaDriverEntryPointSuccess;
  return cudaSuccess;
}
}
