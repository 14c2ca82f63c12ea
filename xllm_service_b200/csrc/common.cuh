// Shared helpers for the ingest kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <mutex>

// Error codes returned through the C-ABI (include/xllm_ingest.h mirrors these).
#define XLLM_OK 0
#define XLLM_ERR_INVALID_ARG (-1)
#define XLLM_ERR_CUDA (-2)
#define XLLM_ERR_IO (-3)
#define XLLM_ERR_FORMAT (-4)
#define XLLM_ERR_UNSUPPORTED (-5)
#define XLLM_ERR_CAPACITY (-6)
#define XLLM_ERR_NOMEM (-7)

namespace xllm {

void set_last_error(const char* fmt, ...);

#define XLLM_CUDA_TRY(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::xllm::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,               \
                             cudaGetErrorString(_e));                                    \
      return XLLM_ERR_CUDA;                                                              \
    }                                                                                    \
  } while (0)

#define XLLM_TRY_RC(expr)          \
  do {                             \
    const int _rc = (expr);        \
    if (_rc != XLLM_OK) return _rc; \
  } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_4(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// Per-device one-time kernel setup (SM count, opt-in shared memory sizes); thread-safe.
struct DeviceOnce {
  static constexpr int kMaxDevices = 64;
  std::once_flag flag[kMaxDevices];
  int n_sm[kMaxDevices] = {0};
  cudaError_t err[kMaxDevices] = {cudaSuccess};
  // runs setup() exactly once per device; returns that device's SM count (0 on error, *e set).  *device, if given, is
  // set to the current device before setup runs.
  template <typename F>
  int get(F&& setup, cudaError_t* e, int* device = nullptr) {
    int dev = 0;
    *e = cudaGetDevice(&dev);
    if (*e != cudaSuccess) return 0;
    if (device) *device = dev;
    if (dev < 0 || dev >= kMaxDevices) { *e = cudaErrorInvalidDevice; return 0; }
    std::call_once(flag[dev], [&] {
      int n = 0;
      cudaError_t r = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
      if (r == cudaSuccess) r = setup();
      n_sm[dev] = n;
      err[dev] = r;
    });
    *e = err[dev];
    return *e == cudaSuccess ? n_sm[dev] : 0;
  }
};

}  // namespace xllm
