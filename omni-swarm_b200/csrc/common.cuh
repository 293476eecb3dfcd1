// common.cuh -- shared plumbing of libomniswarm_b200 (error handling, launch accounting, small device helpers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/omniswarm_b200.h"

namespace osb {

extern thread_local std::string g_last_error;
extern std::atomic<long long> g_launches;

inline void set_error(const char* where, const char* what) {
  g_last_error = std::string(where) + ": " + what;
}

#define OSB_CUDA(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      char _buf[512];                                                                   \
      snprintf(_buf, sizeof(_buf), "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      osb::g_last_error = _buf;                                                         \
      return OSB_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

#define OSB_REQUIRE(cond, msg)                                                          \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      osb::set_error(__func__, msg);                                                    \
      return OSB_ERR_INVALID;                                                           \
    }                                                                                   \
  } while (0)

// every kernel launch of the library goes through this macro so that osb_launch_count() is exact
#define OSB_LAUNCH(kernel, grid, block, smem, stream, ...)                              \
  do {                                                                                  \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                         \
    osb::g_launches.fetch_add(1, std::memory_order_relaxed);                            \
  } while (0)

#define OSB_CHECK_LAUNCH() OSB_CUDA(cudaGetLastError())

// Per-DEVICE (not per-process) state: a host process may open handles on several GPUs (one nodelet per drone on the
// 8-GPU box), so "done once" flags and cached device attributes are keyed by the current device.
inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < 64) ? dev : 0;
}
// Every handle remembers the device it was created on and its entry points run there whatever the calling thread's current
// device is (a new host thread starts on device 0: the reference's nodelet calls from several spinner threads).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    int cur = 0;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != dev) { prev = cur; cudaSetDevice(dev); }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};
struct PerDeviceOnce {                     // first(dev) is true exactly once per device, thread-safe
  std::atomic<unsigned long long> mask{0};
  bool first(int dev) { return !((mask.fetch_or(1ull << dev, std::memory_order_acq_rel) >> dev) & 1ull); }
  void reset(int dev) { mask.fetch_and(~(1ull << dev), std::memory_order_acq_rel); }
};
// opt a kernel into > 48 KB of dynamic shared memory on the CURRENT device, once per device
#define OSB_SMEM_OPT_IN(kernel, bytes)                                                                      \
  do {                                                                                                      \
    static osb::PerDeviceOnce _once;                                                                        \
    const int _dev = osb::current_device();                                                                 \
    if (_once.first(_dev)) {                                                                                \
      cudaError_t _oe = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)); \
      if (_oe != cudaSuccess) { _once.reset(_dev); OSB_CUDA(_oe); }                                           \
    }                                                                                                       \
  } while (0)

inline int num_sms() {
  static std::atomic<int> cache[64];
  const int dev = current_device();
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// SM budget of the PERSISTENT kernels (one CTA per SM, statically strided tiles): such a grid only makes progress at full
// speed when every CTA is resident, so a host that runs something else on the GPU beside the front-end (the pose-graph
// solve holds 16 SMs for milliseconds) caps them with osb_set_sm_budget; 0 = all SMs.
extern std::atomic<int> g_sm_budget;
inline int persistent_ctas(int max_ctas = 0) {
  int n = num_sms();
  const int b = g_sm_budget.load(std::memory_order_relaxed);
  if (b > 0) n = std::min(n, b);
  if (max_ctas > 0) n = std::min(n, max_ctas);
  return std::max(1, n);
}

inline osb_status require_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    cudaGetLastError();
    set_error("osb", "no CUDA device visible: libomniswarm_b200 has no CPU path");
    return OSB_ERR_NO_DEVICE;
  }
  return OSB_OK;
}

template <typename T>
inline osb_status dmalloc(T** p, size_t n) {
  OSB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
  return OSB_OK;
}

// the device allocations of a handle: one cudaMalloc per buffer, every pointer remembered and freed together
struct DeviceAllocs {
  std::vector<void*> ptrs;
  template <typename T>
  osb_status alloc(T** p, size_t n) {        // n elements of T
    OSB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
    ptrs.push_back((void*)*p);
    return OSB_OK;
  }
  void free_all() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
  ~DeviceAllocs() { free_all(); }
};

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// streaming 128-bit load that does not pollute L1 (read-once data: the descriptor database)
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

}  // namespace osb
