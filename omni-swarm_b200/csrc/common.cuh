// common.cuh -- shared plumbing of libomniswarm_b200 (error handling, launch accounting, resource ownership, small
// device helpers).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/omniswarm_b200.h"

namespace osb {

extern thread_local std::string g_last_error;
extern std::atomic<long long> g_launches;
extern std::atomic<long long> g_live_resources;    // held by every Resources of the process (osb_live_resources)

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

// returns the status of an internal call that failed (its error text is already set)
#define OSB_TRY(expr)                                                                   \
  do {                                                                                  \
    const osb_status _s = (expr);                                                       \
    if (_s != OSB_OK) return _s;                                                        \
  } while (0)

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

// The one owner of CUDA resources: every device buffer, pinned host buffer, stream and event of a handle (or of one call)
// is acquired through it, and its destructor releases them all in reverse order of acquisition, on the device it was
// created on.  An early return therefore frees whatever was acquired so far.  Not copyable: nothing is released twice.
class Resources {
 public:
  Resources() = default;
  Resources(const Resources&) = delete;
  Resources& operator=(const Resources&) = delete;
  ~Resources() {
    if (items_.empty() && !sync_) return;
    DeviceGuard dg(device_);
    if (sync_) cudaStreamSynchronize(stream_);
    for (size_t i = items_.size(); i-- > 0;) free_item(items_[i]);
    g_live_resources.fetch_sub((long long)items_.size(), std::memory_order_relaxed);
  }
  template <typename T>
  osb_status alloc(T** p, size_t n) {        // n elements of T, one cudaMalloc
    OSB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
    hold(DEVICE, (void*)*p);
    return OSB_OK;
  }
  template <typename T>
  osb_status upload(T** p, const T* src, size_t n) {     // alloc + synchronous copy of n elements from the host
    OSB_TRY(alloc(p, n));
    OSB_CUDA(cudaMemcpy(*p, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return OSB_OK;
  }
  template <typename T>
  osb_status host_alloc(T** p, size_t n, unsigned flags) {
    OSB_CUDA(cudaHostAlloc((void**)p, n * sizeof(T), flags));
    hold(PINNED, (void*)*p);
    return OSB_OK;
  }
  osb_status stream(cudaStream_t* s, int priority = 0) {  // non-blocking
    OSB_CUDA(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority));
    hold(STREAM, *s);
    return OSB_OK;
  }
  osb_status event(cudaEvent_t* e, unsigned flags = cudaEventDefault) {
    OSB_CUDA(cudaEventCreateWithFlags(e, flags));
    hold(EVENT, *e);
    return OSB_OK;
  }
  // frees one device buffer before the owner goes (a buffer that is replaced by a larger one)
  void release(void* p) {
    for (size_t i = items_.size(); i-- > 0;)
      if (items_[i].kind == DEVICE && items_[i].p == p) {
        free_item(items_[i]);
        items_.erase(items_.begin() + i);
        g_live_resources.fetch_sub(1, std::memory_order_relaxed);
        return;
      }
  }
  // the destructor synchronises `st` before it releases anything: for operands of work launched on a caller's stream
  void sync_before_release(cudaStream_t st) { stream_ = st; sync_ = true; }

 private:
  enum Kind { DEVICE, PINNED, STREAM, EVENT };
  struct Item { Kind kind; void* p; };
  std::vector<Item> items_;
  int device_ = current_device();
  bool sync_ = false;
  cudaStream_t stream_ = nullptr;
  void hold(Kind k, void* p) {
    items_.push_back({k, p});
    g_live_resources.fetch_add(1, std::memory_order_relaxed);
  }
  static void free_item(const Item& it) {
    switch (it.kind) {
      case DEVICE: cudaFree(it.p); break;
      case PINNED: cudaFreeHost(it.p); break;
      case STREAM: cudaStreamDestroy((cudaStream_t)it.p); break;
      case EVENT: cudaEventDestroy((cudaEvent_t)it.p); break;
    }
  }
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
// the same for 4 halves (8 bytes), each converted exactly to fp32
__device__ __forceinline__ float4 ld_stream_h4(const __half* p) {
  unsigned lo, hi;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(lo), "=r"(hi) : "l"(p));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&lo));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  return make_float4(a.x, a.y, b.x, b.y);
}

}  // namespace osb
