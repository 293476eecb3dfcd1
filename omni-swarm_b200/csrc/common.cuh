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

// cudaEventRecord for an event the handle's synchronising calls wait on later: inside a stream capture it becomes an
// external event-record node, so every replay of the graph records the event (a plain record in a capture is only a
// dependency edge, and the event would stay as the last uncaptured record left it)
inline cudaError_t record_event_capturable(cudaEvent_t ev, cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  const cudaError_t e = cudaStreamIsCapturing(st, &cs);
  if (e != cudaSuccess) return e;
  return cs == cudaStreamCaptureStatusActive ? cudaEventRecordWithFlags(ev, st, cudaEventRecordExternal)
                                             : cudaEventRecord(ev, st);
}
// cudaStreamWaitEvent for such an event: inside a stream capture an external event-wait node, which on every replay waits
// for the event's latest record (a plain wait on work recorded outside the capture invalidates the capture)
inline cudaError_t wait_event_capturable(cudaStream_t st, cudaEvent_t ev) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  const cudaError_t e = cudaStreamIsCapturing(st, &cs);
  if (e != cudaSuccess) return e;
  return cudaStreamWaitEvent(st, ev, cs == cudaStreamCaptureStatusActive ? cudaEventWaitExternal : 0);
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

// Host upper bound of row counts that live on the device, kept tight without a synchronisation.  The host charges every
// launch that may add rows with what it may add; the kernel publishes the true counts into mapped pinned memory, tagged with
// what had been charged when it was enqueued, so the last record that has landed gives bound = count + what was charged
// since.  seq_begin / seq_end make a torn read detectable, and a record older than min_seq (from before the counts were
// last made exact on the host) carries nothing new.
struct CountRecord {
  volatile long long seq_begin;
  volatile long long count[2];
  volatile long long status;
  volatile long long charged;
  volatile long long seq_end;
  // one thread, after the kernel's last write of the counts
  __device__ __forceinline__ void publish(long long seq, long long n0, long long n1, long long st, long long ch) {
    seq_begin = seq;
    __threadfence_system();
    count[0] = n0; count[1] = n1; status = st; charged = ch;
    __threadfence_system();
    seq_end = seq;
  }
};
struct CountFeedback {
  CountRecord* host = nullptr;                    // mapped pinned memory
  CountRecord* dev = nullptr;                     // its device alias, what the publishing kernel gets
  cudaEvent_t ev = nullptr;                       // recorded after the last publishing launch, on ITS stream
  bool pending = false;                           // that launch may not have run
  long long seq = 0, min_seq = 1;
  long long charged = 0;                          // summed over every publishing launch

  osb_status init(Resources& R) {
    OSB_TRY(R.host_alloc(&host, 1, cudaHostAllocMapped));
    memset((void*)host, 0, sizeof(CountRecord));
    OSB_CUDA(cudaHostGetDevicePointer((void**)&dev, (void*)host, 0));
    return R.event(&ev, cudaEventDisableTiming);
  }
  // charges the next publishing launch with n rows -> the sequence number it publishes (with `charged`)
  long long charge(long long n) {
    charged += n;
    return ++seq;
  }
  // after the publishing launch and whatever else the waits on `ev` must cover
  cudaError_t record(cudaStream_t st) {
    const cudaError_t e = record_event_capturable(ev, st);
    if (e == cudaSuccess) pending = true;
    return e;
  }
  // the last record that has landed: false when it is torn or older than min_seq
  bool read(long long n[2], long long* since) const {
    const long long e = host->seq_end;
    std::atomic_thread_fence(std::memory_order_acquire);
    n[0] = host->count[0]; n[1] = host->count[1];
    const long long ch = host->charged;
    std::atomic_thread_fence(std::memory_order_acquire);
    const long long b = host->seq_begin;
    *since = charged - ch;
    return b == e && e >= min_seq;
  }
  // the host's counts are exact now: no record already enqueued carries anything new
  void exact() { min_seq = seq + 1; }
};

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// What osb_anchor_sync_dev reads of a pose-graph solver's last device call (graph.cu; not part of the C ABI).  The
// pointers are device memory that the call's launches write; `done` is recorded after them, also inside a capture.
struct SolverDeviceCall {
  int device;
  int n_nodes;                            // the resident graph's node count
  int trials;                             // 0: osb_solver_solve_resident_dev, else the multistart's n_trials
  int base_res;                           // residuals of the resident factors (the tail's are word[3])
  const double* poses;                    // [n_nodes][4] x y z yaw, caller's node order
  const int32_t* word;                    // [0] status, [3] the tail's residuals
  const osb_solve_summary* summary;       // the single solve's
  const int32_t* chosen;                  // the multistart's chosen trial (-1: none)
  cudaEvent_t done;
};
// OSB_ERR_INVALID (error text set) when the solver made no device call since its last host-side pose or graph change
osb_status solver_device_call(osb_solver* h, SolverDeviceCall* out);

// A write into the solver's resident device poses from another handle's kernel (osb_anchor_add_keyframe_dev; graph.cu,
// not part of the C ABI).  solver_pose_write makes the device copy current (uploading the host mirror when the last
// change was host-side), orders `st` after the solver's last device call and marks the host mirror stale; the caller
// launches its write on `st` and then records `written` there.  The next host-side call of the solver waits for that
// event and refreshes its mirror from the device; the next device call starts from the device values.
struct SolverPoseWrite {
  int device;
  int n_nodes;                            // the resident graph's node count
  double* poses;                          // [n_nodes][4] x y z yaw, caller's node order
  cudaEvent_t written;
};
osb_status solver_pose_write(osb_solver* h, cudaStream_t st, SolverPoseWrite* out);
int solver_node_count(osb_solver* h, int* device);   // the resident graph's node count and the solver's device, without
                                                   // waiting for a device call

// good_loops_set of one unordered drone pair in a PCM state's device copy (pcm.cu): a pair with a slot, or one that
// set_inliers named.  Pair keys are (lo << 32) | hi.
struct PcmDir {
  int64_t key;
  int64_t* gptr;               // ascending ids [gn] (duplicates allowed)
  int32_t slot;                // -1: the pair has no loops
  int32_t gn;                  // -1: the pair has no set
  int32_t gcap, reserved;
};
// What osb_anchor_init_by_loops_dev reads of a PCM state (pcm.cu; not part of the C ABI): the directory of its device copy,
// which the state's anchored calls and host-side changes keep current, and the number of entries in use, read on the
// device.  `done` is recorded after the last anchored call made outside a capture (null otherwise).  OSB_ERR_INVALID
// (error text set) when the state has no device copy yet.
struct PcmDeviceDir {
  int device;
  const PcmDir* dir;
  const int32_t* n_dir;
  cudaEvent_t done;
};
osb_status pcm_device_dir(osb_pcm_state* s, PcmDeviceDir* out);

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
// Counter-based draws: a value depends only on (seed, key), not on the launch shape or the other draws.  No FMA, so numpy
// restates it bit for bit (oracle/multistart_ref.py).
__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ double counter_draw(uint64_t seed, uint64_t key, double r) {   // [-r, r)
  const double u = (double)(splitmix64(seed ^ splitmix64(key)) >> 11) * 0x1p-53;          // [0, 1)
  return __dadd_rn(__dmul_rn(2.0 * r, u), -r);
}
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
