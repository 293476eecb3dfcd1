// swarm.cu -- osb_swarm: the swarm-wide keyframe exchange behind the C ABI.
//
// Replaces LoopNet::broadcast_fisheye_desc / image_desc_callback (swarm_loop/src/loop_net.cpp:20-120,142-172 of the
// reference: one LCM header message + one message per landmark over UDP multicast, reassembled with timeouts) by ONE
// ncclAllGather of the fixed-size osb_keyframe_record per keyframe round: on the 8-GPU box the drones are ranks of one
// communicator and the records move over NVLink.  The C++ nodelet (swarm_loop/src/swarm_loop.cpp:167) calls these entry
// points directly; nothing here needs Python.
//
// NCCL is opened with dlopen at the first osb_swarm_unique_id / osb_swarm_init, so libomniswarm_b200.so has no link-time
// dependency on it (a single-drone host without NCCL can still load the library; osb_swarm_* then return OSB_ERR_INVALID
// with a message).  world == 1 needs no NCCL at all.
//
// Two transports:
//   * NCCL (osb_swarm_exchange): one ncclAllGather kernel.
//   * peer-to-peer copy engines (osb_swarm_exchange_async when the ranks can map each other's memory through CUDA IPC;
//     OSB_SWARM_P2P=0 disables it): every rank owns a double-buffered inbox [2][world] of records, exported once with
//     cudaIpcGetMemHandle.  A round is world-1 cudaMemcpyAsync pushes of the 286 KB record straight into the peers' inboxes
//     over NVLink, each followed by a 32-bit round stamp (cuMemsetD32Async) in the peer's flag table; the receiver's stream
//     waits for the stamps with cuStreamWaitValue32 and acknowledges with stamps in the senders' ack tables, which gate the
//     reuse of an inbox slot two rounds later.  No SM is used and nothing spins: an NCCL all-gather kernel that waits for a
//     late peer holds SMs that the persistent convolution CTAs of the next keyframe need (DESIGN.md section 7).
//
// The reference's exchange is asynchronous (its LCM thread delivers remote keyframes whenever they arrive, loop_net.cpp
// :142-172), so nothing forces keyframe i's gather to finish before keyframe i+1's extraction starts:
// osb_swarm_exchange_async runs the collective on the handle's own stream behind an event of the caller's stream, and
// osb_swarm_wait makes a stream wait for it -- the caller ingests round i's foreign records while round i+1 is in flight.
#include <cuda.h>
#include <dlfcn.h>
#include <nccl.h>
#include <stdlib.h>
#include "common.cuh"

namespace osb {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

static NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      api.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (api.lib) break;
    }
    if (!api.lib) return;
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.lib, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.lib, "ncclCommInitRank");
    api.AllGather = (decltype(api.AllGather))dlsym(api.lib, "ncclAllGather");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.lib, "ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.lib, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.CommDestroy || !api.GetErrorString) api.lib = nullptr;
  });
  return api.lib ? &api : nullptr;
}

#define OSB_NCCL(api, expr)                                                                   \
  do {                                                                                        \
    ncclResult_t _r = (expr);                                                                 \
    if (_r != ncclSuccess) {                                                                  \
      char _buf[512];                                                                         \
      snprintf(_buf, sizeof(_buf), "%s:%d %s -> %s", __FILE__, __LINE__, #expr, (api)->GetErrorString(_r)); \
      osb::g_last_error = _buf;                                                               \
      return OSB_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

}  // namespace osb

using namespace osb;

typedef CUresult (*PFN_streamWaitValue32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
typedef CUresult (*PFN_memsetD32Async)(CUdeviceptr, unsigned int, size_t, CUstream);

constexpr int SWARM_MAX_WORLD = 64;

struct osb_swarm {
  Resources res;                               // the side stream and the two events
  int device = 0;
  int rank = 0, world = 1;
  ncclComm_t comm = nullptr;
  cudaStream_t side = nullptr;                 // the exchange's own stream (exchange_async)
  cudaEvent_t ev_ready = nullptr, ev_done = nullptr;
  bool in_flight = false;
  std::mutex mu;
  // peer-to-peer transport
  bool p2p = false;
  uint8_t* inbox = nullptr;                    // own allocation: records [2][world], then data stamps [2][world], ack stamps [2][world]
  uint8_t* peer[SWARM_MAX_WORLD] = {};         // IPC-mapped inboxes of the other ranks (peer[rank] = inbox)
  uint32_t round = 0;                          // rounds issued so far
  osb_keyframe_record* last_gathered = nullptr;
  PFN_streamWaitValue32 wait32 = nullptr;
  PFN_memsetD32Async memset32 = nullptr;
  size_t rec_off(int b, int r) const { return ((size_t)b * world + r) * sizeof(osb_keyframe_record); }
  size_t data_off(int b, int r) const { return (size_t)2 * world * sizeof(osb_keyframe_record) + ((size_t)b * world + r) * 4; }
  size_t ack_off(int b, int r) const { return data_off(2, 0) + ((size_t)b * world + r) * 4; }
  size_t bytes() const { return ack_off(2, 0); }
};

// set up the copy-engine transport: allocate the inbox, exchange IPC handles over the NCCL communicator, map the peers
static bool swarm_setup_p2p(osb_swarm* h, NcclApi* api) {
  if (const char* e = getenv("OSB_SWARM_P2P")) if (atoi(e) == 0) return false;
  if (h->world > SWARM_MAX_WORLD) return false;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
  h->wait32 = (PFN_streamWaitValue32)fn;
  if (cudaGetDriverEntryPoint("cuMemsetD32Async", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
  h->memset32 = (PFN_memsetD32Async)fn;
  if (cudaMalloc(&h->inbox, h->bytes()) != cudaSuccess) { cudaGetLastError(); h->inbox = nullptr; return false; }
  cudaMemset(h->inbox, 0, h->bytes());
  cudaIpcMemHandle_t mine;
  bool ok = cudaIpcGetMemHandle(&mine, h->inbox) == cudaSuccess;
  // all ranks must take the same decision: gather (handle, ok) from everyone
  struct Slot { cudaIpcMemHandle_t hdl; int ok; int pad[3]; };
  Slot local; memset(&local, 0, sizeof(local)); local.hdl = mine; local.ok = ok ? 1 : 0;
  Slot* d_all = nullptr;
  std::vector<Slot> all(h->world);
  if (cudaMalloc(&d_all, h->world * sizeof(Slot)) != cudaSuccess) { cudaGetLastError(); return false; }
  cudaMemcpy(d_all + h->rank, &local, sizeof(Slot), cudaMemcpyHostToDevice);
  bool gathered = api->AllGather(d_all + h->rank, d_all, sizeof(Slot), ncclUint8, h->comm, h->side) == ncclSuccess &&
                  cudaStreamSynchronize(h->side) == cudaSuccess;
  if (gathered) cudaMemcpy(all.data(), d_all, h->world * sizeof(Slot), cudaMemcpyDeviceToHost);
  cudaFree(d_all);
  if (!gathered) { cudaGetLastError(); return false; }
  for (int r = 0; r < h->world; ++r) ok = ok && all[r].ok;
  if (ok) {
    for (int r = 0; r < h->world; ++r) {
      if (r == h->rank) { h->peer[r] = h->inbox; continue; }
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, all[r].hdl, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
      h->peer[r] = (uint8_t*)p;
    }
  }
  // second agreement round: did every rank map every peer?
  int* d_flag = nullptr;
  std::vector<int> flags(h->world, 0);
  const int mine_ok = ok ? 1 : 0;
  if (cudaMalloc(&d_flag, h->world * sizeof(int)) == cudaSuccess) {
    cudaMemcpy(d_flag + h->rank, &mine_ok, sizeof(int), cudaMemcpyHostToDevice);
    if (api->AllGather(d_flag + h->rank, d_flag, sizeof(int), ncclUint8, h->comm, h->side) == ncclSuccess &&
        cudaStreamSynchronize(h->side) == cudaSuccess)
      cudaMemcpy(flags.data(), d_flag, h->world * sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(d_flag);
  }
  for (int r = 0; r < h->world; ++r) ok = ok && flags[r];
  if (!ok) {
    for (int r = 0; r < h->world; ++r) if (r != h->rank && h->peer[r]) { cudaIpcCloseMemHandle(h->peer[r]); h->peer[r] = nullptr; }
    cudaGetLastError();
  }
  return ok;
}

static_assert(sizeof(ncclUniqueId) == OSB_SWARM_ID_BYTES, "ncclUniqueId size");

extern "C" osb_status osb_swarm_unique_id(uint8_t* id_out) {
  OSB_REQUIRE(id_out != nullptr, "null id");
  NcclApi* api = nccl_api();
  if (!api) { set_error("osb_swarm_unique_id", "libnccl.so.2 could not be opened"); return OSB_ERR_INVALID; }
  ncclUniqueId id;
  OSB_NCCL(api, api->GetUniqueId(&id));
  memcpy(id_out, &id, sizeof(id));
  return OSB_OK;
}

extern "C" osb_status osb_swarm_destroy(osb_swarm* h) {
  if (!h) return OSB_OK;
  if (h->side) cudaStreamSynchronize(h->side);
  for (int r = 0; r < SWARM_MAX_WORLD; ++r)
    if (r != h->rank && h->peer[r]) cudaIpcCloseMemHandle(h->peer[r]);
  if (h->inbox) cudaFree(h->inbox);
  if (h->comm) { NcclApi* api = nccl_api(); if (api) api->CommDestroy(h->comm); }
  delete h;
  return OSB_OK;
}

extern "C" osb_status osb_swarm_init(osb_swarm** out, const uint8_t* id, int rank, int world) {
  OSB_REQUIRE(out != nullptr && world >= 1 && rank >= 0 && rank < world, "bad rank / world");
  OSB_TRY(require_device());
  // nothing but the owner's stream and events exists until the communicator does, so an early return needs no destroy
  std::unique_ptr<osb_swarm> h(new osb_swarm());
  h->rank = rank; h->world = world;
  h->device = current_device();
  OSB_TRY(h->res.stream(&h->side));
  OSB_TRY(h->res.event(&h->ev_ready, cudaEventDisableTiming));
  OSB_TRY(h->res.event(&h->ev_done, cudaEventDisableTiming));
  if (world > 1) {
    NcclApi* api = nccl_api();
    if (!api || !id) {
      set_error("osb_swarm_init", api ? "null unique id" : "libnccl.so.2 could not be opened");
      return OSB_ERR_INVALID;
    }
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof(uid));
    ncclResult_t r = api->CommInitRank(&h->comm, world, uid, rank);
    if (r != ncclSuccess) {
      set_error("osb_swarm_init: ncclCommInitRank", api->GetErrorString(r));
      return OSB_ERR_CUDA;
    }
    h->p2p = swarm_setup_p2p(h.get(), api);
  }
  *out = h.release();
  return OSB_OK;
}

// `bytes` of every rank's src -> gathered[world * bytes] in rank order on st
static osb_status swarm_gather(osb_swarm* h, const void* src, void* gathered, size_t bytes, cudaStream_t st) {
  if (h->world == 1) {
    if (gathered != src) OSB_CUDA(cudaMemcpyAsync(gathered, src, bytes, cudaMemcpyDeviceToDevice, st));
    return OSB_OK;
  }
  NcclApi* api = nccl_api();
  OSB_NCCL(api, api->AllGather(src, gathered, bytes, ncclUint8, h->comm, st));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OSB_OK;
}

extern "C" osb_status osb_swarm_exchange(osb_swarm* h, const osb_keyframe_record* record_dev,
                                         osb_keyframe_record* gathered_dev, void* stream) {
  OSB_REQUIRE(h && record_dev && gathered_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return swarm_gather(h, record_dev, gathered_dev, sizeof(osb_keyframe_record), (cudaStream_t)stream);
}

extern "C" osb_status osb_swarm_exchange_meta(osb_swarm* h, const osb_keyframe_meta* meta_dev, osb_keyframe_meta* gathered_dev,
                                              void* stream) {
  OSB_REQUIRE(h && meta_dev && gathered_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return swarm_gather(h, meta_dev, gathered_dev, sizeof(osb_keyframe_meta), (cudaStream_t)stream);
}

extern "C" osb_status osb_swarm_exchange_async(osb_swarm* h, const osb_keyframe_record* record_dev,
                                               osb_keyframe_record* gathered_dev, void* stream) {
  OSB_REQUIRE(h && record_dev && gathered_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_CUDA(cudaEventRecord(h->ev_ready, (cudaStream_t)stream));      // the record is complete on the caller's stream
  OSB_CUDA(cudaStreamWaitEvent(h->side, h->ev_ready, 0));
  if (h->p2p) {
    // copy-engine transport: push my record into slot [b][rank] of every inbox, then its round stamp
    const uint32_t i = h->round;
    const int b = (int)(i & 1u);
    OSB_CUDA(cudaMemcpyAsync(h->inbox + h->rec_off(b, h->rank), record_dev, sizeof(osb_keyframe_record), cudaMemcpyDeviceToDevice, h->side));
    for (int k = 1; k < h->world; ++k) {
      const int p = (h->rank + k) % h->world;                         // staggered: rank r starts with r+1
      if (i >= 2) {
        // peer p acknowledged round i-2 (stamp i-1 in MY ack table) before its slot of buffer b is overwritten
        CUresult r = h->wait32((CUstream)h->side, (CUdeviceptr)(h->inbox + h->ack_off(b, p)), i - 1, CU_STREAM_WAIT_VALUE_GEQ);
        if (r != CUDA_SUCCESS) { set_error("osb_swarm_exchange_async", "cuStreamWaitValue32 failed"); return OSB_ERR_CUDA; }
      }
      OSB_CUDA(cudaMemcpyAsync(h->peer[p] + h->rec_off(b, h->rank), record_dev, sizeof(osb_keyframe_record), cudaMemcpyDeviceToDevice, h->side));
      CUresult r = h->memset32((CUdeviceptr)(h->peer[p] + h->data_off(b, h->rank)), i + 1, 1, (CUstream)h->side);
      if (r != CUDA_SUCCESS) { set_error("osb_swarm_exchange_async", "cuMemsetD32Async on peer memory failed"); return OSB_ERR_CUDA; }
    }
    OSB_CUDA(cudaEventRecord(h->ev_done, h->side));
    h->last_gathered = gathered_dev;
    h->round = i + 1;
    h->in_flight = true;
    return OSB_OK;
  }
  osb_status s = swarm_gather(h, record_dev, gathered_dev, sizeof(osb_keyframe_record), h->side);
  if (s != OSB_OK) return s;
  OSB_CUDA(cudaEventRecord(h->ev_done, h->side));
  h->in_flight = true;
  return OSB_OK;
}

extern "C" osb_status osb_swarm_wait(osb_swarm* h, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  if (!h->in_flight) return OSB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  OSB_CUDA(cudaStreamWaitEvent(st, h->ev_done, 0));
  if (h->p2p) {
    // the last round's records have arrived when every peer's stamp is there; then hand them to the caller's buffer and
    // acknowledge, which frees my slot in the peers' inboxes for the round after next
    const uint32_t i = h->round - 1;
    const int b = (int)(i & 1u);
    for (int p = 0; p < h->world; ++p) {
      if (p == h->rank) continue;
      CUresult r = h->wait32((CUstream)st, (CUdeviceptr)(h->inbox + h->data_off(b, p)), i + 1, CU_STREAM_WAIT_VALUE_GEQ);
      if (r != CUDA_SUCCESS) { set_error("osb_swarm_wait", "cuStreamWaitValue32 failed"); return OSB_ERR_CUDA; }
    }
    OSB_CUDA(cudaMemcpyAsync(h->last_gathered, h->inbox + h->rec_off(b, 0), (size_t)h->world * sizeof(osb_keyframe_record),
                             cudaMemcpyDeviceToDevice, st));
    for (int p = 0; p < h->world; ++p) {
      if (p == h->rank) continue;
      CUresult r = h->memset32((CUdeviceptr)(h->peer[p] + h->ack_off(b, h->rank)), i + 1, 1, (CUstream)st);
      if (r != CUDA_SUCCESS) { set_error("osb_swarm_wait", "cuMemsetD32Async on peer memory failed"); return OSB_ERR_CUDA; }
    }
    h->in_flight = false;
  }
  return OSB_OK;
}

extern "C" int osb_swarm_transport(osb_swarm* h) { return h ? (h->p2p ? 1 : 0) : -1; }

extern "C" int osb_swarm_rank(osb_swarm* h) { return h ? h->rank : -1; }
extern "C" int osb_swarm_world(osb_swarm* h) { return h ? h->world : -1; }
