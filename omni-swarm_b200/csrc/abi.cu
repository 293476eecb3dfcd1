// abi.cu -- library-wide state of the C ABI (error text, version, launch and resource accounting).
#include "common.cuh"

namespace osb {
thread_local std::string g_last_error;
std::atomic<long long> g_launches{0};
std::atomic<long long> g_live_resources{0};
std::atomic<int> g_sm_budget{0};
}  // namespace osb

extern "C" const char* osb_last_error(void) { return osb::g_last_error.c_str(); }
extern "C" const char* osb_version(void) { return "omniswarm_b200 0.3.0 (sm_90a)"; }
extern "C" int osb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}
extern "C" void osb_set_sm_budget(int n_sms) { osb::g_sm_budget.store(n_sms > 0 ? n_sms : 0); }
extern "C" int64_t osb_launch_count(void) { return (int64_t)osb::g_launches.load(); }
extern "C" int64_t osb_live_resources(void) { return (int64_t)osb::g_live_resources.load(); }
