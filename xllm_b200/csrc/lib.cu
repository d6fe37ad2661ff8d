// Library-level plumbing of libxllm_b200_ops.so: error string, launch counter, PDL switch, SM count.
#include "common.cuh"

namespace xb {
std::atomic<uint64_t> g_launch_count{0};
std::atomic<int> g_pdl_enabled{1};
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int device_sm_count() {
  static const int sms = [] {
    int d = 0, n = 132;
    cudaGetDevice(&d);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
    return n;
  }();
  return sms;
}
}  // namespace xb

extern "C" int xb_abi_version(void) { return XB_ABI_VERSION; }
extern "C" const char* xb_last_error(void) { return xb::g_err; }
extern "C" uint64_t xb_launch_count(void) { return xb::g_launch_count.load(); }
extern "C" void xb_set_pdl(int enable) { xb::g_pdl_enabled.store(enable ? 1 : 0); }
