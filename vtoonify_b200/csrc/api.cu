// api.cu — error plumbing, build info, launch counter.
#include "common.cuh"
#include <atomic>
#include <string.h>

static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};

int vt_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
void vt_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int vt_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

extern "C" {
int vt_abi_version(void) { return VT_ABI_VERSION; }
const char* vt_last_error(void) { return g_err; }
const char* vt_build_info(void) {
#define VT_STR2(x) #x
#define VT_STR(x) VT_STR2(x)
  return "libvtoonify_b200 abi=" VT_STR(VT_ABI_VERSION) " arch=sm_90a cuda="
      VT_STR(__CUDACC_VER_MAJOR__) "." VT_STR(__CUDACC_VER_MINOR__) " built " __DATE__;
}
int64_t vt_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
}
