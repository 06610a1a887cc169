// api.cu -- error plumbing, launch counter and device queries for liblmod_b200.
#include <stdarg.h>
#include <atomic>
#include "common.cuh"

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void lmod_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void lmod_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int lmod_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) sms = v;
    else { (void)cudaGetLastError(); sms = LMOD_NUM_SMS_FALLBACK; }
  }
  return sms;
}

extern "C" const char* lmod_last_error(void) { return g_err; }
extern "C" int lmod_version(void) { return 101; }
extern "C" int64_t lmod_launch_count(void) { return g_launches.load(); }
extern "C" void lmod_launch_count_reset(void) { g_launches.store(0); }
