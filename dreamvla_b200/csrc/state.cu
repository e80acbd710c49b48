// Process-wide state of libdvla_sm90.so: the thread-local error text, the launch counter and the SM budget.  Each dvla_*
// entry point is defined in the file of the op it runs.
#include <atomic>
#include <stdarg.h>
#include <stdio.h>

#include "../../include/dvla.h"
#include "host.cuh"

namespace dvla {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
static std::atomic<int> g_sm_budget{0};
// SMs the persistent kernels (one CTA, or CTA pair, per SM) may size their grids for: the device's SM count, or the
// caller's budget while a collective shares the GPU (dvla_set_sm_budget) -- a persistent grid that cannot place every CTA
// runs its stragglers as a second wave.
int num_sms() {
  static const int n = [] {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;   // H100 SXM
    return v;
  }();
  const int b = g_sm_budget.load(std::memory_order_relaxed);
  return (b > 0 && b < n) ? b : n;
}

}  // namespace dvla

using namespace dvla;

extern "C" int dvla_version(void) { return 100; }
extern "C" const char* dvla_last_error(void) { return g_err; }
extern "C" int64_t dvla_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" int dvla_set_sm_budget(int n_sms) {
  const int prev = g_sm_budget.exchange(n_sms > 0 ? (n_sms & ~1) : 0, std::memory_order_relaxed);   // even: CTA pairs
  return prev;
}
