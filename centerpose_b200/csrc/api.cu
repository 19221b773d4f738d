// Library-wide state of the centerpose_b200 C ABI (error text, launch counter, route log, version).
#include "common.cuh"

#include <cxxabi.h>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

namespace cpb {
thread_local char g_err[512] = {0};
std::atomic<unsigned long long> g_launches{0};

static std::atomic<bool> g_route_on{false};
static std::mutex g_route_mu;
static std::vector<const void *> g_route;

void note_launch(const void *kernel) {
  if (!g_route_on.load(std::memory_order_relaxed)) return;
  std::lock_guard<std::mutex> lk(g_route_mu);
  g_route.push_back(kernel);
}
}  // namespace cpb

extern "C" void cpb200_route_log_start(void) {
  std::lock_guard<std::mutex> lk(cpb::g_route_mu);
  cpb::g_route.clear();
  cpb::g_route_on.store(true);
}

extern "C" int cpb200_route_log_read(char *buf, size_t n) {
  std::vector<const void *> kernels;
  {
    std::lock_guard<std::mutex> lk(cpb::g_route_mu);
    cpb::g_route_on.store(false);
    kernels.swap(cpb::g_route);
  }
  if (!buf || n == 0) return cpb::fail(CPB200_ERR_ARG, "route_log_read: no buffer"), -1;
  size_t used = 0;
  buf[0] = '\0';
  for (const void *k : kernels) {
    const char *mangled = nullptr;
    cudaError_t e = cudaFuncGetName(&mangled, k);
    if (e != cudaSuccess || !mangled) return cpb::fail(CPB200_ERR_CUDA, "route_log_read: cudaFuncGetName: %s", cudaGetErrorString(e)), -1;
    int st = 0;
    char *dem = abi::__cxa_demangle(mangled, nullptr, nullptr, &st);
    const char *name = (st == 0 && dem) ? dem : mangled;
    const size_t len = strlen(name);
    if (used + len + 2 > n) { free(dem); return cpb::fail(CPB200_ERR_ARG, "route_log_read: buffer of %zu bytes too small", n), -1; }
    memcpy(buf + used, name, len);
    used += len;
    buf[used++] = '\n';
    buf[used] = '\0';
    free(dem);
  }
  return (int)kernels.size();
}

extern "C" int cpb200_version(void) { return 100; }
extern "C" const char *cpb200_last_error(void) { return cpb::g_err; }
extern "C" unsigned long long cpb200_launch_count(void) { return cpb::g_launches.load(); }
