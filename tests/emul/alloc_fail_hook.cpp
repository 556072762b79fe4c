// TEST INFRASTRUCTURE ONLY — allocation failures on demand for the CPU emulation (alloc_failure_sweep.py).
// Preloaded (LD_PRELOAD) in front of librsp_b200_emul.so ($RSP_TEST_EMUL_LIB), it takes the place of the emulation's cudaMalloc /
// cudaHostAlloc / cudaFree, forwards to them and adds two things, exported for ctypes:
//   emul_fail_alloc_after(k)   the next k device or pinned allocations succeed, the one after fails with
//                              cudaErrorMemoryAllocation; k < 0 disarms.  emul_fail_alloc_armed(): 1 until it has fired.
//   emul_live_device_bytes()   device bytes allocated and not freed since the library was loaded.
// The engine's sources and the emulation are compiled as they are; nvcc builds never see any of this.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>

namespace {
std::mutex g_mu;
std::map<void*, size_t> g_blocks;
size_t g_live = 0;
long g_countdown = -1;

template <class F>
F next(const char* mangled) {  // the emulation's own definition (its library is loaded RTLD_LOCAL by ctypes)
  const char* path = getenv("RSP_TEST_EMUL_LIB");
  void* lib = path ? dlopen(path, RTLD_LAZY | RTLD_NOLOAD) : nullptr;
  void* f = lib ? dlsym(lib, mangled) : nullptr;
  if (!f) { fprintf(stderr, "[alloc_fail_hook] %s not found\n", mangled); abort(); }
  return reinterpret_cast<F>(f);
}
bool fire() {  // g_mu held
  return g_countdown >= 0 && g_countdown-- == 0;
}
}  // namespace

cudaError_t cudaMalloc(void** p, size_t n) {
  static auto real = next<cudaError_t (*)(void**, size_t)>("_Z10cudaMallocPPvm");
  std::lock_guard<std::mutex> g(g_mu);
  if (fire()) { *p = nullptr; return cudaErrorMemoryAllocation; }
  const cudaError_t rc = real(p, n);
  if (rc == cudaSuccess) { g_blocks[*p] = n; g_live += n; }
  return rc;
}
cudaError_t cudaFree(void* p) {
  static auto real = next<cudaError_t (*)(void*)>("_Z8cudaFreePv");
  {
    std::lock_guard<std::mutex> g(g_mu);
    auto it = g_blocks.find(p);
    if (it != g_blocks.end()) { g_live -= it->second; g_blocks.erase(it); }
  }
  return real(p);
}
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned flags) {
  static auto real = next<cudaError_t (*)(void**, size_t, unsigned)>("_Z13cudaHostAllocPPvmj");
  {
    std::lock_guard<std::mutex> g(g_mu);
    if (fire()) { *p = nullptr; return cudaErrorMemoryAllocation; }
  }
  return real(p, n, flags);
}

extern "C" void emul_fail_alloc_after(long k) {
  std::lock_guard<std::mutex> g(g_mu);
  g_countdown = k;
}
extern "C" int emul_fail_alloc_armed() {
  std::lock_guard<std::mutex> g(g_mu);
  return g_countdown >= 0;
}
extern "C" size_t emul_live_device_bytes() {
  std::lock_guard<std::mutex> g(g_mu);
  return g_live;
}
