// TEST INFRASTRUCTURE ONLY — a CPU emulation of the small slice of CUDA that rocksplicator_b200/csrc uses, so that the
// engine's host logic and the kernels' LOGIC can be exercised (and run under AddressSanitizer) on a machine without a
// GPU.  It is compiled into tests/emul/build/librsp_b200_emul.so by tests/emul/build_emul.py and loaded only by
// tests/test_emul_cpu.py.  It is not a product path and not a fallback: librsp_b200.so (the product) is CUDA-only and
// fails loudly without a device.  The only trace in the product sources is `#ifdef RSP_EMUL` alternatives next to the
// inline-PTX helpers (cache-policy loads, the TMA bulk copy + mbarrier) and the dynamic shared-memory declaration: nvcc
// never defines RSP_EMUL, and tools/sass_identity.py shows the kernels' SASS is unchanged by them.  The emulation says
// nothing about performance and nothing about memory-model races — every parity claim is made by the `-m gpu` tests
// on an H100.
//
// Execution model: a launch runs synchronously in the calling thread, block after block.  Every CUDA thread of a
// block is a fiber (ucontext); fibers run until they reach a warp collective (__shfl*_sync, __ballot_sync,
// __syncwarp), a block barrier (__syncthreads), an explicit emul_yield() or return.  A collective completes when all
// lanes named in its mask have arrived (or exited) with the same mask — arrival at different call sites is fine, as
// with independent thread scheduling.  __shared__ variables are statics (one block at a time, launches serialised).
#pragma once
#define RSP_EMUL 1
#ifndef __CUDACC__
#define __CUDACC__ 1
#endif
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static
#define __restrict__

struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct emul_idx { unsigned x, y, z; };
extern emul_idx threadIdx, blockIdx;
extern dim3 blockDim, gridDim;

// ---- runtime ------------------------------------------------------------------------------------------------
typedef int cudaError_t;
typedef struct emul_stream* cudaStream_t;
typedef struct emul_event* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyHostToHost = 0 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0, cudaHostAllocPortable = 1, cudaHostAllocMapped = 2 };
enum cudaLimit { cudaLimitMaxL2FetchGranularity = 5 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };

cudaError_t cudaGetDeviceCount(int* n);
cudaError_t cudaSetDevice(int d);
cudaError_t cudaGetDevice(int* d);
cudaError_t cudaDeviceSetLimit(cudaLimit, size_t);
cudaError_t cudaDeviceSynchronize();
cudaError_t cudaMalloc(void** p, size_t n);
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
cudaError_t cudaFree(void* p);
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned flags);
template <class T> static inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned f) { return cudaHostAlloc((void**)p, n, f); }
cudaError_t cudaFreeHost(void* p);
static inline cudaError_t cudaHostGetDevicePointer(void** d, void* h, unsigned) { *d = h; return cudaSuccess; }  // one address space
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k);
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t st = nullptr);
cudaError_t cudaMemset(void* d, int v, size_t n);
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st = nullptr);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned flags);
cudaError_t cudaStreamDestroy(cudaStream_t s);
cudaError_t cudaStreamSynchronize(cudaStream_t s);
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned flags = 0);
cudaError_t cudaEventCreate(cudaEvent_t* e);
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags);
cudaError_t cudaEventDestroy(cudaEvent_t e);
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr);
cudaError_t cudaEventSynchronize(cudaEvent_t e);
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b);
cudaError_t cudaPeekAtLastError();
cudaError_t cudaGetLastError();
const char* cudaGetErrorName(cudaError_t e);
const char* cudaGetErrorString(cudaError_t e);
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

// ---- launches: `k<<<grid, block, smem, stream>>>(args)` is rewritten to EMUL_LAUNCH by build_emul.py ------------
void emul_launch(dim3 grid, dim3 block, size_t dyn_smem, const std::function<void()>& body);
extern unsigned char* emul_dyn_smem;  // `extern __shared__` arrays
#define EMUL_LAUNCH(kernel, grid, block, smem, stream, ...) \
  emul_launch(dim3(grid), dim3(block), (size_t)(smem), [&] { kernel(__VA_ARGS__); })

// ---- warp / block collectives ----------------------------------------------------------------------------------
enum { EMUL_SHFL_IDX, EMUL_SHFL_UP, EMUL_SHFL_XOR, EMUL_BALLOT, EMUL_SYNCWARP };
uint64_t emul_collective(int op, unsigned mask, uint64_t value, unsigned arg);
void emul_syncthreads();
void emul_yield();  // inside a loop that waits for another thread
template <class T> static inline T emul_shfl(int op, unsigned mask, T v, unsigned arg) {
  static_assert(sizeof(T) <= 8, "shuffle of a type wider than 8 bytes");
  uint64_t w = 0;
  memcpy(&w, &v, sizeof(T));
  w = emul_collective(op, mask, w, arg);
  T r;
  memcpy(&r, &w, sizeof(T));
  return r;
}
template <class T> static inline T __shfl_sync(unsigned mask, T v, int lane, int = 32) { return emul_shfl(EMUL_SHFL_IDX, mask, v, (unsigned)lane); }
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned d, int = 32) { return emul_shfl(EMUL_SHFL_UP, mask, v, d); }
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int m, int = 32) { return emul_shfl(EMUL_SHFL_XOR, mask, v, (unsigned)m); }
static inline unsigned __ballot_sync(unsigned mask, int pred) { return (unsigned)emul_collective(EMUL_BALLOT, mask, pred ? 1 : 0, 0); }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, !pred) == 0; }
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emul_collective(EMUL_SYNCWARP, mask, 0, 0); }
template <class T> static inline unsigned __match_any_sync(unsigned mask, T v) {  // lanes of `mask` holding the same value
  unsigned r = 0;
  for (int l = 0; l < 32; l++)
    if ((mask >> l) & 1u) { const T o = __shfl_sync(mask, v, l); if (o == v) r |= 1u << l; }
  return r;
}
static inline void __syncthreads() { emul_syncthreads(); }
extern int emul_sync_acc;  // one block at a time, fibers are cooperative: a plain accumulator between barriers
static inline int __syncthreads_count(int pred) {
  emul_sync_acc += pred ? 1 : 0;
  emul_syncthreads();
  const int v = emul_sync_acc;
  emul_syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) emul_sync_acc = 0;
  emul_syncthreads();
  return v;
}
static inline void __threadfence() {}

// ---- loads, atomics, bit tricks -----------------------------------------------------------------------------------
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline void __stcg(T* p, T v) { *p = v; }
template <class T> struct emul_same { typedef T type; };
template <class T> static inline T atomicCAS(T* p, typename emul_same<T>::type cmp, typename emul_same<T>::type val) {
  T old = *p;
  if (old == cmp) *p = val;
  return old;
}
template <class T> static inline T atomicAdd(T* p, typename emul_same<T>::type v) { T old = *p; *p = old + v; return old; }
template <class T> static inline T atomicMax(T* p, typename emul_same<T>::type v) { T old = *p; if (v > old) *p = v; return old; }
template <class T> static inline T atomicMin(T* p, typename emul_same<T>::type v) { T old = *p; if (v < old) *p = v; return old; }
template <class T> static inline T atomicOr(T* p, typename emul_same<T>::type v) { T old = *p; *p = old | v; return old; }
template <class T> static inline T atomicExch(T* p, typename emul_same<T>::type v) { T old = *p; *p = v; return old; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline void __nanosleep(unsigned) {}
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
  const uint64_t src = ((uint64_t)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; i++) r |= (unsigned)((src >> (8 * ((s >> (4 * i)) & 7u))) & 0xffu) << (8 * i);
  return r;
}
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
using std::max;
using std::min;
static inline unsigned min(unsigned a, unsigned long b) { return (unsigned)std::min<unsigned long>(a, b); }
