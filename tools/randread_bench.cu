// randread_bench.cu — what can HBM3 on an H100 deliver for the MultiGet access pattern?
// Per lookup one 32-byte sector from an `idx_mb` MB index region and one 96-byte entry (3 sectors, 32-byte aligned)
// from a `heap_mb` MB heap, 64 bytes written out coalesced.  Addresses come from a hash of the thread id.  With
// dep=0 nothing is serialised: the ceiling k_multi_get16 could approach with enough lookups in flight.  With dep=1
// the entry address depends on the index sector, as in the engine's probe.
// idx_mb = 0 skips the index read: one random access per lookup, what an always-L2-resident index would approach.
// hints = 1 loads the index sector with an L2::evict_last policy, as k_multi_get16 does, and the entry units with
// L2::evict_first, where k_multi_get16 uses plain loads (DESIGN §4 has how much of the index that keeps in L2).
// The L2 fetch granularity is set to the engine's 32 bytes (RSP_L2_FETCH_BYTES), so every random access is its own
// sector transaction.
// The default n is one bench.py MultiGet launch (8.4 M lookups).
// persist_mb > 0 sets aside that much L2 for persisting (evict_last) lines for this process
// (cudaLimitPersistingL2CacheSize, capped at the device's persistingL2CacheMaxSize); the engine sets none.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o randread_bench randread_bench.cu
//   randread_bench [heap_mb=960] [idx_mb=80] [n=8388608] [stride=96] [hints=1] [persist_mb=0]
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <algorithm>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t pol_last() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t pol_first() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
template <bool HINTS>
__device__ __forceinline__ uint4 ld(const uint4* p, uint64_t pol) {
  if (!HINTS) return __ldg(p);
  uint4 v;
  asm("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
      : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
  return v;
}
template <int LANES, bool DEP, bool HINTS>
__global__ void k(const uint4* __restrict__ heap, uint64_t heap_entries, const uint4* __restrict__ idx, uint64_t idx_sectors,
                  uint4* __restrict__ out, uint32_t n, uint64_t salt, uint32_t stride_units) {
  const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / LANES;
  const uint32_t lane = threadIdx.x % LANES;
  if (q >= n) return;
  const uint64_t pe = HINTS ? pol_first() : 0, pi = HINTS ? pol_last() : 0;
  const uint64_t r = mix(q ^ salt);
  uint64_t e = (r >> 20) % heap_entries;
  uint4 acc = make_uint4(0, 0, 0, 0);
  if (idx_sectors) {
    // index sector: 2 x 16 B
    const uint64_t is = (uint32_t)r % idx_sectors;
    uint4 s = ld<HINTS>(idx + is * 2 + (lane & 1), pi);
    if (DEP) e = (e + (s.x & 1)) % heap_entries;  // entry address depends on the index read
    acc.x = s.x ^ s.y;
  }
  // entry: 6 units of 16 B; value = units 2..5
  const uint4* ep = heap + e * stride_units;
  if (LANES == 2) {
    uint4 hd = ld<HINTS>(ep, pe), ky = ld<HINTS>(ep + 1, pe);
    uint4 v0 = ld<HINTS>(ep + 2 + lane, pe), v1 = ld<HINTS>(ep + 4 + lane, pe);
    if (hd.x == 0x12345 && ky.y == 77) v0.x ^= acc.x;
    out[(uint64_t)q * 4 + lane] = v0;
    out[(uint64_t)q * 4 + lane + 2] = v1;
  } else {  // LANES == 8: lane L loads unit L (6 used)
    uint4 u = lane < 6 ? ld<HINTS>(ep + lane, pe) : make_uint4(0, 0, 0, 0);
    if (lane >= 2 && lane < 6) out[(uint64_t)q * 4 + lane - 2] = u;
  }
}
template <int LANES, bool DEP, bool HINTS>
static void launch(uint32_t grid, int tpb, const uint4* heap, uint64_t he, const uint4* idx, uint64_t is, uint4* out,
                   uint32_t n, uint64_t salt, uint32_t su) {
  k<LANES, DEP, HINTS><<<grid, tpb>>>(heap, he, idx, is, out, n, salt, su);
}
typedef void (*launch_fn)(uint32_t, int, const uint4*, uint64_t, const uint4*, uint64_t, uint4*, uint32_t, uint64_t, uint32_t);
int main(int argc, char** argv) {
  size_t heap_mb = argc > 1 ? atoi(argv[1]) : 960, idx_mb = argc > 2 ? atoi(argv[2]) : 80;
  uint32_t n = argc > 3 ? atoi(argv[3]) : (8u << 20);
  uint32_t stride = argc > 4 ? atoi(argv[4]) : 96;  // bytes between entries: 96 = packed (half of them straddle a 128-byte line), 128 = line-aligned
  const int hints = argc > 5 ? atoi(argv[5]) : 1;
  const size_t persist_mb = argc > 6 ? atoi(argv[6]) : 0;
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  size_t persist = 0;
  if (persist_mb) {
    cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, std::min<size_t>(persist_mb << 20, prop.persistingL2CacheMaxSize));
    cudaDeviceGetLimit(&persist, cudaLimitPersistingL2CacheSize);
  }
  printf("%s: L2 %d KB, persisting set-aside %zu KB (max %d KB)\n", prop.name, prop.l2CacheSize >> 10, persist >> 10,
         prop.persistingL2CacheMaxSize >> 10);
  uint64_t heap_entries = heap_mb * 1048576ull / stride, idx_sectors = idx_mb * 1048576ull / 32;
  uint4 *heap, *idx = nullptr, *out;
  cudaMalloc(&heap, heap_entries * stride); cudaMalloc(&out, (size_t)n * 64);
  cudaMemset(heap, 1, heap_entries * stride);
  if (idx_sectors) { cudaMalloc(&idx, idx_sectors * 32); cudaMemset(idx, 2, idx_sectors * 32); }
  // [dep][lanes == 8][hints]
  const launch_fn fns[2][2][2] = {
      {{launch<2, false, false>, launch<2, false, true>}, {launch<8, false, false>, launch<8, false, true>}},
      {{launch<2, true, false>, launch<2, true, true>}, {launch<8, true, false>, launch<8, true, true>}}};
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int dep = 0; dep < 2; dep++)
    for (int lanes : {2, 8})
      for (int tpb : {256, 512}) {
        float best = 1e9;
        for (int it = 0; it < 8; it++) {  // the first two launches warm the index into L2
          cudaEventRecord(a);
          uint32_t grid = (uint32_t)(((uint64_t)n * lanes + tpb - 1) / tpb);
          fns[dep][lanes == 8][hints != 0](grid, tpb, heap, heap_entries, idx, idx_sectors, out, n, it * 7919ull, stride / 16);
          cudaEventRecord(b); cudaEventSynchronize(b);
          float ms; cudaEventElapsedTime(&ms, a, b);
          if (it >= 2 && ms < best) best = ms;
        }
        printf("dep=%d lanes=%d tpb=%d hints=%d persist=%zuMB n=%u heap=%zuMB idx=%zuMB: %.1f us -> %.2f G lookups/s, %.0f GB/s algorithmic(168B)\n",
               dep, lanes, tpb, hints, persist >> 20, n, heap_mb, idx_mb, best * 1e3, n / (best * 1e-3) / 1e9, 168.0 * n / (best * 1e-3) / 1e9);
      }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
