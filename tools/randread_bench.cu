// randread_bench.cu — what can HBM3 on an H100 deliver for the MultiGet access pattern?
// Independent (no dependent chain) random reads: per lookup one 32-byte sector from an `idx_mb` MB index
// region and one 96-byte entry (3 sectors, 32-byte aligned) from an `heap_mb` MB heap, 64 bytes written
// out coalesced.  Addresses come from a hash of the thread id, so nothing is serialised: this is the
// ceiling the dependent-chain kernel k_multi_get16 can approach with enough lookups in flight.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o randread_bench randread_bench.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
template <int LANES, bool DEP>
__global__ void k(const uint4* __restrict__ heap, uint64_t heap_entries, const uint4* __restrict__ idx, uint64_t idx_sectors,
                  uint4* __restrict__ out, uint32_t n, uint64_t salt, uint32_t stride_units) {
  const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / LANES;
  const uint32_t lane = threadIdx.x % LANES;
  if (q >= n) return;
  const uint64_t r = mix(q ^ salt);
  uint64_t e = (r >> 20) % heap_entries;
  uint4 acc = make_uint4(0, 0, 0, 0);
  // index sector: 2 x 16 B
  const uint64_t is = (uint32_t)r % idx_sectors;
  uint4 s = __ldg(idx + is * 2 + (lane & 1));
  if (DEP) e = (e + (s.x & 1)) % heap_entries;  // entry address depends on the index read
  acc.x = s.x ^ s.y;
  // entry: 6 units of 16 B; value = units 2..5
  const uint4* ep = heap + e * stride_units;
  if (LANES == 2) {
    uint4 hd = __ldg(ep), ky = __ldg(ep + 1);
    uint4 v0 = __ldg(ep + 2 + lane), v1 = __ldg(ep + 4 + lane);
    if (hd.x == 0x12345 && ky.y == 77) v0.x ^= acc.x;
    out[(uint64_t)q * 4 + lane] = v0;
    out[(uint64_t)q * 4 + lane + 2] = v1;
  } else {  // LANES == 8: lane L loads unit L (6 used)
    uint4 u = lane < 6 ? __ldg(ep + lane) : make_uint4(0, 0, 0, 0);
    if (lane >= 2 && lane < 6) out[(uint64_t)q * 4 + lane - 2] = u;
  }
}
int main(int argc, char** argv) {
  size_t heap_mb = argc > 1 ? atoi(argv[1]) : 960, idx_mb = argc > 2 ? atoi(argv[2]) : 80;
  uint32_t n = argc > 3 ? atoi(argv[3]) : (1u << 20);
  uint32_t stride = argc > 4 ? atoi(argv[4]) : 96;  // bytes between entries: 96 = packed (half of them straddle a 128-byte line), 128 = line-aligned
  uint64_t heap_entries = heap_mb * 1048576ull / stride, idx_sectors = idx_mb * 1048576ull / 32;
  uint4 *heap, *idx, *out;
  cudaMalloc(&heap, heap_entries * stride); cudaMalloc(&idx, idx_sectors * 32); cudaMalloc(&out, (size_t)n * 64);
  cudaMemset(heap, 1, heap_entries * stride); cudaMemset(idx, 2, idx_sectors * 32);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int dep = 0; dep < 2; dep++)
    for (int lanes : {2, 8})
      for (int tpb : {256, 512}) {
        float best = 1e9;
        for (int it = 0; it < 8; it++) {
          cudaEventRecord(a);
          uint32_t grid = (uint32_t)(((uint64_t)n * lanes + tpb - 1) / tpb);
          if (lanes == 2) { if (dep) k<2, true><<<grid, tpb>>>(heap, heap_entries, idx, idx_sectors, out, n, it * 7919ull, stride / 16);
                            else k<2, false><<<grid, tpb>>>(heap, heap_entries, idx, idx_sectors, out, n, it * 7919ull, stride / 16); }
          else { if (dep) k<8, true><<<grid, tpb>>>(heap, heap_entries, idx, idx_sectors, out, n, it * 7919ull, stride / 16);
                 else k<8, false><<<grid, tpb>>>(heap, heap_entries, idx, idx_sectors, out, n, it * 7919ull, stride / 16); }
          cudaEventRecord(b); cudaEventSynchronize(b);
          float ms; cudaEventElapsedTime(&ms, a, b);
          if (it >= 2 && ms < best) best = ms;
        }
        printf("dep=%d lanes=%d tpb=%d n=%u heap=%zuMB idx=%zuMB: %.1f us -> %.2f G lookups/s, %.0f GB/s algorithmic(168B)\n", dep, lanes, tpb, n,
               heap_mb, idx_mb, best * 1e3, n / (best * 1e-3) / 1e9, 168.0 * n / (best * 1e-3) / 1e9);
      }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
