// randread.cu — random-read throughput/latency of HBM vs table size, access size and
// parallelism: grounds the latency model of the index lookups (keys: 32 B sectors, rows: 128 B).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o randread randread.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t z) {
  z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31);
}
// each thread: ITERS rounds of DEP-independent batches of ILP random 16-byte loads (per lane or per 8-lane group)
template <int ILP, bool ROW128>
__global__ void k(const uint4* __restrict__ tab, uint64_t mask16, int iters, uint64_t seed, uint4* out, int dependent) {
  uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t s = mix(seed + (ROW128 ? tid / 8 : tid));
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (int it = 0; it < iters; ++it) {
    uint4 v[ILP];
#pragma unroll
    for (int j = 0; j < ILP; ++j) {
      uint64_t a = mix(s + j + (dependent ? acc.x : 0)) & mask16;
      if (ROW128) a = (a & ~7ull) | (threadIdx.x & 7);   // 8 lanes cover one 128-byte row
      else a = a & ~1ull;                                   // 32-byte sector aligned, first half
      v[j] = __ldg(tab + a);
    }
#pragma unroll
    for (int j = 0; j < ILP; ++j) { acc.x ^= v[j].x; acc.y += v[j].y; }
    s = mix(s + 17);
  }
  if (acc.x == 0x12345 && acc.y == 0x999) out[0] = acc;
}
int main() {
  size_t sizes[] = {64ull << 20, 256ull << 20, 1ull << 30, 4ull << 30, 16ull << 30};
  uint4* out; cudaMalloc(&out, 64);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (size_t S : sizes) {
    uint4* tab; if (cudaMalloc(&tab, S) != cudaSuccess) { printf("alloc %zu failed\n", S); continue; }
    cudaMemset(tab, 1, S);
    uint64_t mask16 = S / 16 - 1;
    for (int warps_per_sm : {8, 16, 32, 64}) {
      for (int variant = 0; variant < 4; ++variant) {
        int grid = 132 * warps_per_sm / 8, block = 256, iters = 64;
        float ms = 0; double bytes = 0; const char* name = "";
        for (int rep = 0; rep < 2; ++rep) {
          cudaEventRecord(e0);
          if (variant == 0) { k<1, false><<<grid, block>>>(tab, mask16, iters, 7 + rep, out, 1); name = "sector32 ILP1 dependent"; bytes = 32.0; }
          if (variant == 1) { k<4, false><<<grid, block>>>(tab, mask16, iters, 7 + rep, out, 0); name = "sector32 ILP4"; bytes = 32.0 * 4; }
          if (variant == 2) { k<1, true><<<grid, block>>>(tab, mask16, iters, 7 + rep, out, 1); name = "row128  ILP1 dependent"; bytes = 128.0 / 8; }
          if (variant == 3) { k<8, true><<<grid, block>>>(tab, mask16, iters, 7 + rep, out, 0); name = "row128  ILP8"; bytes = 128.0 / 8 * 8; }
          cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
        }
        double threads = (double)grid * block;
        double total = threads * iters * bytes;       // DRAM bytes moved (sector / row granularity)
        double acc_per_s = threads * iters * (variant == 1 ? 4 : variant == 3 ? 8 : 1) / (ms * 1e-3) / (variant >= 2 ? 8 : 1);
        double lat_us = (variant == 0 || variant == 2) ? ms * 1e3 / iters : 0;
        printf("table %6zu MB  warps/SM %2d  %-26s  %8.1f us  %7.1f GB/s  %7.2f G acc/s  %s%.2f us/round\n", S >> 20, warps_per_sm, name,
               ms * 1e3, total / (ms * 1e-3) / 1e9, acc_per_s / 1e9, lat_us ? "dep-lat " : "", lat_us);
      }
    }
    cudaFree(tab);
  }
  return 0;
}
