// recread.cu — does one record {32 B header | 128 B row} cost one DRAM transaction or two?
// (a) row only; (b) row + its adjacent header (same 160-byte record); (c) row + an unrelated random
// sector (today's layout: key sector in one array, row in another).  Accesses/s are per block.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t z) {
  z += 0x9E3779B97F4A7C15ULL; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31);
}
template <int MODE, int ILP>
__global__ void k(const uint4* __restrict__ tab, uint64_t nrec, uint32_t stride16, int iters, uint64_t seed, uint4* out) {
  uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t s = mix(seed + tid / 8);
  uint4 acc = make_uint4(0, 0, 0, 0);
  const uint32_t t = threadIdx.x & 7;
  for (int it = 0; it < iters; ++it) {
    uint4 v[ILP], hd[ILP];
#pragma unroll
    for (int j = 0; j < ILP; ++j) {
      uint64_t rec = mix(s + j) % nrec;
      const uint4* base = tab + rec * stride16;
      v[j] = __ldg(base + 2 + t);                          // row: 8 lanes x 16 B at offset 32
      hd[j] = make_uint4(0, 0, 0, 0);
      if (MODE == 1 && t == 0) hd[j] = __ldg(base);        // adjacent header
      if (MODE == 2 && t == 0) hd[j] = __ldg(tab + (mix(s + j + 99) % nrec) * stride16);  // unrelated sector
    }
#pragma unroll
    for (int j = 0; j < ILP; ++j) { acc.x ^= v[j].x ^ hd[j].x; acc.y += v[j].y + hd[j].y; }
    s = mix(s + 17);
  }
  if (acc.x == 0x12345 && acc.y == 0x999) out[0] = acc;
}
int main() {
  uint4* out; cudaMalloc(&out, 64);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (uint32_t stride : {160u, 256u}) {
    size_t S = 12ull << 30; uint64_t nrec = S / stride;
    uint4* tab; if (cudaMalloc(&tab, S) != cudaSuccess) { printf("alloc failed\n"); return 1; }
    cudaMemset(tab, 1, S);
    for (int wps : {16, 32, 64}) for (int mode = 0; mode < 3; ++mode) {
      int grid = 132 * wps / 8, block = 256, iters = 64; float ms = 0;
      for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0);
        if (mode == 0) k<0, 8><<<grid, block>>>(tab, nrec, stride / 16, iters, 3 + rep, out);
        if (mode == 1) k<1, 8><<<grid, block>>>(tab, nrec, stride / 16, iters, 3 + rep, out);
        if (mode == 2) k<2, 8><<<grid, block>>>(tab, nrec, stride / 16, iters, 3 + rep, out);
        cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      }
      double blocks = (double)grid * block / 8 * iters * 8;
      const char* names[] = {"row only", "row + adjacent header", "row + unrelated sector"};
      printf("stride %3u  warps/SM %2d  %-24s %8.1f us  %6.2f G blocks/s\n", stride, wps, names[mode], ms * 1e3, blocks / (ms * 1e-3) / 1e9);
    }
    cudaFree(tab);
  }
  return 0;
}
