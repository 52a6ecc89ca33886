// chainlat.cu — how many cycles does ONE link of the block-hash chain cost a lone warp?
// (chain_finalize_kernel measured ~200 cycles per link although ptxas' stall counts add up to ~115.)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I fusioninfer_b200/csrc -o tools/microbench/chainlat tools/microbench/chainlat.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "xxh64.cuh"
#include "xxh64_sm100.cuh"
using namespace fi;

// A: registers only — the bare dependency chain
__global__ void pure_chain(uint64_t* out, int links, long long* cyc) {
  uint64_t h = threadIdx.x * 0x9E3779B97F4A7C15ull + blockIdx.x;
  uint64_t pre = h ^ 0x1234567ull;
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < links; i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) h = chain_step(pre + k, h);
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = h;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// B: two independent chains per thread (does ILP help, i.e. is the chain latency- or issue-bound?)
__global__ void two_chains(uint64_t* out, int links, long long* cyc) {
  uint64_t h = threadIdx.x * 0x9E3779B97F4A7C15ull + blockIdx.x, g = ~h;
  uint64_t pre = h ^ 0x1234567ull;
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < links; i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      h = chain_step(pre + k, h);
      g = chain_step(pre - k, g);
    }
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = h ^ g;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// C: the same link written on 32-bit halves by hand, with the multiplies by constants spelled as mul.lo / mad
__device__ __forceinline__ uint64_t mul64c(uint64_t x, uint64_t c) {
  const uint32_t xl = (uint32_t)x, xh = (uint32_t)(x >> 32), cl = (uint32_t)c, ch = (uint32_t)(c >> 32);
  const uint64_t lo = (uint64_t)xl * cl;
  const uint32_t hi = (uint32_t)(lo >> 32) + xl * ch + xh * cl;
  return ((uint64_t)hi << 32) | (uint32_t)lo;
}
__device__ __forceinline__ uint64_t chain_step_manual(uint64_t pre, uint64_t prev) {
  uint64_t r = mul64c(prev, XP2);
  r = (r << 31) | (r >> 33);
  r = mul64c(r, XP1);
  uint64_t h = pre ^ r;
  h = (h << 27) | (h >> 37);
  h = mul64c(h, XP1) + XP4;
  h ^= h >> 33;
  h = mul64c(h, XP2);
  h ^= h >> 29;
  h = mul64c(h, XP3);
  h ^= h >> 32;
  return h;
}
__global__ void manual_chain(uint64_t* out, int links, long long* cyc) {
  uint64_t h = threadIdx.x * 0x9E3779B97F4A7C15ull + blockIdx.x;
  uint64_t pre = h ^ 0x1234567ull;
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < links; i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) h = chain_step_manual(pre + k, h);
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = h;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// D: the link of xxh64_sm100.cuh (IMAD.WIDE + 2 IMAD + IADD3 per product, funnel-shift rotates)
__global__ void hand_chain(uint64_t* out, int links, long long* cyc) {
  uint64_t h0 = threadIdx.x * 0x9E3779B97F4A7C15ull + blockIdx.x;
  uint64_t pre = h0 ^ 0x1234567ull;
  U2 h = u2_of(h0);
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < links; i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) h = chain_step2(u2_of(pre + k), h);
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = u64_of(h);
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
// E: the same with the serial three-IMAD product (fewer instructions, longer dependency chain)
__device__ __forceinline__ U2 chain_step2_serial(U2 pre, U2 prev) {
  const U2 z{0u, 0u};
  U2 m = mulc<XP2>(prev, z);
  m = rotl2<31>(m);
  m = mulc<XP1>(m, z);
  U2 x{pre.lo ^ m.lo, pre.hi ^ m.hi};
  x = rotl2<27>(x);
  x = mulc<XP1>(x, u2_of(XP4));
  x.lo ^= x.hi >> 1;
  x = mulc<XP2>(x, z);
  const uint32_t s_lo = __funnelshift_r(x.lo, x.hi, 29);
  x.lo ^= s_lo;
  x.hi ^= x.hi >> 29;
  x = mulc<XP3>(x, z);
  x.lo ^= x.hi;
  return x;
}
__global__ void hand_serial(uint64_t* out, int links, long long* cyc) {
  uint64_t h0 = threadIdx.x * 0x9E3779B97F4A7C15ull + blockIdx.x;
  uint64_t pre = h0 ^ 0x1234567ull;
  U2 h = u2_of(h0);
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < links; i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) h = chain_step2_serial(u2_of(pre + k), h);
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = u64_of(h);
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
// check: D and E equal A on the same inputs (printed by main)
__global__ void check_links(int* bad) {
  uint64_t h = threadIdx.x * 0x9E3779B97F4A7C15ull + 77, pre = h ^ 0x1234567ull;
  U2 a = u2_of(h), b = u2_of(h);
  for (int k = 0; k < 64; ++k) {
    h = chain_step(pre + k, h);
    a = chain_step2(u2_of(pre + k), a);
    b = chain_step2_serial(u2_of(pre + k), b);
    if (u64_of(a) != h || u64_of(b) != h) atomicAdd(bad, 1);
  }
}

template <typename K>
void run(const char* name, K kern, int grid, int block, int links) {
  uint64_t* out;
  long long* cyc;
  cudaMalloc(&out, sizeof(uint64_t) * grid * block);
  cudaMallocManaged(&cyc, sizeof(long long) * grid);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  kern<<<grid, block>>>(out, links, cyc);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  kern<<<grid, block>>>(out, links, cyc);
  cudaEventRecord(b);
  cudaDeviceSynchronize();
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  long long mx = 0;
  for (int i = 0; i < grid; ++i) mx = cyc[i] > mx ? cyc[i] : mx;
  printf("%-14s grid %4d x %4d threads, %d links: %.1f cycles/link (clock64), %.2f us wall -> %.1f ns/link\n", name, grid, block,
         links, (double)mx / links, ms * 1e3, ms * 1e6 / links);
  cudaFree(out);
  cudaFree(cyc);
}

int main() {
  const int links = 4096;
  for (int block : {32, 128, 256, 512}) {
    run("pure_chain", pure_chain, 1, block, links);
    run("pure_chain", pure_chain, 128, block, links);
  }
  run("two_chains", two_chains, 1, 32, links);
  run("two_chains", two_chains, 128, 128, links);
  run("manual_chain", manual_chain, 1, 32, links);
  run("manual_chain", manual_chain, 128, 128, links);
  for (int block : {32, 128, 256}) {
    run("hand_chain", hand_chain, 128, block, links);
    run("hand_serial", hand_serial, 128, block, links);
  }
  int* bad;
  cudaMallocManaged(&bad, sizeof(int));
  *bad = 0;
  check_links<<<1, 32>>>(bad);
  cudaDeviceSynchronize();
  printf("hand-written links vs xxh64.cuh chain_step: %d mismatches\n", *bad);
  return 0;
}
