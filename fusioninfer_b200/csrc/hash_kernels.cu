// hash_kernels.cu — batched token-block hashing for sm_90a (integer, HBM-stream bound).
//
// Computes the chained block keys of SURVEY.md Appendix A.1 (upstream
// prefix.hashPrompt; block size / cap from /root/reference/pkg/router/
// strategy.go:57-58,147-148):  h_i = XXH64(0, block_i ‖ LE64(h_{i-1})).
//
//   hash_chain    block sizes that are a multiple of 32: hashing warps compute every block's pre-state (the
//                 block_bytes/32 stripes, merge and length add — everything that does not depend on h_{i-1}) into a
//                 shared-memory ring, walker warps of the same CTA walk the chains as it fills.  32, 64 and 128
//                 bytes have their stripe count compiled in; other multiples of 32 read it at run time.
//   hash_generic  block sizes that are not a multiple of 32 (e.g. the reference's
//                 blockSize: 5): fully serial per request, byte loads.
#include "kernels.cuh"
#include "xxh64.cuh"
#include "xxh64_sm100.cuh"

namespace fi {

namespace {

// Prompt bytes are read exactly once: stream them through L2 with an evict-first policy so they
// do not push out the index rows/keys of the popular prefixes, which the match kernel re-reads
// every batch (its latency is L2-hit-rate bound, and the 50 MB L2 of an H100 holds only part of the hot set).
__device__ __forceinline__ uint64_t make_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint4 ld_stream_v4(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L1::evict_first.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;\n"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}

// one 32-byte stripe = two 16-byte loads: 128 bits is the widest global load of sm_90.  The loads allocate in L1
// (evict-first) so that the second half of each 32-byte sector is an L1 hit: with L1::no_allocate both halves went
// to L2: at cfg 3 on one H100 SXM (700 W), the earlier one-thread-per-block hashing kernel took 121-123 us that way
// against 105-107 us with these loads (one run alternating the two builds, two bench runs each).
struct Stripe {
  uint32_t w[8];
};
__device__ __forceinline__ void xacc2_stripe(XAcc2& a, const Stripe& q) {
  a.v1 = xround2(a.v1, U2{q.w[0], q.w[1]});
  a.v2 = xround2(a.v2, U2{q.w[2], q.w[3]});
  a.v3 = xround2(a.v3, U2{q.w[4], q.w[5]});
  a.v4 = xround2(a.v4, U2{q.w[6], q.w[7]});
}

__device__ __forceinline__ void st_row16(ulonglong2* p, const ulonglong2& v) {
  asm volatile("st.global.v2.u64 [%0], {%1, %2};\n" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
}
__device__ __forceinline__ ulonglong2 lds16(const ulonglong2* p) {
  ulonglong2 v;
  const unsigned sa = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];\n" : "=l"(v.x), "=l"(v.y) : "r"(sa) : "memory");
  return v;
}

// ---- hash_chain: block hashing and chain walk in one kernel --------------------------------------------------
// One CTA of WARPS warps owns a tile of 32 * WALK requests.  WARPS = 32 runs on an SM of its own (1 024 threads at 64
// registers fill the register file); WARPS = 16 is the half-SM tile, two CTAs per SM.  Warps WALK .. WARPS-1 hash the
// tile's blocks column chunk by column chunk: group g = blocks [8g, 8g+8) of
// all the tile's requests is one slot of a shared-memory ring of 8-byte pre-states, laid out [walker warp][16-byte
// unit][lane] (conflict-free for the walker).  Warps 0 .. WALK-1, on different SM sub-partitions, walk the chains of
// 32 requests each in groups of 8 links, taking the pre-states from the ring as they land.  The walk (~43 us at
// cfg 3) then runs under the tile's prompt stream (~120 us) instead of after it, and the pre-states never go to
// HBM.  Batches of up to 64 requests per SM take whole-SM tiles of 32 or 64 requests so that they still spread over
// every SM; larger ones take half-SM tiles of 64 requests (2 walkers + 14 hashers, the same 28 : 4 warps per SM as a
// whole-SM tile of 128 would have).  A half-SM CTA starts as soon as half an SM's registers are free, which matters
// when the previous batch's match_pick is draining off the SMs (pipelined submits), and 16 384 requests make 256
// CTAs over 264 slots where 128-request tiles left 4 of 132 SMs idle (launch_hash_chain; DESIGN.md §4.0).
// STRIPES = block_bytes / 32 for 32-, 64- and 128-byte blocks; STRIPES = 0 reads it from block_bytes at run time
// (every other multiple of 32).  Only the hashing lanes depend on it: the ring, the handshake and the walkers do not.
// Handshake per slot: mbarrier `full` (every hashing lane that filled part of the slot arrives; the walkers wait)
// and `empty` (every walker lane arrives once it has the slot in registers; the hashers wait before they refill it).
constexpr int kFuseRingBytesPerWarp = 1024;  // ring of 32 KiB per full-SM CTA, 16 KiB per half-SM CTA, in slots of 2 KiB per walker

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.shared::cta.b64 st, [%0];\n}\n" ::"r"(
                   (unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred p;\n"
      "WAIT_%=:\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      " @!p bra WAIT_%=;\n}\n" ::"r"((unsigned)__cvta_generic_to_shared(bar)),
      "r"(parity)
      : "memory");
}

// One stripe at byte shift sh (0, 8, .., 56) into the aligned 64-bit words wp[0..4]: funnel-shifted 8-byte loads
// (wp[4] is read only when sh != 0, where the stripe reaches into it).
__device__ __forceinline__ void xacc2_stripe_at(XAcc2& a, const uint64_t* wp, uint32_t sh) {
  uint64_t w[5];
#pragma unroll
  for (int k = 0; k < 4; ++k) w[k] = __ldg(wp + k);
  w[4] = sh ? __ldg(wp + 4) : 0;
  if (sh) {
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = (w[k] >> sh) | (w[k + 1] << (64 - sh));
  }
  xacc2_stripe(a, Stripe{{(uint32_t)w[0], (uint32_t)(w[0] >> 32), (uint32_t)w[1], (uint32_t)(w[1] >> 32),
                          (uint32_t)w[2], (uint32_t)(w[2] >> 32), (uint32_t)w[3], (uint32_t)(w[3] >> 32)}});
}

// Pre-state of one B-byte block at arbitrary byte alignment (STRIPES = 0: B / 32 stripes, counted at run time).
template <int STRIPES>
__device__ __forceinline__ uint64_t pre_unaligned(const uint8_t* blk, uint32_t B) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(blk);
  const uint64_t* wp = reinterpret_cast<const uint64_t*>(addr & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(addr & 7) * 8;
  XAcc2 a = xacc2_init();
  if constexpr (STRIPES == 0) {
    // two stripes' loads in flight: on one H100 80GB HBM3 at 400 W, cfg 3 prompts in 96- / 160-byte blocks hashed in
    // 124 / 145 us per batch this way, 135 / 167 us one stripe at a time (unrolled by 4: 134 / 144 us)
#pragma unroll 2
    for (uint32_t s = 0; s < B / 32; ++s) xacc2_stripe_at(a, wp + 4 * (uint64_t)s, sh);
  } else {
#pragma unroll
    for (int s = 0; s < STRIPES; ++s) xacc2_stripe_at(a, wp + 4 * s, sh);
  }
  return xacc2_finish(a, (uint64_t)B + 8);
}

template <int STRIPES, int WALK, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 32 / WARPS) hash_chain_kernel(const uint8_t* __restrict__ prompts,
                                                                   const uint64_t* __restrict__ offsets,
                                                                   const uint64_t* __restrict__ h0, uint32_t R,
                                                                   uint32_t M, uint32_t MP,
                                                                   uint64_t* __restrict__ chain,
                                                                   uint32_t* __restrict__ nblocks,
                                                                   uint32_t block_bytes) {
  const uint32_t B = STRIPES ? STRIPES * 32 : block_bytes;
  // A hashing warp's job: 8 blocks of 4 * BPL requests, BPL blocks per lane (two blocks' loads in flight per
  // thread, one at 128-byte blocks and at run-time stripe counts, blocks of 96 bytes or more).  Lanes 8j .. 8j+7
  // read one request's 8 blocks: 512 contiguous bytes at 64-byte blocks.
  constexpr uint32_t BPL = STRIPES == 4 || STRIPES == 0 ? 1 : 2;
  constexpr uint32_t kFuseReq = 32 * WALK;  // requests per CTA
  constexpr uint32_t kFuseHashWarps = WARPS - WALK;
  constexpr uint32_t kFuseRing = WARPS * kFuseRingBytesPerWarp / (WALK * 4 * 32 * 16);
  constexpr uint32_t kJobs = kFuseReq / (4 * BPL);  // jobs per group
  __shared__ __align__(16) ulonglong2 s_ring[kFuseRing][WALK][4][32];
  __shared__ uint64_t s_full[kFuseRing], s_empty[kFuseRing];
  __shared__ const uint8_t* s_base[kFuseReq];
  __shared__ uint32_t s_n[kFuseReq];
  __shared__ uint32_t s_groups;

  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t r_tile = blockIdx.x * kFuseReq;
  if (tid == 0) {
    s_groups = 0;
    for (uint32_t s = 0; s < kFuseRing; ++s) {
      mbar_init(&s_full[s], kJobs * 32);
      mbar_init(&s_empty[s], WALK * 32);
    }
  }
  __syncthreads();
  if (tid < kFuseReq) {
    const uint32_t r = r_tile + tid;
    uint32_t n = 0;
    const uint8_t* base = prompts;
    if (r < R) {
      const uint64_t off = offsets[r];
      const uint64_t nb64 = (offsets[r + 1] - off) / B;
      n = nb64 > M ? M : (uint32_t)nb64;
      base = prompts + off;
      nblocks[r] = n;
    }
    s_n[tid] = n;
    s_base[tid] = base;
    atomicMax(&s_groups, (n + 7) / 8);
  }
  __syncthreads();
  const uint32_t ng = s_groups;  // groups of the tile's longest request: every slot up to it is produced and consumed

  if (warp >= WALK) {
    // ---------------- hashing warps
    const uint64_t pol = make_evict_first_policy();
    const uint32_t b = lane & 7;
#pragma unroll 1
    for (uint32_t t = warp - WALK; t < ng * kJobs; t += kFuseHashWarps) {
      const uint32_t g = t / kJobs, job = t % kJobs;
      const uint32_t i = g * 8 + b;  // block index within the row
      uint32_t q[BPL];
      bool ok[BPL], al[BPL], mis = false;
      const uint8_t* src[BPL];
      uint64_t pre[BPL];
#pragma unroll
      for (uint32_t k = 0; k < BPL; ++k) {
        q[k] = job * 4 * BPL + k * 4 + (lane >> 3);
        ok[k] = i < s_n[q[k]];
        src[k] = s_base[q[k]] + (uint64_t)i * B;
        al[k] = (reinterpret_cast<uintptr_t>(src[k]) & 15) == 0;
        mis = mis || (ok[k] && !al[k]);
      }
      if constexpr (STRIPES == 0) {
        // run-time stripe count: the 8-byte path at every alignment
        if (ok[0]) pre[0] = pre_unaligned<0>(src[0], B);
      } else if (__any_sync(0xFFFFFFFFu, mis)) {
        // some prompt of the job is not 16-byte aligned: the whole warp takes the 8-byte path (it is right for
        // aligned blocks too), so the 128-bit loads below never share registers with it
#pragma unroll
        for (uint32_t k = 0; k < BPL; ++k)
          if (ok[k]) pre[k] = pre_unaligned<STRIPES>(src[k], B);
      } else {
        uint4 v[BPL][2 * STRIPES];
#pragma unroll
        for (uint32_t k = 0; k < BPL; ++k)
          if (ok[k]) {
#pragma unroll
            for (int s = 0; s < 2 * STRIPES; ++s) v[k][s] = ld_stream_v4(reinterpret_cast<const uint4*>(src[k]) + s, pol);
          }
#pragma unroll
        for (uint32_t k = 0; k < BPL; ++k)
          if (ok[k]) {
            XAcc2 a = xacc2_init();
#pragma unroll
            for (int s = 0; s < STRIPES; ++s)
              xacc2_stripe(a, Stripe{{v[k][2 * s].x, v[k][2 * s].y, v[k][2 * s].z, v[k][2 * s].w, v[k][2 * s + 1].x,
                                      v[k][2 * s + 1].y, v[k][2 * s + 1].z, v[k][2 * s + 1].w}});
            pre[k] = xacc2_finish(a, (uint64_t)B + 8);
          }
      }
      const uint32_t slot = g % kFuseRing;
      if (g >= kFuseRing) mbar_wait(&s_empty[slot], ((g / kFuseRing) + 1) & 1);  // the walkers took use g/kFuseRing - 1
      // pre-state of (request q, block b of the group): walker warp q/32, lane q%32, unit b/2, half b&1
      uint64_t* ring = reinterpret_cast<uint64_t*>(s_ring[slot]);
#pragma unroll
      for (uint32_t k = 0; k < BPL; ++k)
        if (ok[k]) ring[(((q[k] >> 5) * 4 + (b >> 1)) * 32 + (q[k] & 31)) * 2 + (b & 1)] = pre[k];
      mbar_arrive(&s_full[slot]);
    }
    return;
  }

  // ---------------- walker warps: one lane per request, h_i = chain_step(pre_i, h_{i-1}) in groups of 8 links.  The
  // walk is a pure dependency chain (5 dependent 64-bit multiplies per link).  A group's pre-states are read from
  // the ring right after its wait and its 8 hashes go straight to the lane's chain row as four 16-byte stores
  // (row-major [r][i]: what the match kernel stages and chains_out returns): the hashers set the pace here (the walk
  // alone takes less than half the time of the tile's prompt stream), and reading a group one ahead does not fit in
  // 64 registers beside the rest.  Rows are padded to whole groups (MP % 8 == 0); entries [n, MP) are zeroed.
  const uint32_t r = r_tile + warp * 32 + lane;
  const bool valid = r < R;
  const uint32_t n = s_n[warp * 32 + lane];
  uint64_t h = valid ? h0[r] : 0;
  const uint32_t MP2 = MP / 2;
  ulonglong2* out = reinterpret_cast<ulonglong2*>(chain) + (uint64_t)(valid ? r : 0) * MP2;
  uint32_t ng_full = valid ? n / 8 : 0;  // groups in which every lane of the warp has 8 blocks
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) ng_full = min(ng_full, __shfl_xor_sync(0xFFFFFFFFu, ng_full, d));

  // group g's pre-states into registers, then the slot goes back to the hashers
  ulonglong2 in[4], res[4];
  auto take = [&](uint32_t g) {
    const uint32_t slot = g % kFuseRing;
    mbar_wait(&s_full[slot], (g / kFuseRing) & 1);
#pragma unroll
    for (int k = 0; k < 4; ++k) in[k] = lds16(&s_ring[slot][warp][k][lane]);
    mbar_arrive(&s_empty[slot]);
  };

  uint32_t g = 0;
#pragma unroll 1
  for (; g < ng_full; ++g) {
    take(g);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      h = chain_step(in[k].x, h);
      res[k].x = h;
      h = chain_step(in[k].y, h);
      res[k].y = h;
    }
    ulonglong2* o = out + g * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) st_row16(o + k, res[k]);  // (ng_full > 0: every lane is valid)
  }
  // ragged groups up to the tile's longest request: some lane's chain ends inside, or has ended (zeros stored)
#pragma unroll 1
  for (; g < ng; ++g) {
    take(g);
    ulonglong2* o = out + g * 4;
    const uint32_t i0 = g * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ulonglong2 v;
      uint64_t t = chain_step(in[k].x, h);
      const bool v0 = i0 + 2 * k < n;
      h = v0 ? t : h;
      v.x = v0 ? t : 0;
      t = chain_step(in[k].y, h);
      const bool v1 = i0 + 2 * k + 1 < n;
      h = v1 ? t : h;
      v.y = v1 ? t : 0;
      if (valid) st_row16(o + k, v);
    }
  }
  if (valid) {
    const ulonglong2 z = make_ulonglong2(0, 0);
    for (uint32_t u = g * 4; u < MP2; ++u) st_row16(out + u, z);
  }
}

// Fully serial path for block sizes that are not a multiple of 32.
__global__ void __launch_bounds__(128) hash_generic_kernel(const uint8_t* __restrict__ prompts,
                                                          const uint64_t* __restrict__ offsets,
                                                          const uint64_t* __restrict__ h0, uint32_t R, uint32_t B,
                                                          uint32_t M, uint32_t MP, uint64_t* __restrict__ chain,
                                                          uint32_t* __restrict__ nblocks) {
  const uint32_t r = blockIdx.x * 128 + threadIdx.x;  // 4 warps per CTA: one per SM sub-partition
  if (r >= R) return;
  const uint64_t off = offsets[r];
  const uint64_t len = offsets[r + 1] - off;
  const uint64_t nb64 = len / B;
  const uint32_t n = nb64 > M ? M : (uint32_t)nb64;
  nblocks[r] = n;
  uint64_t* out = chain + (uint64_t)r * MP;
  uint64_t h = h0[r];
  const uint8_t* base = prompts + off;
  for (uint32_t i = 0; i < n; ++i) {
    ChainMsg m{base + (uint64_t)i * B, B, h, true};
    h = xxh64_msg(m);
    out[i] = h;
  }
  for (uint32_t i = n; i < MP; ++i) out[i] = 0;
}

}  // namespace

// One tile shape: WALK = 1 or 2 on a whole SM, or the half-SM tile (16 warps, WALK = 2).
template <int STRIPES>
static void launch_hash_chain_tile(uint32_t walk, uint32_t warps, uint32_t grid, cudaStream_t s, const uint8_t* prompts,
                                   const uint64_t* offsets, const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M,
                                   uint32_t MP, uint64_t* chain, uint32_t* nblocks) {
  if (warps == 16)
    hash_chain_kernel<STRIPES, 2, 16><<<grid, 512, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B);
  else if (walk == 2)
    hash_chain_kernel<STRIPES, 2, 32><<<grid, 1024, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B);
  else
    hash_chain_kernel<STRIPES, 1, 32><<<grid, 1024, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B);
}

cudaError_t launch_hash_chain_shape(uint32_t walk, uint32_t warps, const uint8_t* prompts, const uint64_t* offsets,
                                    const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain,
                                    uint32_t* nblocks, cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  if (!((warps == 32 && (walk == 1 || walk == 2)) || (warps == 16 && walk == 2))) return cudaErrorInvalidValue;
  const uint32_t grid = (R + 32 * walk - 1) / (32 * walk);
  if (B == 64)
    launch_hash_chain_tile<2>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  else if (B == 32)
    launch_hash_chain_tile<1>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  else if (B == 128)
    launch_hash_chain_tile<4>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  else if (B % 32 == 0)
    launch_hash_chain_tile<0>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_hash_chain(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                              uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks, int sm_count,
                              cudaStream_t s) {
  // the smallest whole-SM tile whose grid still fits one CTA per SM; half-SM tiles beyond that
  const uint32_t walk = (R + 31) / 32 > (uint32_t)sm_count ? 2 : 1;
  const uint32_t warps = (R + 63) / 64 > (uint32_t)sm_count ? 16 : 32;
  return launch_hash_chain_shape(walk, warps, prompts, offsets, h0, R, B, M, MP, chain, nblocks, s);
}

cudaError_t launch_hash_generic(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                                uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks,
                                cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  hash_generic_kernel<<<(R + 127) / 128, 128, 0, s>>>(prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  return cudaGetLastError();
}


}  // namespace fi
