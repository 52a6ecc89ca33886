// hash_kernels.cu — batched token-block hashing for sm_90a (integer, HBM-stream bound).
//
// Computes the chained block keys of SURVEY.md Appendix A.1 (upstream
// prefix.hashPrompt; block size / cap from /root/reference/pkg/router/
// strategy.go:57-58,147-148):  h_i = XXH64(0, block_i ‖ LE64(h_{i-1})).
//
//   hash_blocks     one thread per block: the two (block_bytes/32) stripes, merge
//                   and length add — everything that does not depend on h_{i-1}.
//                   128-bit loads, 64 B per thread, a warp covers 2 KiB contiguous.
//   chain_finalize  one thread per request walks the serial tail+avalanche link.
//   hash_chain      both in one kernel (block sizes 32, 64, 128): hashing warps fill a shared-memory ring of
//                   pre-states, walker warps of the same CTA walk the chains as it fills.
//   hash_generic    block sizes that are not a multiple of 32 (e.g. the reference's
//                   blockSize: 5): fully serial per request, byte loads.
#include "kernels.cuh"
#include "xxh64.cuh"
#include "xxh64_sm100.cuh"

namespace fi {

namespace {

__device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

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

// Pre-state layout: tiled request-minor within groups of 32 requests, in 16-byte units
// (two consecutive blocks):  unit u of request r lives at  ((r/32)*MP2 + u)*32 + r%32.
// The chain walker (one lane per request) then reads 512 contiguous bytes per warp load — 4 L1TEX
// wavefronts instead of the 32 of a row-major layout, which would saturate the wavefront rate.
__device__ __forceinline__ uint64_t pre_index(uint32_t r, uint32_t i, uint32_t MP2) {
  return ((((uint64_t)(r >> 5) * MP2 + (i >> 1)) * 32 + (r & 31)) << 1) + (i & 1);
}

// one 32-byte stripe = two 16-byte loads: 128 bits is the widest global load of sm_90.  The loads allocate in L1
// (evict-first) so that the second half of each 32-byte sector is an L1 hit: with L1::no_allocate both halves went
// to L2: at cfg 3 on one H100 SXM (700 W), hash_blocks took 121-123 us that way against 105-107 us with these
// loads (one run alternating the two builds, two bench runs each).
struct Stripe {
  uint32_t w[8];
};
__device__ __forceinline__ void xacc2_stripe(XAcc2& a, const Stripe& q) {
  a.v1 = xround2(a.v1, U2{q.w[0], q.w[1]});
  a.v2 = xround2(a.v2, U2{q.w[2], q.w[3]});
  a.v3 = xround2(a.v3, U2{q.w[4], q.w[5]});
  a.v4 = xround2(a.v4, U2{q.w[6], q.w[7]});
}

template <int STRIPES>
__global__ void __launch_bounds__(256, STRIPES <= 2 ? 8 : 5) hash_blocks_kernel(const uint8_t* __restrict__ prompts,
                                                          const uint64_t* __restrict__ offsets, uint32_t M,
                                                          uint32_t MP, uint64_t* __restrict__ pre,
                                                          uint32_t* __restrict__ nblocks) {
  constexpr uint32_t B = STRIPES * 32;
  const uint32_t MP2 = MP / 2;
  const uint64_t pol = make_evict_first_policy();
  const uint32_t r = blockIdx.x;  // one request per CTA
  const uint64_t off = offsets[r];
  const uint64_t len = offsets[r + 1] - off;
  const uint64_t nb64 = len / B;
  const uint32_t n = nb64 > M ? M : (uint32_t)nb64;
  if (threadIdx.x == 0) nblocks[r] = n;
  const uint8_t* base = prompts + off;
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(base) & 15);
  if (mis == 0) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint4* p = reinterpret_cast<const uint4*>(base + (uint64_t)i * B);
      uint4 q[2 * STRIPES];
#pragma unroll
      for (int s = 0; s < 2 * STRIPES; ++s) q[s] = ld_stream_v4(p + s, pol);
      XAcc2 a = xacc2_init();
#pragma unroll
      for (int s = 0; s < STRIPES; ++s)
        xacc2_stripe(a, Stripe{{q[2 * s].x, q[2 * s].y, q[2 * s].z, q[2 * s].w, q[2 * s + 1].x, q[2 * s + 1].y,
                                q[2 * s + 1].z, q[2 * s + 1].w}});
      pre[pre_index(r, i, MP2)] = xacc2_finish(a, (uint64_t)B + 8);
    }
  } else {
    // arbitrary byte alignment: aligned 64-bit windows + funnel shift
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uintptr_t addr = reinterpret_cast<uintptr_t>(base + (uint64_t)i * B);
      const uint64_t* wp = reinterpret_cast<const uint64_t*>(addr & ~(uintptr_t)7);
      const uint32_t sh = (uint32_t)(addr & 7) * 8;
      uint64_t w[4 * STRIPES + 1];
#pragma unroll
      for (int k = 0; k < 4 * STRIPES; ++k) w[k] = __ldg(wp + k);
      w[4 * STRIPES] = sh ? __ldg(wp + 4 * STRIPES) : 0;
      if (sh) {
#pragma unroll
        for (int k = 0; k < 4 * STRIPES; ++k) w[k] = (w[k] >> sh) | (w[k + 1] << (64 - sh));
      }
      XAcc2 a = xacc2_init();
#pragma unroll
      for (int s = 0; s < STRIPES; ++s)
        xacc2_stripe(a, Stripe{{(uint32_t)w[4 * s], (uint32_t)(w[4 * s] >> 32), (uint32_t)w[4 * s + 1],
                                (uint32_t)(w[4 * s + 1] >> 32), (uint32_t)w[4 * s + 2], (uint32_t)(w[4 * s + 2] >> 32),
                                (uint32_t)w[4 * s + 3], (uint32_t)(w[4 * s + 3] >> 32)}});
      pre[pre_index(r, i, MP2)] = xacc2_finish(a, (uint64_t)B + 8);
    }
  }
}

// any block size that is a multiple of 32 (runtime stripe count)
__global__ void __launch_bounds__(256) hash_blocks_any_kernel(const uint8_t* __restrict__ prompts,
                                                              const uint64_t* __restrict__ offsets, uint32_t B,
                                                              uint32_t M, uint32_t MP, uint64_t* __restrict__ pre,
                                                              uint32_t* __restrict__ nblocks) {
  const uint32_t r = blockIdx.x;
  const uint64_t off = offsets[r];
  const uint64_t len = offsets[r + 1] - off;
  const uint64_t nb64 = len / B;
  const uint32_t n = nb64 > M ? M : (uint32_t)nb64;
  if (threadIdx.x == 0) nblocks[r] = n;
  const uint8_t* base = prompts + off;
  const uint32_t MP2 = MP / 2;
  const uint32_t stripes = B / 32;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uintptr_t addr = reinterpret_cast<uintptr_t>(base + (uint64_t)i * B);
    const uint64_t* wp = reinterpret_cast<const uint64_t*>(addr & ~(uintptr_t)7);
    const uint32_t sh = (uint32_t)(addr & 7) * 8;
    XAcc a = xacc_init();
    uint64_t cur = __ldg(wp);
    for (uint32_t s = 0; s < stripes; ++s) {
      uint64_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (sh) {
          uint64_t nxt = __ldg(wp + 4 * s + k + 1);
          w[k] = (cur >> sh) | (nxt << (64 - sh));
          cur = nxt;
        } else {
          w[k] = __ldg(wp + 4 * s + k);
        }
      }
      xacc_stripe(a, w[0], w[1], w[2], w[3]);
    }
    pre[pre_index(r, i, MP2)] = xacc_finish(a, (uint64_t)B + 8);
  }
}

// One lane per request, one warp per group of 32 requests: h_i = chain_step(pre_i, h_{i-1}), in
// groups of 8 links.  The walk is a pure dependency chain — 5 dependent 64-bit multiplies per link — run by ONE
// warp per scheduler, in order: every other instruction in the loop and every scoreboard wait adds straight to the
// batch's critical path.  What the loop is built around:
//   * pre-states are prefetched kAhead groups ahead with cp.async into a shared-memory ring (register
//     prefetching does not work: ptxas puts every ring load on one counting scoreboard, so waiting for the
//     oldest also waits for the newest; cp.async commit/wait groups have the needed "all but the N newest"
//     semantics), and the ring is read into registers one group EARLY (volatile ld.shared at the top of the
//     iteration), so neither the wait nor the shared-memory latency sits between two links;
//   * each lane stores its 8 hashes straight to its chain row as four 16-byte stores (row-major [r][i]: what
//     the match kernel stages and chains_out returns) — but one group LATE, at the top of the next iteration,
//     from registers nothing else writes for a whole group.  Stored right after the links, the four scattered
//     STG.128 would share one set of data registers, and each would
//     have to wait for the previous one's operand read behind 32 L1 wavefronts;
//   * the loop is unrolled by two groups with the register roles swapped, so no buffer is ever copied;
//   * the buffers are padded to whole groups (MP % 8 == 0): no per-unit predicates.
// Entries [n, MP) of every row are zeroed.
// kRing ring slots, prefetch distance kRing - 1 groups, and the whole register file: there is one warp per scheduler
// when the 128 CTAs of a 16 384-request batch spread over the whole GPU, so nothing else hides the pre-state loads.

__device__ __forceinline__ void cp_async16_cg(void* smem, const void* gmem) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
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

// Four warps (128 requests) per CTA, one per SM sub-partition.
constexpr int kChainWarps = 4;
constexpr int kRing = 4;

// (the minimum of 1 CTA per SM is the register allocation the walker was measured with: 68 registers; without the
// bound ptxas allocates 66 and schedules the loop differently)
__global__ void __launch_bounds__(kChainWarps * 32, 1) chain_finalize_kernel(const uint64_t* __restrict__ pre,
                                                                       const uint32_t* __restrict__ nblocks,
                                                                       const uint64_t* __restrict__ h0, uint32_t R,
                                                                       uint32_t MP, uint64_t* __restrict__ chain) {
  constexpr int kAhead = kRing - 1;
  __shared__ __align__(16) ulonglong2 s_ring[kChainWarps][kRing][4][32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t grp = blockIdx.x * kChainWarps + warp;
  if (grp * 32 >= R) return;  // whole warp out of range (no block-wide barriers below)
  ulonglong2(*ring)[4][32] = s_ring[warp];
  const uint32_t r = grp * 32 + lane;
  const bool valid = r < R;
  const uint32_t n = valid ? nblocks[r] : 0;
  uint64_t h = valid ? h0[r] : 0;
  const uint32_t MP2 = MP / 2;  // 16-byte units per row; MP % 8 == 0: whole groups of 4 units
  const ulonglong2* p = reinterpret_cast<const ulonglong2*>(pre) + ((uint64_t)grp * MP2) * 32 + lane;  // unit u at p[u*32]
  ulonglong2* out = reinterpret_cast<ulonglong2*>(chain) + (uint64_t)(valid ? r : 0) * MP2;
  uint32_t ng_warp = (n + 7) / 8;        // groups that need arithmetic: warp-uniform maximum ...
  uint32_t ng_full = valid ? n / 8 : 0;  // ... and the groups in which every lane has 8 blocks: minimum
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    ng_warp = max(ng_warp, __shfl_xor_sync(0xFFFFFFFFu, ng_warp, d));
    ng_full = min(ng_full, __shfl_xor_sync(0xFFFFFFFFu, ng_full, d));
  }

  auto issue = [&](uint32_t g) {  // one commit group per call, empty or not: keeps the count uniform
    if (g < ng_warp) {
      ulonglong2* dst = &ring[g % kRing][0][lane];
      const ulonglong2* src = p + (uint64_t)g * 128;
#pragma unroll
      for (int k = 0; k < 4; ++k) cp_async16_cg(dst + k * 32, src + k * 32);
    }
    cp_async_commit();
  };
#pragma unroll
  for (int s = 0; s < kAhead; ++s) issue((uint32_t)s);

  ulonglong2 inA[4], inB[4], outA[4], outB[4];
  cp_async_wait<kAhead - 1>();  // group 0 has landed (a lane reads only its own copies: no barrier)
#pragma unroll
  for (int k = 0; k < 4; ++k) inA[k] = lds16(&ring[0][k][lane]);

  // one group: refill the ring, store the PREVIOUS group's hashes (if any), fetch the NEXT group's pre-states
  // into `nxt`, then the 8 links of `cur` into `res`
  auto group = [&](uint32_t g, const ulonglong2 (&cur)[4], ulonglong2 (&nxt)[4], const ulonglong2 (&prev)[4],
                   ulonglong2 (&res)[4], bool store_prev) {
    issue(g + kAhead);  // refills the slot whose registers were taken one group ago
    if (store_prev && valid) {
      ulonglong2* o = out + (g - 1) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) st_row16(o + k, prev[k]);
    }
    cp_async_wait<kAhead - 1>();  // group g + 1 has landed; its registers are needed only by the next group
#pragma unroll
    for (int k = 0; k < 4; ++k) nxt[k] = lds16(&ring[(g + 1) % kRing][k][lane]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      h = chain_step(cur[k].x, h);
      res[k].x = h;
      h = chain_step(cur[k].y, h);
      res[k].y = h;
    }
  };

  uint32_t g = 0;
  bool pending = false;  // outA / outB of group g - 1 not stored yet (which one: parity of g)
  // ---- groups in which every lane of the warp has all 8 blocks, two per iteration (A/B roles swap)
  if (ng_full >= 1) {
    group(0, inA, inB, outB, outA, false);
    g = 1;
    pending = true;
#pragma unroll 1
    for (; g + 1 < ng_full; g += 2) {
      group(g, inB, inA, outA, outB, true);
      group(g + 1, inA, inB, outB, outA, true);
    }
    if (g < ng_full) {  // one more (odd position): B in, A out
      group(g, inB, inA, outA, outB, true);
      ++g;
      // bring the roles back to "next input in inA, last output in outA"
#pragma unroll
      for (int k = 0; k < 4; ++k) outA[k] = outB[k];
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) inA[k] = inB[k];
    }
  }
  if (pending && valid) {
    ulonglong2* o = out + (g - 1) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) st_row16(o + k, outA[k]);
  }
  // ---- ragged groups: some lane's chain ends inside (next input is in inA)
#pragma unroll 1
  for (; g < ng_warp; ++g) {
    issue(g + kAhead);
    cp_async_wait<kAhead - 1>();
#pragma unroll
    for (int k = 0; k < 4; ++k) inB[k] = lds16(&ring[(g + 1) % kRing][k][lane]);
    ulonglong2* o = out + g * 4;
    const uint32_t i0 = g * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ulonglong2 v;
      uint64_t t = chain_step(inA[k].x, h);
      const bool v0 = i0 + 2 * k < n;
      h = v0 ? t : h;
      v.x = v0 ? t : 0;
      t = chain_step(inA[k].y, h);
      const bool v1 = i0 + 2 * k + 1 < n;
      h = v1 ? t : h;
      v.y = v1 ? t : 0;
      if (valid) st_row16(o + k, v);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) inA[k] = inB[k];
  }
  cp_async_wait<0>();
  // ---- the rest of every row is zero
  if (valid) {
    const ulonglong2 z = make_ulonglong2(0, 0);
    for (uint32_t u = g * 4; u < MP2; ++u) st_row16(out + u, z);
  }
}

// ---- hash_chain: hash_blocks + chain_finalize in one kernel -------------------------------------------------
// One CTA owns a tile of 32 * WALK requests and runs on an SM of its own (1 024 threads at 64 registers fill the
// register file).  Warps WALK-31 hash the tile's blocks column chunk by column chunk: group g = blocks [8g, 8g+8) of
// all the tile's requests is one slot of a shared-memory ring, laid out as chain_finalize's cp.async ring ([walker
// warp][unit][lane], conflict-free for the walker).  Warps 0 .. WALK-1, on different SM sub-partitions, walk the
// chains of 32 requests each in groups of 8 links, taking the pre-states from the ring as they land.  The walk
// (~43 us at cfg 3) then runs under the tile's prompt stream (~120 us) instead of after it, and the pre-states never
// go to HBM.  WALK = 4 (128 requests per CTA) when the batch has at least ~4 requests per 128 per SM; smaller
// batches take smaller tiles so that they still spread over every SM (launch_hash_chain).
// Handshake per slot: mbarrier `full` (every hashing lane that filled part of the slot arrives; the walkers wait)
// and `empty` (every walker lane arrives once it has the slot in registers; the hashers wait before they refill it).
constexpr int kFuseWarps = 32;           // warps 0 .. WALK-1 walk, the rest hash
constexpr int kFuseRingBytes = 32768;    // ring of 8 KiB (WALK = 4) to 2 KiB (WALK = 1) slots

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

// Pre-state of one block at arbitrary byte alignment: aligned 64-bit windows + funnel shift (hash_blocks' slow path).
template <int STRIPES>
__device__ __forceinline__ uint64_t pre_unaligned(const uint8_t* blk) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(blk);
  const uint64_t* wp = reinterpret_cast<const uint64_t*>(addr & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(addr & 7) * 8;
  XAcc2 a = xacc2_init();
#pragma unroll
  for (int s = 0; s < STRIPES; ++s) {
    uint64_t w[5];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = __ldg(wp + 4 * s + k);
    w[4] = sh ? __ldg(wp + 4 * s + 4) : 0;
    if (sh) {
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = (w[k] >> sh) | (w[k + 1] << (64 - sh));
    }
    xacc2_stripe(a, Stripe{{(uint32_t)w[0], (uint32_t)(w[0] >> 32), (uint32_t)w[1], (uint32_t)(w[1] >> 32),
                            (uint32_t)w[2], (uint32_t)(w[2] >> 32), (uint32_t)w[3], (uint32_t)(w[3] >> 32)}});
  }
  return xacc2_finish(a, (uint64_t)STRIPES * 32 + 8);
}

template <int STRIPES, int WALK>
__global__ void __launch_bounds__(kFuseWarps * 32, 1) hash_chain_kernel(const uint8_t* __restrict__ prompts,
                                                                   const uint64_t* __restrict__ offsets,
                                                                   const uint64_t* __restrict__ h0, uint32_t R,
                                                                   uint32_t M, uint32_t MP,
                                                                   uint64_t* __restrict__ chain,
                                                                   uint32_t* __restrict__ nblocks) {
  constexpr uint32_t B = STRIPES * 32;
  // A hashing warp's job: 8 blocks of 4 * BPL requests, BPL blocks per lane (two blocks' loads in flight per
  // thread, one at 128-byte blocks).  Lanes 8j .. 8j+7 read one request's 8 blocks: 512 contiguous bytes.
  constexpr uint32_t BPL = STRIPES == 4 ? 1 : 2;
  constexpr uint32_t kFuseReq = 32 * WALK;  // requests per CTA
  constexpr uint32_t kFuseHashWarps = kFuseWarps - WALK;
  constexpr uint32_t kFuseRing = kFuseRingBytes / (WALK * 4 * 32 * 16);
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
      if (__any_sync(0xFFFFFFFFu, mis)) {
        // some prompt of the job is not 16-byte aligned: the whole warp takes the 8-byte path (it is right for
        // aligned blocks too), so the 128-bit loads below never share registers with it
#pragma unroll
        for (uint32_t k = 0; k < BPL; ++k)
          if (ok[k]) pre[k] = pre_unaligned<STRIPES>(src[k]);
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

  // ---------------- walker warps: one lane per request, groups of 8 links as in chain_finalize_kernel.  A group's
  // pre-states are read from the ring right after its wait: the hashers set the pace here (the walk alone takes
  // less than half the time of the tile's prompt stream), and chain_finalize's one-group-early register copy
  // does not fit in 64 registers beside the rest.
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

cudaError_t launch_hash_blocks(const uint8_t* prompts, const uint64_t* offsets, uint32_t R, uint32_t B, uint32_t M,
                               uint32_t MP, uint64_t* pre, uint32_t* nblocks, cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  uint32_t threads = (M + 31) / 32 * 32;
  if (threads > 256) threads = 256;
  if (B == 64)
    hash_blocks_kernel<2><<<R, threads, 0, s>>>(prompts, offsets, M, MP, pre, nblocks);
  else if (B == 32)
    hash_blocks_kernel<1><<<R, threads, 0, s>>>(prompts, offsets, M, MP, pre, nblocks);
  else if (B == 128)
    hash_blocks_kernel<4><<<R, threads, 0, s>>>(prompts, offsets, M, MP, pre, nblocks);
  else
    hash_blocks_any_kernel<<<R, threads, 0, s>>>(prompts, offsets, B, M, MP, pre, nblocks);
  return cudaGetLastError();
}

cudaError_t launch_chain_finalize(const uint64_t* pre, const uint32_t* nblocks, const uint64_t* h0, uint32_t R,
                                  uint32_t MP, uint64_t* chain, cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  const uint32_t groups = (R + 31) / 32;
  const uint32_t grid = (groups + kChainWarps - 1) / kChainWarps;
  chain_finalize_kernel<<<grid, kChainWarps * 32, 0, s>>>(pre, nblocks, h0, R, MP, chain);
  return cudaGetLastError();
}

template <int STRIPES>
static void launch_hash_chain_tile(uint32_t walk, uint32_t grid, cudaStream_t s, const uint8_t* prompts,
                                   const uint64_t* offsets, const uint64_t* h0, uint32_t R, uint32_t M, uint32_t MP,
                                   uint64_t* chain, uint32_t* nblocks) {
  constexpr uint32_t threads = kFuseWarps * 32;
  if (walk == 4)
    hash_chain_kernel<STRIPES, 4><<<grid, threads, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks);
  else if (walk == 2)
    hash_chain_kernel<STRIPES, 2><<<grid, threads, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks);
  else
    hash_chain_kernel<STRIPES, 1><<<grid, threads, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks);
}

cudaError_t launch_hash_chain(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                              uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks, int sm_count,
                              cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  // the smallest tile whose grid still fits one CTA per SM; 128 requests per CTA beyond that
  uint32_t walk = 1;
  while (walk < 4 && (R + 32 * walk - 1) / (32 * walk) > (uint32_t)sm_count) walk *= 2;
  const uint32_t grid = (R + 32 * walk - 1) / (32 * walk);
  if (B == 64)
    launch_hash_chain_tile<2>(walk, grid, s, prompts, offsets, h0, R, M, MP, chain, nblocks);
  else if (B == 32)
    launch_hash_chain_tile<1>(walk, grid, s, prompts, offsets, h0, R, M, MP, chain, nblocks);
  else if (B == 128)
    launch_hash_chain_tile<4>(walk, grid, s, prompts, offsets, h0, R, M, MP, chain, nblocks);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_hash_generic(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                                uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks,
                                cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  hash_generic_kernel<<<(R + 127) / 128, 128, 0, s>>>(prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  return cudaGetLastError();
}


}  // namespace fi
