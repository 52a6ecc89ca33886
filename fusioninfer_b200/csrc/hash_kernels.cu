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
#include "index_device.cuh"

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

// ---- early exit: hash a request only up to its first block no endpoint holds -----------------------------------
// A pick reads a request's chain up to a, its first block that no endpoint holds (match_kernels.cu
// resolve_request_nodes: both match modes stop there), plus chain[0] for the tie seed.  When nothing else reads the
// chain (no chains_out, no device-LRU Add: the host decides, engine.cu early_exit_hashing) hash_chain runs with
// MODE = kHashEarly, and one warp of the tile, the checker, looks up each request's latest stored hash in the index
// (index_find, the presence test match_pick uses).  A miss at block i proves a <= i, and i's group is already hashed,
// so the request stops after that group: hashers issue no prompt loads for its later groups and the walkers store
// zeros there.  A hit proves nothing about the blocks before it (a hole), so the request simply goes on.
// Contract: chain[r][0 .. min(n, a+1)) is the true chain, nblocks[r] = n, and every later entry is either true or 0.
// A zero never verifies in the match (key_is_special), and entries past a cannot change its walk
// (resolve_request_nodes returns at a whatever they hold), so the picks are those of the full chain.
// The checker needs no run of consecutive nodes, so an index built out of chain order stops requests as early.
enum : int { kHashFull = 0, kHashFullCounted = 1, kHashEarly = 2 };

__device__ __forceinline__ uint32_t ld_volatile_shared(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
// a chain entry a walker warp of this CTA stored (ordered by the walker's fence before it counted the group and the
// checker's after it read the count)
__device__ __forceinline__ uint64_t ld_chain_cta(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.cta.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
  return v;
}

template <int STRIPES, int WALK, int WARPS, int MODE>
__global__ void __launch_bounds__(WARPS * 32, 32 / WARPS) hash_chain_kernel(const uint8_t* __restrict__ prompts,
                                                                   const uint64_t* __restrict__ offsets,
                                                                   const uint64_t* __restrict__ h0, uint32_t R,
                                                                   uint32_t M, uint32_t MP,
                                                                   uint64_t* __restrict__ chain,
                                                                   uint32_t* __restrict__ nblocks,
                                                                   uint32_t block_bytes, const IndexView ix,
                                                                   unsigned long long* hashed) {
  constexpr bool EARLY = MODE == kHashEarly;
  const uint32_t B = STRIPES ? STRIPES * 32 : block_bytes;
  // A hashing warp's job: 8 blocks of 4 * BPL requests, BPL blocks per lane (two blocks' loads in flight per
  // thread, one at 128-byte blocks and at run-time stripe counts, blocks of 96 bytes or more).  Lanes 8j .. 8j+7
  // read one request's 8 blocks: 512 contiguous bytes at 64-byte blocks.
  constexpr uint32_t BPL = STRIPES == 4 || STRIPES == 0 ? 1 : 2;
  constexpr uint32_t kFuseReq = 32 * WALK;  // requests per CTA
  constexpr uint32_t kFuseHashWarps = WARPS - WALK - (EARLY ? 1 : 0);  // (early exit: warp WALK is the checker)
  constexpr uint32_t kFuseRing = WARPS * kFuseRingBytesPerWarp / (WALK * 4 * 32 * 16);
  constexpr uint32_t kJobs = kFuseReq / (4 * BPL);  // jobs per group
  __shared__ __align__(16) ulonglong2 s_ring[kFuseRing][WALK][4][32];
  __shared__ uint64_t s_full[kFuseRing], s_empty[kFuseRing];
  __shared__ const uint8_t* s_base[kFuseReq];
  __shared__ uint32_t s_n[kFuseReq];
  __shared__ uint32_t s_groups;
  // early exit: s_stop[q] = first group of request q not to hash (~0: none yet; written by the checker only, once);
  // s_walked[w] = groups walker warp w has stored
  // s_hashed = the tile's hashed blocks (profiling)
  __shared__ uint32_t s_stop[EARLY ? kFuseReq : 1], s_walked[EARLY ? WALK : 1], s_hashed;

  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t r_tile = blockIdx.x * kFuseReq;
  if (tid == 0) {
    s_groups = 0;
    for (uint32_t s = 0; s < kFuseRing; ++s) {
      mbar_init(&s_full[s], kJobs * 32);
      mbar_init(&s_empty[s], WALK * 32);
    }
    if constexpr (EARLY)
      for (uint32_t w = 0; w < WALK; ++w) s_walked[w] = 0;
    if constexpr (MODE != kHashFull) s_hashed = 0;
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
    if constexpr (EARLY) s_stop[tid] = 0xFFFFFFFFu;
    if constexpr (MODE == kHashFullCounted)
      if (n) atomicAdd(&s_hashed, n);
    atomicMax(&s_groups, (n + 7) / 8);
  }
  __syncthreads();
  const uint32_t ng = s_groups;  // groups of the tile's longest request: every slot up to it is produced and consumed
  if constexpr (MODE == kHashFullCounted)
    if (tid == 0 && s_hashed) atomicAdd(hashed, (unsigned long long)s_hashed);

  if constexpr (EARLY) {
    if (warp == WALK) {
      // ---------------- checker warp: lane l looks after requests l, l + 32, .. (one per walker warp).  Each round
      // probes the last stored block of every live request's latest walked group, the lane's requests in flight
      // together: one 8-byte read of the chain row, then the home bucket.  It checks the newest group rather than
      // every group so that it never falls behind the walkers by more than a round.
      uint32_t done_g[WALK];  // groups of the request already probed
      bool live[WALK];
#pragma unroll
      for (int j = 0; j < WALK; ++j) {
        done_g[j] = 0;
        live[j] = r_tile + j * 32 + lane < R && s_n[j * 32 + lane] > 0;
      }
#pragma unroll 1
      for (;;) {
        uint32_t gw[WALK];  // groups walker warp j has stored
        bool any = false, fresh = false;
#pragma unroll
        for (int j = 0; j < WALK; ++j) {
          gw[j] = ld_volatile_shared(&s_walked[j]);
          live[j] = live[j] && done_g[j] * 8 < s_n[j * 32 + lane];  // not yet stored in full
          any = any || live[j];
          fresh = fresh || (live[j] && gw[j] > done_g[j]);
        }
        if (!__any_sync(0xFFFFFFFFu, any)) break;
        if (!__any_sync(0xFFFFFFFFu, fresh)) {
          __nanosleep(64);
          continue;
        }
        __threadfence_block();
        uint64_t hk[WALK];
#pragma unroll
        for (int j = 0; j < WALK; ++j) {
          const uint32_t q = j * 32 + lane;
          hk[j] = 0;
          if (live[j] && gw[j] > done_g[j]) {
            const uint32_t i = min(gw[j] * 8, s_n[q]) - 1;  // last stored block
            hk[j] = ld_chain_cta(chain + (uint64_t)(r_tile + q) * MP + i);
          }
        }
#pragma unroll
        for (int j = 0; j < WALK; ++j) {
          const uint32_t q = j * 32 + lane;
          if (live[j] && gw[j] > done_g[j]) {
            if (index_find(ix, hk[j]) == SLOT_MISS) {  // a <= the probed block, whose group gw - 1 is hashed
              *reinterpret_cast<volatile uint32_t*>(&s_stop[q]) = gw[j];
              live[j] = false;
            }
            done_g[j] = gw[j];
          }
        }
      }
      return;
    }
  }

  if (warp >= WALK) {
    // ---------------- hashing warps
    const uint64_t pol = make_evict_first_policy();
    const uint32_t b = lane & 7;
#pragma unroll 1
    for (uint32_t t = warp - WALK - (EARLY ? 1 : 0); t < ng * kJobs; t += kFuseHashWarps) {
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
        if constexpr (EARLY) ok[k] = ok[k] && g < ld_volatile_shared(&s_stop[q[k]]);
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
      if constexpr (EARLY) {
        if (hashed) {  // profiling: the job's hashed blocks (counted before the arrive: the walkers add them up)
          uint32_t c = 0;
#pragma unroll
          for (uint32_t k = 0; k < BPL; ++k) c += __popc(__ballot_sync(0xFFFFFFFFu, ok[k]));
          if (lane == 0) atomicAdd(&s_hashed, c);
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

  // early exit: the group's hashes are in the row; tell the checker (the fence orders every lane's stores before the
  // count, __syncwarp the other lanes' before lane 0's fence)
  auto publish = [&](uint32_t g) {
    if constexpr (EARLY) {
      __syncwarp();
      if (lane == 0) {
        __threadfence_block();
        *reinterpret_cast<volatile uint32_t*>(&s_walked[warp]) = g + 1;
      }
    }
  };
  // early exit: false once the checker stopped this request before group g.  Read after take(g): every hasher of
  // the group read s_stop before it arrived, so a stop they saw is seen here too and the ring's stale entries of a
  // stopped request are never stored (a stop they missed only costs the group's hashing).
  auto hashed_group = [&](uint32_t g) { return !EARLY || g < ld_volatile_shared(&s_stop[warp * 32 + lane]); };

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
    if constexpr (EARLY) {
      if (!hashed_group(g))  // (h goes on over the ring's stale entries: it is never stored again)
#pragma unroll
        for (int k = 0; k < 4; ++k) res[k] = make_ulonglong2(0, 0);
    }
    ulonglong2* o = out + g * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) st_row16(o + k, res[k]);  // (ng_full > 0: every lane is valid)
    publish(g);
  }
  // ragged groups up to the tile's longest request: some lane's chain ends inside, or has ended (zeros stored)
#pragma unroll 1
  for (; g < ng; ++g) {
    take(g);
    ulonglong2* o = out + g * 4;
    const uint32_t i0 = g * 8;
    const bool hg = hashed_group(g);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ulonglong2 v;
      uint64_t t = chain_step(in[k].x, h);
      const bool v0 = i0 + 2 * k < n && hg;
      h = v0 ? t : h;
      v.x = v0 ? t : 0;
      t = chain_step(in[k].y, h);
      const bool v1 = i0 + 2 * k + 1 < n && hg;
      h = v1 ? t : h;
      v.y = v1 ? t : 0;
      if (valid) st_row16(o + k, v);
    }
    publish(g);
  }
  if (valid) {
    const ulonglong2 z = make_ulonglong2(0, 0);
    for (uint32_t u = g * 4; u < MP2; ++u) st_row16(out + u, z);
  }
  if constexpr (EARLY) {
    // every job arrived on its full barrier after counting, and this warp has waited on all of them
    if (hashed && warp == 0 && lane == 0 && s_hashed) atomicAdd(hashed, (unsigned long long)s_hashed);
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
template <int STRIPES, int MODE>
static void launch_hash_chain_tile(uint32_t walk, uint32_t warps, uint32_t grid, cudaStream_t s, const uint8_t* prompts,
                                   const uint64_t* offsets, const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M,
                                   uint32_t MP, uint64_t* chain, uint32_t* nblocks, const IndexView& ix,
                                   unsigned long long* hashed) {
  if (warps == 16)
    hash_chain_kernel<STRIPES, 2, 16, MODE><<<grid, 512, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B, ix, hashed);
  else if (walk == 2)
    hash_chain_kernel<STRIPES, 2, 32, MODE><<<grid, 1024, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B, ix, hashed);
  else
    hash_chain_kernel<STRIPES, 1, 32, MODE><<<grid, 1024, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B, ix, hashed);
}

// Early exit runs in half-SM tiles only.  A whole-SM tile's ring is 8 or 16 groups deep (64 or 128 blocks), so its
// hashers run that far ahead of the walkers and the checker, and the warp the checker takes costs more than the
// stops save: at cfg 2 (4 096 requests of 128 blocks, whole-SM tiles of 32) the stream-ordered step took 49.6-50.3 us
// with early exit against 49.1-49.3 us without (one H100 80GB HBM3 at 700 W, three runs of each alternated).
template <int STRIPES>
static void launch_hash_chain_mode(uint32_t walk, uint32_t warps, uint32_t grid, cudaStream_t s, const uint8_t* prompts,
                                   const uint64_t* offsets, const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M,
                                   uint32_t MP, uint64_t* chain, uint32_t* nblocks, const IndexView* early,
                                   unsigned long long* hashed) {
  if (early && warps == 16)
    hash_chain_kernel<STRIPES, 2, 16, kHashEarly><<<grid, 512, 0, s>>>(prompts, offsets, h0, R, M, MP, chain, nblocks, B,
                                                                        *early, hashed);
  else if (hashed)
    launch_hash_chain_tile<STRIPES, kHashFullCounted>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks,
                                                      IndexView{}, hashed);
  else
    launch_hash_chain_tile<STRIPES, kHashFull>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks,
                                               IndexView{}, nullptr);
}

cudaError_t launch_hash_chain_shape(uint32_t walk, uint32_t warps, const uint8_t* prompts, const uint64_t* offsets,
                                    const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain,
                                    uint32_t* nblocks, cudaStream_t s, const IndexView* early, unsigned long long* hashed) {
  if (R == 0) return cudaSuccess;
  if (!((warps == 32 && (walk == 1 || walk == 2)) || (warps == 16 && walk == 2))) return cudaErrorInvalidValue;
  const uint32_t grid = (R + 32 * walk - 1) / (32 * walk);
  if (B == 64)
    launch_hash_chain_mode<2>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks, early, hashed);
  else if (B == 32)
    launch_hash_chain_mode<1>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks, early, hashed);
  else if (B == 128)
    launch_hash_chain_mode<4>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks, early, hashed);
  else if (B % 32 == 0)
    launch_hash_chain_mode<0>(walk, warps, grid, s, prompts, offsets, h0, R, B, M, MP, chain, nblocks, early, hashed);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_hash_chain(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                              uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks, int sm_count,
                              cudaStream_t s, const IndexView* early, unsigned long long* hashed) {
  // the smallest whole-SM tile whose grid still fits one CTA per SM; half-SM tiles beyond that
  const uint32_t walk = (R + 31) / 32 > (uint32_t)sm_count ? 2 : 1;
  const uint32_t warps = (R + 63) / 64 > (uint32_t)sm_count ? 16 : 32;
  return launch_hash_chain_shape(walk, warps, prompts, offsets, h0, R, B, M, MP, chain, nblocks, s, early, hashed);
}

cudaError_t launch_hash_generic(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                                uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks,
                                cudaStream_t s) {
  if (R == 0) return cudaSuccess;
  hash_generic_kernel<<<(R + 127) / 128, 128, 0, s>>>(prompts, offsets, h0, R, B, M, MP, chain, nblocks);
  return cudaGetLastError();
}


}  // namespace fi
