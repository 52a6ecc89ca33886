// match_kernels.cu — batched longest-prefix-match + weighted score + warp-shuffle
// argmax over all endpoints, sm_90a.  Bound by per-warp latency (dependent index / row reads and the
// counting arithmetic); no tensor cores (there is no dense contraction on this path).
//
// One warp per request (persistent grid, dynamic queue):
//   1. stage the request's block-hash chain in shared memory (cp.async);
//   2. 32 blocks at a time, one block per lane: find the block's index NODE.  The index numbers its
//      nodes in insertion order (index_device.cuh), so after one table lookup for the first block the
//      lanes check "my node = the previous block's node + 1" with a coalesced read of klog; the table is
//      probed again only where that fails — normally at the first block the index does not hold, which
//      ends the walk (upstream Plugin.matchLongestPrefix stops at the first block no pod holds —
//      SURVEY.md Appendix A.3).  The next chunk's check is issued before this chunk's rows are read;
//      the rows (consecutive 128-byte bitsets over the local endpoints) are read 2 per load instruction,
//      16 in flight per lane group;
//   3. per-endpoint match counts accumulate in bit-planes (bitslice.cuh);
//   4. only endpoints with a non-zero count are scored individually, in fp64 with
//      explicit round-to-nearest mul/add in profile order (SURVEY.md Appendix A.4,
//      weights of /root/reference/pkg/router/strategy.go:66,157,163); all others
//      share the per-batch "zero-match best" precomputed by prepare_endpoints —
//      valid because every scorer weight is >= 0, so a total is monotone in the
//      match count;
//   5. warp-shuffle argmax (the RANKED variant: k selection rounds, ranked_profile; its SUBSET twin scores only each
//      request's candidate subset, S.5a); equal totals are resolved by the request's tie rotation (tiebreak.cuh — upstream's
//      MaxScorePicker shuffles, Appendix A.5), then the pd-profile-handler threshold rule (Appendix A.6,
//      /root/reference/pkg/router/strategy.go:129-133).
//   The COUNTS variant (fi_epp_match_counts, docs/SPEC.md S.3a) replaces 4./5. with counts_row: every local endpoint's
//   match count, written as the request's row of a dense [R][ep_count] u16 matrix.  Its LISTS form (fi_epp_match_lists,
//   S.3b) writes only the matched endpoints, into the request's slot of a scratch that list_scan_kernel and
//   list_copy_kernel then pack.
//
// Rows narrower than 32 words (fewer than 1024 local endpoints, e.g. an
// endpoint-range shard of a multi-GPU pool) are read G = 32/L rows per load
// instruction by G lane groups whose counters are merged at the end.
//
// Sharded pools run the SAME kernel: every rank's table is a directory of the whole pool's keys
// (index_kernels.cu), so "the first block no pod holds" is a local lookup; the only exchange of the step is
// the rank's (score, endpoint) pick, stored straight into every rank's memory (PeerXchg) and reduced by
// merge_picks_kernel.
#include <climits>
#include <map>
#include <mutex>
#include <utility>

#include "bitslice.cuh"
#include "index_device.cuh"
#include "kernels.cuh"
#include "tiebreak.cuh"

namespace fi {

namespace {

constexpr int kWarps = 8;
// match_window_kernel: blocks per window (the chain staged at once), and counter planes for counts up to 4095
constexpr int kWindow = 1024;
constexpr int kWindowPlanes = 12;
#ifndef FI_MATCH_MIN_BLOCKS
#define FI_MATCH_MIN_BLOCKS 2
#endif
constexpr unsigned FULL = 0xFFFFFFFFu;

struct Best {
  double score;
  uint32_t e;  // local endpoint or FI_NO_ENDPOINT
  uint32_t m;
  uint32_t k;  // tie key of e: its distance from the request's rotation start (smaller wins among equal totals)
};

// the request's tie rotation (tiebreak.cuh), in this rank's local endpoint numbering
struct TieRot {
  uint32_t start;     // global rotation start in [0, E)
  uint32_t E;         // pool size
  uint32_t ep_begin;  // first global endpoint of this rank
  __device__ __forceinline__ uint32_t key(uint32_t e_local) const { return tie_rot(e_local + ep_begin, start, E); }
};

__device__ __forceinline__ bool better(double s, uint32_t k, const Best& b) { return s > b.score || (s == b.score && k < b.k); }

// First member, in rotation order, of a set of LOCAL endpoints given as W bit words (warp-cooperative; every
// lane gets the result; FI_NO_ENDPOINT if the set is empty); the word arithmetic is tiebreak.cuh's.
__device__ __forceinline__ uint32_t tie_first_local(const uint32_t* __restrict__ T, uint32_t W, const TieRot& tr,
                                                    uint32_t ep_count, int lane) {
  const uint32_t p = tie_local_origin(tr.start, tr.ep_begin, ep_count);
  const uint32_t mask = W * 32u - 1u;  // W is a power of two
  uint32_t best = 0xFFFFFFFFu;         // smallest (position - p) mod (32 W)
  for (uint32_t wi = lane; wi < W; wi += 32) best = min(best, tie_word_min(__ldg(T + wi), wi, p, mask));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, d));
  return best == 0xFFFFFFFFu ? FI_NO_ENDPOINT : ((best + p) & mask);
}

// SURVEY.md Appendix A.4 — identical operation order to oracle/epp_oracle.cpp:total_score
// upstream lora-affinity-scorer (SURVEY.md §8a row a11): adapter active on the endpoint 1.0, endpoint
// has room for one more adapter 0.8, adapter queued there 0.6, else 0
__device__ __forceinline__ double lora_score(const LoraDev& l, uint64_t adapter) {
  bool active = false, waiting = false;
#pragma unroll
  for (int i = 0; i < (int)FI_EPP_MAX_LORA; ++i) {
    active |= (uint32_t)i < l.n_active && l.active[i] == adapter;
    waiting |= (uint32_t)i < l.n_waiting && l.waiting[i] == adapter;
  }
  if (active) return 1.0;
  if (l.n_active + l.n_waiting < l.max_active) return 0.8;
  return waiting ? 0.6 : 0.0;
}

// REQ_QUEUE (subset picks, S.5a): the queue scorer's value is q_v, normalised over the request's own eligible set,
// instead of the per-batch table entry
template <bool REQ_QUEUE = false>
__device__ __forceinline__ double total_score(const ProfileDev& pr, const double* __restrict__ sc_p, uint32_t Epad,
                                              uint32_t e, uint32_t m, uint32_t n, double lora_v = 0.0, double q_v = 0.0) {
  double total = 0.0;
#pragma unroll
  for (int s = 0; s < (int)FI_EPP_MAX_SCORERS; ++s) {
    if (s < (int)pr.n_scorers) {
      double v;
      if (pr.kind[s] == FI_SCORER_PREFIX)
        v = n ? __ddiv_rn((double)m, (double)n) : 0.0;
      else if (pr.kind[s] == FI_SCORER_LORA)
        v = lora_v;
      else if (REQ_QUEUE && pr.kind[s] == FI_SCORER_QUEUE)
        v = q_v;
      else
        v = sc_p[(uint64_t)s * Epad + e];
      total = __dadd_rn(total, __dmul_rn(v, pr.weight[s]));
    }
  }
  return total;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
// ---- peer-memory exchange (sharded mode): tagged 64-bit words, see PeerXchg in kernels.cuh ------
__device__ __forceinline__ void ll_store(uint64_t* p, uint32_t data, uint32_t tag) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(p), "l"(((uint64_t)tag << 32) | data) : "memory");
}
__device__ __forceinline__ uint64_t ll_load(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
  return v;
}
constexpr long long kPollTimeoutCycles = 20000000000ll;  // ~10 s: a peer died or never launched
// PD rule shared by the single-GPU kernel and the multi-GPU merge kernel
__device__ __forceinline__ bool pd_prefill_runs(uint32_t dec_endpoint, uint32_t dec_match, uint32_t n, uint64_t len,
                                                double threshold) {
  double hit = (dec_endpoint != FI_NO_ENDPOINT && n) ? __ddiv_rn((double)dec_match, (double)n) : 0.0;
  double miss_bytes = __dmul_rn(__dsub_rn(1.0, hit), (double)len);
  return miss_bytes >= threshold;
}

// load VEC consecutive words of a row (16-byte vectors for full rows)
template <int VEC>
__device__ __forceinline__ void load_row_words(const uint32_t* __restrict__ p, bool ok, uint32_t (&out)[VEC]) {
  if (VEC == 4) {
    uint4 v = make_uint4(0, 0, 0, 0);
    if (ok) v = __ldg(reinterpret_cast<const uint4*>(p));
    out[0] = v.x;
    out[1 % VEC] = v.y;
    out[2 % VEC] = v.z;
    out[3 % VEC] = v.w;
  } else if (VEC == 2) {
    uint2 v = make_uint2(0, 0);
    if (ok) v = __ldg(reinterpret_cast<const uint2*>(p));
    out[0] = v.x;
    out[1 % VEC] = v.y;
  } else {
    out[0] = ok ? __ldg(p) : 0u;
  }
}

// Nodes of ALL blocks of a request, before any row is read.  A cached prefix was inserted in chain order, so its
// nodes are consecutive (index_device.cuh): after ONE table lookup for block `pos` every later block i checks
// "my node = that node + (i - pos)" — coalesced reads of klog, kSpecChunks chunks of 32 blocks in flight at once.  The
// table is probed again only where that fails: normally at the first block the index does not hold, which ends
// the walk (both match modes stop at the first block no pod holds).  A prefix whose nodes are scattered (an index
// built out of chain order) gets kSpecTries such rounds, then its remaining blocks probe the table in parallel,
// 64 at a time, as a plain hash index would.
// Returns m = number of leading blocks the index holds (the first miss, or n); s_node[0 .. m) = their nodes.
//
// (Resolving chunk c+1 while chunk c's rows are in flight makes a request's serial chain two dependent memory
// round trips per 32 blocks, and the last fully cached prompt keeps the other warps waiting.  With the nodes
// known up front the rows of a request are independent loads.)
constexpr int kSpecTries = 4;
// Chunks of 32 blocks verified per round; a round is issued only when every block of the one before it verified.  Two
// (64 blocks): at cfg 3 the walk ends at block 103 on average, and checking all 256 blocks of a chain at once read
// about 1 KB of klog per request that no one used.  cfg 3 on one H100 80GB HBM3 (700 W), us per pipelined step,
// three runs each in one call: 8 chunks 171.7-172.0, 3 chunks 168.1-168.2, 2 chunks 168.4-168.5, 1 chunk 169.4-169.5.
constexpr int kSpecChunks = 2;

__device__ __forceinline__ uint32_t resolve_request_nodes(const IndexView& ix, const uint64_t* __restrict__ s_chain,
                                                          uint32_t* __restrict__ s_node, uint32_t n, int lane, bool have_first,
                                                          uint32_t first_node) {
  uint32_t pos = 0;  // blocks [0, pos) are resolved and present
  for (int tries = 0; pos < n; ++tries) {
    if (tries < kSpecTries) {
      uint32_t nf = SLOT_MISS;
      if (tries == 0 && have_first) {
        nf = first_node;  // block 0's table lookup was issued during the previous request (warp-uniform)
      } else {
        if (lane == 0) nf = index_find(ix, s_chain[pos]);
        nf = __shfl_sync(FULL, nf, 0);
      }
      if (nf == SLOT_MISS) return pos;  // first miss of the request
      if (lane == 0) s_node[pos] = nf;
      uint32_t fail = n;  // first block after pos whose node is not nf + distance
      if (nf >= ix.C) {
        fail = pos + 1;  // the hashes 0 / ~0 own fixed nodes: nothing to speculate from
      } else {
        for (uint32_t i0 = pos + 1; i0 < n && fail == n; i0 += 32 * kSpecChunks) {
          uint64_t hk[kSpecChunks], kk[kSpecChunks];
#pragma unroll
          for (int c = 0; c < kSpecChunks; ++c) {
            const uint32_t idx = i0 + 32 * c + lane;
            hk[c] = 0;
            kk[c] = 1;  // (!= hk: a lane without a block never verifies)
            if (idx < n) {
              hk[c] = s_chain[idx];
              const uint64_t cand = (uint64_t)nf + (idx - pos);
              if (cand < ix.C) kk[c] = __ldg(ix.klog + cand);
            }
          }
#pragma unroll
          for (int c = 0; c < kSpecChunks; ++c) {
            const uint32_t idx = i0 + 32 * c + lane;
            if (fail != n || i0 + 32 * c >= n) break;  // warp-uniform
            const bool ok = idx < n && kk[c] == hk[c] && !key_is_special(hk[c]);
            const unsigned bad = __ballot_sync(FULL, idx < n && !ok);
            const uint32_t upto = bad ? (uint32_t)(__ffs(bad) - 1) : 32u;
            if ((uint32_t)lane < upto && idx < n) s_node[idx] = nf + (idx - pos);
            if (bad) fail = i0 + 32 * c + upto;
          }
        }
      }
      pos = fail;
    } else {
      // scattered prefix: every remaining block of the next 64 probes the table
      const uint32_t ia = pos + lane, ib = pos + 32 + lane;
      uint32_t na = SLOT_MISS, nb = SLOT_MISS;
      if (ia < n) na = index_find_lazy(ix, s_chain[ia]);
      if (ib < n) nb = index_find_lazy(ix, s_chain[ib]);
      const unsigned ma = __ballot_sync(FULL, ia < n && na == SLOT_MISS);
      const unsigned mb = __ballot_sync(FULL, ib < n && nb == SLOT_MISS);
      const uint32_t upto = ma ? (uint32_t)(__ffs(ma) - 1) : (mb ? 32u + (uint32_t)(__ffs(mb) - 1) : 64u);
      if ((uint32_t)lane < upto && ia < n) s_node[ia] = na;
      if ((uint32_t)lane + 32 < upto && ib < n) s_node[ib] = nb;
      if (ma || mb) return pos + upto;
      pos = pos + 64 < n ? pos + 64 : n;
    }
  }
  return n;
}

// next request of the launch's dynamic queue.  Plain PTX on purpose: for `if (lane == 0) atomicAdd(..)` the
// compiler emits its warp-aggregated form — ATOMG followed at once by a SHFL of the result — which makes every
// request wait out the atomic's round trip.  Here the result
// register is not touched until the shuffle at the end of the request.
__device__ __forceinline__ uint32_t take_ticket(uint32_t* counter, uint32_t opaque_zero) {
  uint32_t t;
  asm volatile("atom.relaxed.gpu.global.add.u32 %0, [%1], 1;\n" : "=r"(t) : "l"(counter + opaque_zero) : "memory");
  return t;
}

// docs/SPEC.md S.6a, the ranked pick of one profile (RANKED variant of match_pick_kernel): out[(r*P + pi)*k + j] for
// j < k.  Every eligible endpoint is scored, the way the LoRA branch does: after the merge every lane group holds
// the full counters, so group g takes bits [g*32/G, (g+1)*32/G) of its lanes' words (the per-batch zero-match best
// does not apply; lora_score only when the configuration has a LoRA scorer).  k rounds then select in the single
// pick's order — better(): total desc, then the tie rotation, a strict total order because tie keys are unique.
// Each lane keeps its best endpoint among those ranked after the previous round's winner; a warp butterfly picks
// the round's winner and only the lane that owned it rescans its endpoints, bounded by the winner's (score, key).
// No "taken" mask: a round is one butterfly plus one lane's rescan.  Once every lane is out of candidates the
// rounds write the padding entry (FI_NO_ENDPOINT, match 0, score 0).
// SUBSET (S.5a): sub[x] is the request's candidate word t*VEC + x.  The eligible words become elig & sub, and the
// queue scorer is normalised by the min / max queue depth over those endpoints (a warp reduction over the raw
// endpoint state), in prepare_endpoints' arithmetic; the per-batch queue column does not apply.
template <int VEC, int G, bool SUBSET, int NP>
__device__ __forceinline__ void ranked_profile(const MatchParams& p, uint32_t pi, const BitCounter<NP> (&cnt)[VEC],
                                               const uint32_t (&sub)[VEC], const TieRot& tr, uint32_t n, uint32_t r,
                                               int lane, int t, int g, uint32_t& dec_e, uint32_t& dec_m) {
  const ProfileDev& pr = p.st.prof[pi];
  const double* sc_p = p.st.sc + (uint64_t)pi * FI_EPP_MAX_SCORERS * p.st.Epad;
  const bool lora = p.st.has_lora != 0;
  const uint64_t adapter = (lora && p.adapters) ? p.adapters[r] : 0;
  constexpr uint32_t BPG = 32 / G;
  const uint32_t gmask_bits = (BPG >= 32 ? 0xFFFFFFFFu : ((1u << BPG) - 1u)) << (g * BPG);
  bool has_q = false;  // SUBSET: the profile has a queue scorer
  int minq = 0, maxq = 0;
  if constexpr (SUBSET) {
#pragma unroll
    for (int s = 0; s < (int)FI_EPP_MAX_SCORERS; ++s) has_q |= s < (int)pr.n_scorers && pr.kind[s] == FI_SCORER_QUEUE;
    if (has_q) {  // warp-uniform
      int mn = INT_MAX, mx = INT_MIN;
#pragma unroll
      for (int x = 0; x < VEC; ++x) {
        const uint32_t wi = t * VEC + x;
        uint32_t cand = p.st.elig[(uint64_t)pi * p.ix.W + wi] & sub[x] & gmask_bits;
        while (cand) {
          const uint32_t bit = __ffs(cand) - 1;
          cand &= cand - 1;
          const int q = __ldg(&p.eps[p.ep_begin + wi * 32 + bit].queue_depth);
          mn = min(mn, q);
          mx = max(mx, q);
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        mn = min(mn, __shfl_xor_sync(FULL, mn, d));
        mx = max(mx, __shfl_xor_sync(FULL, mx, d));
      }
      minq = mn;
      maxq = mx;
    }
  }
  // this lane's best endpoint ranked strictly after (ts, tk); ts < 0: no bound (totals are >= 0)
  auto scan = [&](double ts, uint32_t tk) {
    Best b;
    b.score = -1.0;
    b.e = FI_NO_ENDPOINT;
    b.m = 0;
    b.k = 0xFFFFFFFFu;
#pragma unroll
    for (int x = 0; x < VEC; ++x) {
      const uint32_t wi = t * VEC + x;
      uint32_t cand = p.st.elig[(uint64_t)pi * p.ix.W + wi] & gmask_bits;
      if constexpr (SUBSET) cand &= sub[x];
      while (cand) {
        const uint32_t bit = __ffs(cand) - 1;
        cand &= cand - 1;
        const uint32_t e = wi * 32 + bit;
        const uint32_t m = bc_get(cnt[x], bit);
        double qv = 0.0;
        if constexpr (SUBSET) {
          if (has_q) {
            const int q = __ldg(&p.eps[p.ep_begin + e].queue_depth);
            qv = (maxq == minq) ? 1.0
                                : __ddiv_rn((double)((long long)maxq - (long long)q), (double)((long long)maxq - (long long)minq));
            qv = qv < 0.0 ? 0.0 : (qv > 1.0 ? 1.0 : qv);
          }
        }
        const double s = total_score<SUBSET>(pr, sc_p, p.st.Epad, e, m, n, lora ? lora_score(p.st.lora[e], adapter) : 0.0, qv);
        const uint32_t k = tr.key(e);
        if (ts >= 0.0 && !(ts > s || (ts == s && tk < k))) continue;  // ranked before or at the bound
        if (better(s, k, b)) {
          b.score = s;
          b.e = e;
          b.m = m;
          b.k = k;
        }
      }
    }
    return b;
  };
  Best b = scan(-1.0, 0u);
  const uint32_t K = p.k;
  fi_pick* out = p.out + ((uint64_t)r * p.st.n_profiles + pi) * K;
  for (uint32_t j = 0; j < K; ++j) {
    Best w = b;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const double os = __shfl_xor_sync(FULL, w.score, d);
      const uint32_t oe = __shfl_xor_sync(FULL, w.e, d);
      const uint32_t om = __shfl_xor_sync(FULL, w.m, d);
      const uint32_t ok = __shfl_xor_sync(FULL, w.k, d);
      if (better(os, ok, w)) {
        w.score = os;
        w.e = oe;
        w.m = om;
        w.k = ok;
      }
    }
    const bool none = w.e == FI_NO_ENDPOINT;  // warp-uniform
    if (j == 0 && pi == p.pd_decode) {
      dec_e = w.e;
      dec_m = w.m;
    }
    if (lane == 0) {
      fi_pick pk;
      pk.endpoint = none ? FI_NO_ENDPOINT : w.e + p.ep_begin;
      pk.match_blocks = none ? 0 : (uint16_t)w.m;
      pk.n_blocks = (uint16_t)n;
      pk.score = none ? 0.0 : w.score;
      out[j] = pk;
    }
    if (!none && b.e == w.e) b = scan(w.score, w.k);  // endpoints belong to one lane each: only the winner's rescans
  }
}

// docs/SPEC.md S.3a, the epilogue of the COUNTS variant: request r's row counts[r * ep_count + j] = the match count of
// local endpoint j.  After the merge every lane group holds the full counters, so group g unpacks bits
// [g*32/G, (g+1)*32/G) of its lanes' words (as the LoRA branch splits them) into the warp's staging row in shared
// memory, placed at the offset the row has in its first 32-byte sector of global memory.  The warp then stores 16
// bytes per lane from that sector on: whole sectors, except the row's first and last, which it shares with the rows
// before and after it and writes with 2-byte stores (any 2-byte aligned counts pointer works).  Words without a
// matched endpoint store zeros without unpacking; a request without a matched block skips the staging row.
template <int VEC, int G, int NP>
__device__ __forceinline__ void counts_row(const MatchParams& p, const BitCounter<NP> (&cnt)[VEC], uint32_t r, bool nothing,
                                           uint16_t* __restrict__ s_row, int lane, int t, int g) {
  constexpr int BPG = 32 / G;
  const uint64_t a = reinterpret_cast<uint64_t>(p.counts + (uint64_t)r * p.ep_count);
  const uint32_t shift = (uint32_t)(a & 31u) >> 1;  // counts of the rows before this one in its first sector
  uint16_t* const base = reinterpret_cast<uint16_t*>(a - 2u * shift);
  const uint32_t end = shift + p.ep_count;
  if (!nothing) {
#pragma unroll
    for (int x = 0; x < VEC; ++x) {
      uint16_t* o = s_row + shift + (uint32_t)(t * VEC + x) * 32u + (uint32_t)(g * BPG);
      if (bc_nonzero(cnt[x])) {
        bc_unpack<BPG>(cnt[x], (uint32_t)(g * BPG), o);
      } else {
#pragma unroll
        for (int i = 0; i < BPG; ++i) o[i] = 0;
      }
    }
    __syncwarp();  // the staging row is written by each lane group and read by every lane
  }
  for (uint32_t c = lane; c < (end + 7) / 8; c += 32) {
    const uint32_t j0 = c * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (!nothing) v = *reinterpret_cast<const uint4*>(s_row + j0);
    if (j0 >= shift && j0 + 8 <= end) {
      *reinterpret_cast<uint4*>(base + j0) = v;
    } else {  // the row's first or last 16 bytes
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (j0 + i >= shift && j0 + i < end) base[j0 + i] = (uint16_t)(w[i >> 1] >> (16 * (i & 1)));
    }
  }
}

// docs/SPEC.md S.3b, the epilogue of the LISTS variant (a COUNTS variant that writes lists instead of rows): request
// r's matched local endpoints, ascending, packed as (column << 12) | count into its slot p.lists[r * ep_count ..], and
// their number into p.nnz[r].  No dense row is staged.  After the merge every lane group holds the full counters, so
// group g takes bits [g*32/G, (g+1)*32/G) of its lanes' words (as counts_row does) and unpacks only the matched ones.
// An entry's position in the slot is the number of matched endpoints before it: those of the group's lanes before this
// one (an inclusive shuffle scan over the LPR lanes of the group, which every group computes alike), of this lane's
// words before x, and of the bits of word x below the group's range.  The slot index is the request's, so the result
// does not depend on the order in which the dynamic queue finishes requests.
template <int VEC, int G, int NP>
__device__ __forceinline__ void lists_slot(const MatchParams& p, const BitCounter<NP> (&cnt)[VEC], uint32_t r, bool nothing,
                                           int lane, int t, int g) {
  constexpr int LPR = 32 / G;
  constexpr uint32_t BPG = 32 / G;
  if (!nothing) {  // warp-uniform
    // a word's matched endpoints: its non-zero counters below ep_count (rows hold no bits past it)
    auto matched = [&](int x) {
      const uint32_t e0 = (uint32_t)(t * VEC + x) * 32u;
      const uint32_t lim = p.ep_count > e0 ? p.ep_count - e0 : 0u;
      return bc_nonzero(cnt[x]) & (lim >= 32 ? 0xFFFFFFFFu : ((1u << lim) - 1u));
    };
    uint32_t mine = 0;
#pragma unroll
    for (int x = 0; x < VEC; ++x) mine += __popc(matched(x));
    uint32_t incl = mine;
#pragma unroll
    for (int d = 1; d < LPR; d <<= 1) {
      const uint32_t o = __shfl_up_sync(FULL, incl, d, LPR);
      if (t >= d) incl += o;
    }
    const uint32_t total = __shfl_sync(FULL, incl, LPR - 1, LPR);
    if (lane == 0) p.nnz[r] = total;
    // (32-bit positions within the slot, indexed from the parameter at each store: no 64-bit pointer stays live)
    uint32_t pos = incl - mine;
    const uint32_t gmask = (BPG >= 32 ? 0xFFFFFFFFu : ((1u << BPG) - 1u)) << (g * BPG);
    const uint32_t below = (1u << (g * BPG)) - 1u;  // g * BPG < 32
#pragma unroll
    for (int x = 0; x < VEC; ++x) {
      const uint32_t nz = matched(x);
      const uint32_t e0 = (uint32_t)(t * VEC + x) * 32u;
      uint32_t at = pos + __popc(nz & below);
      for (uint32_t cand = nz & gmask; cand; cand &= cand - 1) {
        const uint32_t bit = __ffs(cand) - 1;
        p.lists[(uint64_t)r * p.ep_count + at++] = ((e0 + bit) << 12) | bc_get(cnt[x], bit);
      }
      pos += __popc(nz);
    }
  } else if (lane == 0) {
    p.nnz[r] = 0;
  }
}

// LPR lanes read one row (VEC words each, LPR*VEC = words per row); a load
// instruction therefore covers G = 32/LPR rows.  E = 1024 → LPR 16, VEC 2: a 128-byte
// row is 16 × 8-byte loads and one instruction brings in 2 rows; 16 rows in flight.
// (The RANKED variant keeps the counters live through its selection rounds: it asks for two CTAs per SM, the
// register budget of the four-word shape, instead of spilling under the three-CTA budget of the two-word one.)
// SUBSET (with RANKED only): every request carries a candidate bitset (docs/SPEC.md S.5a).  Steps 1-3 do not look
// at it — the walk and the counts stay pool-wide — and its words are loaded when the request starts, so they
// arrive under the walk; only the scoring of ranked_profile uses them.
// COUNTS (not with LORA / RANKED): steps 1-3 as for a pick, then counts_row writes the request's match counts instead
// of steps 4-5 and the PD rule.  Its staging rows follow the node buffers in shared memory, Epad + 16 counts per warp.
// LISTS (with COUNTS only): lists_slot writes the request's matched endpoints instead of counts_row's dense row; no
// staging row.
// WIN (match_window_kernel, handles with max_blocks > 1023; DESIGN.md §4.9): steps 1-3 run once per window of up to
// kWindow blocks, in staging buffers of kWindow entries, and the counters have 12 bit-planes; steps 4-5 are the same.
template <int LPR, int VEC, bool LPM, bool LORA, bool RANKED, bool SUBSET, bool COUNTS, bool LISTS, bool WIN>
__device__ __forceinline__ void match_pick_body(const MatchParams& p) {
  constexpr int G = 32 / LPR;                 // rows per load instruction
  constexpr int NP = WIN ? kWindowPlanes : NPLANES;
#ifndef FI_MATCH_BATCH
#define FI_MATCH_BATCH 16
#endif
  // load instructions in flight per lane: 16 (= 32 rows at E = 1024) where the registers allow it
  constexpr int BATCH_MAX = (LPM || VEC >= 4) ? 8 : FI_MATCH_BATCH;
  constexpr int BATCH = LPR < BATCH_MAX ? LPR : BATCH_MAX;
  extern __shared__ __align__(16) uint64_t s_mem[];
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int t = lane % LPR;  // position within the row
  const int g = lane / LPR;  // row group
  // per warp: two chain buffers (the next request's chain is staged while this one is matched) and the nodes
  // entries per buffer: a whole chain row, or one window.  An expression at each use, not a local: a local holding
  // p.MP moved the register allocation of several unwindowed instantiations.
#define SP (WIN ? (uint32_t)kWindow : p.MP)
  uint64_t* const s_chain_base = s_mem + (size_t)(2 * warp) * SP;  // buffer b at s_chain_base + b * SP
  uint32_t* s_node = reinterpret_cast<uint32_t*>(s_mem + (size_t)2 * kWarps * SP) + (size_t)warp * SP;  // node of every block
  uint16_t* s_row = nullptr;  // COUNTS: the warp's staging row
  if constexpr (COUNTS && !LISTS)
    s_row = reinterpret_cast<uint16_t*>(s_mem + (size_t)2 * kWarps * SP) + (size_t)2 * kWarps * SP +
            (size_t)warp * (p.st.Epad + 16);
  const IndexView ix = p.ix;
  const uint32_t P = COUNTS ? 0u : p.st.n_profiles;  // COUNTS: no profile is scored
  const char* row_base = reinterpret_cast<const char*>(ix.rows + t * VEC);
  const uint32_t row_bytes = 4u << ix.logW;
  const uint32_t zero_slot = (uint32_t)(ix.C + 2);  // never written: all-zero row

  // Dynamic work queue (requests differ a lot in how many rows they touch), software-pipelined across requests:
  // while request r is matched, the ticket of the request after next is in flight, the chain of the next one is
  // being staged into the other buffer, and the home bucket of its first block is being fetched (lanes 0-3:
  // one key + node each) — a request starts with its chain and its first node already there instead of waiting
  // out three dependent round trips (ticket -> chain -> table).
  const uint32_t row_units = p.MP / 2;  // 16-byte units of a chain row (rows are zero-padded to MP by the walker)
  auto stage = [&](uint32_t rr, uint64_t* dst) {
    const uint64_t* crow = p.chain + (uint64_t)rr * p.MP;
    for (uint32_t u = lane; u < row_units; u += 32) cp_async16(dst + 2 * u, crow + 2 * u);
  };
  // WIN: entries [w0, w0 + kWindow) of the row (w0 a multiple of kWindow; MP - w0 is even)
  auto stage_window = [&](uint32_t rr, uint32_t w0, uint64_t* dst) {
    const uint64_t* crow = p.chain + (uint64_t)rr * p.MP + w0;
    const uint32_t units = min(p.MP - w0, (uint32_t)kWindow) / 2;
    for (uint32_t u = lane; u < units; u += 32) cp_async16(dst + 2 * u, crow + 2 * u);
  };
  uint32_t r_next = 0;
  if (lane == 0) r_next = take_ticket(p.work_counter, threadIdx.x & p.lane_zero);
  r_next = __shfl_sync(FULL, r_next, 0);
  int buf = 0;
  if constexpr (WIN) {
    if (r_next < p.R) stage_window(r_next, 0, s_chain_base);
  } else {
    if (r_next < p.R) stage(r_next, s_chain_base);
  }
  // prefetched home bucket of the current request's first block (valid when pf_ok)
  bool pf_ok = false;
  uint64_t pf_h = 0, pf_key = 0;
  uint32_t pf_node = 0;
  for (;;) {
    const uint32_t r = r_next;
    if (r >= p.R) break;
    if (lane == 0) r_next = take_ticket(p.work_counter, threadIdx.x & p.lane_zero);
    const uint32_t n = p.nblocks[r];
    uint32_t sub[VEC];  // SUBSET: this lane's words of the request's candidate bitset
#pragma unroll
    for (int x = 0; x < VEC; ++x) {
      sub[x] = 0u;
      if constexpr (SUBSET) {
        const uint32_t wi = t * VEC + x;
        if (wi < p.sub_pitch) sub[x] = __ldg(p.subsets + (uint64_t)r * p.sub_pitch + wi);
      }
    }
    uint64_t* s_chain = s_chain_base + (size_t)buf * SP;
#ifdef FI_MATCH_TIMING
    const long long tm0 = clock64();
#endif
    // ---- 1. the chain was staged during the previous request (or just above)
    cp_async_wait_all();
    __syncwarp();
    // first block's node from the prefetched bucket
    bool have_first = false;
    uint32_t first_node = SLOT_MISS;
    if (pf_ok && n) {
      const unsigned hit = __ballot_sync(FULL, lane < BUCKET_KEYS && pf_key == pf_h);
      const unsigned emp = __ballot_sync(FULL, lane < BUCKET_KEYS && pf_key == KEY_EMPTY);
      if (hit) {
        first_node = __shfl_sync(FULL, pf_node, __ffs(hit) - 1);
        have_first = true;
      } else if (emp) {
        have_first = true;  // definite miss
      }  // else: home bucket full without a match — resolve_request_nodes probes on
    }
    if constexpr (LISTS) {
      // The bucket is read: end its registers' live range here.  Assigned only when a bucket is fetched, they would
      // otherwise stay live around the whole request for the requests that fetch none, which made
      // match_window_kernel<16, 2, upstream, .., LISTS> spill pf_node under its 80-register bound.
      pf_key = 0;
      pf_node = 0;
    }

#ifdef FI_MATCH_TIMING
    const long long tm1 = clock64();
    long long tm2 = 0;
#endif
    BitCounter<NP> cnt[VEC];
    uint32_t alive[VEC];
#pragma unroll
    for (int x = 0; x < VEC; ++x) {
      bc_clear(cnt[x]);
      alive[x] = 0xFFFFFFFFu;
    }
    uint32_t matched_rows = 0;
    bool real_miss = false;
    uint64_t h_first = 0;  // WIN: block 0's hash (the tie seed), read before the buffer holds a later window
    if constexpr (WIN) h_first = n ? s_chain[0] : 0ull;

    if constexpr (!WIN) {
      // ---- 2. the index node of every block up to the first one no endpoint holds ---------------
      const uint32_t m_rows = resolve_request_nodes(ix, s_chain, s_node, n, lane, have_first, first_node);
      real_miss = m_rows < n;
      __syncwarp();  // s_node is written by some lanes and read by others
      // ---- the next request: its ticket has long arrived; stage its chain and read its first hash
      r_next = __shfl_sync(FULL, r_next, 0);
      pf_ok = false;
      if (r_next < p.R) {
        stage(r_next, s_chain_base + (size_t)(buf ^ 1) * p.MP);
        pf_h = __ldg(p.chain + (uint64_t)r_next * p.MP);
      }
#ifdef FI_MATCH_TIMING
      tm2 = clock64();
#endif
      // ---- 3. the rows of those blocks: independent loads, BATCH instructions (BATCH * G rows) in flight --
#pragma unroll 1
      for (uint32_t b0 = 0; b0 < m_rows; b0 += BATCH * G) {
        uint32_t w[VEC][BATCH];
#pragma unroll
        for (int qi = 0; qi < BATCH; ++qi) {
          const uint32_t j = b0 + qi * G + g;  // row this lane helps read; rows past the end read the permanently
          const uint32_t sn = j < m_rows ? s_node[j] : zero_slot;  // zero row instead of being predicated off
          uint32_t tmp[VEC];
          load_row_words<VEC>(reinterpret_cast<const uint32_t*>(row_base + (uint64_t)sn * row_bytes), true, tmp);
#pragma unroll
          for (int x = 0; x < VEC; ++x) w[x][qi] = tmp[x];
        }
        if (LPM) {
#pragma unroll
          for (int qi = 0; qi < BATCH; ++qi) {
#pragma unroll
            for (int x = 0; x < VEC; ++x) {
              uint32_t v = w[x][qi];
              if (G > 1) {  // prefix-AND over the G rows of this instruction
#pragma unroll
                for (int d = 1; d < G; d <<= 1) {
                  const uint32_t o = __shfl_up_sync(FULL, v, d * LPR);
                  if (g >= d) v &= o;
                }
                v &= alive[x];
                alive[x] = __shfl_sync(FULL, v, (G - 1) * LPR + t);
              } else {
                v &= alive[x];
                alive[x] = v;
              }
              w[x][qi] = v;
            }
          }
        }
#pragma unroll
        for (int x = 0; x < VEC; ++x) {
          // membership rows are sparse: most 32-endpoint words of a batch are zero for every lane,
          // and adding zeros is a no-op — skip the carry-save tree then (warp-uniform branch)
          uint32_t any = 0;
#pragma unroll
          for (int qi = 0; qi < BATCH; ++qi) any |= w[x][qi];
          if (__any_sync(FULL, any != 0)) bc_add<BATCH>(cnt[x], w[x]);
        }
        matched_rows = min(m_rows, b0 + BATCH * G);
        if (LPM) {  // every local endpoint already dropped out: nothing more can match
          bool any = false;
#pragma unroll
          for (int x = 0; x < VEC; ++x) any |= alive[x] != 0;
          if (!__ballot_sync(FULL, any)) break;
        }
      }
    } else {
      // the next request: its ticket has long arrived; stage its first window and read its first hash
      auto stage_next_request = [&]() {
        r_next = __shfl_sync(FULL, r_next, 0);
        pf_ok = false;
        if (r_next < p.R) {
          stage_window(r_next, 0, s_chain_base + (size_t)(buf ^ 1) * SP);
          pf_h = __ldg(p.chain + (uint64_t)r_next * p.MP);
        }
      };
      // ---- 3. the rows of s_node[0, m_rows) (blocks w0 ..), as above.  Returns true when LPM has dropped every
      // local endpoint.
      auto read_rows = [&](uint32_t m_rows, uint32_t w0) -> bool {
#pragma unroll 1
        for (uint32_t b0 = 0; b0 < m_rows; b0 += BATCH * G) {
          uint32_t w[VEC][BATCH];
#pragma unroll
          for (int qi = 0; qi < BATCH; ++qi) {
            const uint32_t j = b0 + qi * G + g;  // row this lane helps read; rows past the end read the permanently
            const uint32_t sn = j < m_rows ? s_node[j] : zero_slot;  // zero row instead of being predicated off
            uint32_t tmp[VEC];
            load_row_words<VEC>(reinterpret_cast<const uint32_t*>(row_base + (uint64_t)sn * row_bytes), true, tmp);
#pragma unroll
            for (int x = 0; x < VEC; ++x) w[x][qi] = tmp[x];
          }
          if (LPM) {
#pragma unroll
            for (int qi = 0; qi < BATCH; ++qi) {
#pragma unroll
              for (int x = 0; x < VEC; ++x) {
                uint32_t v = w[x][qi];
                if (G > 1) {  // prefix-AND over the G rows of this instruction
#pragma unroll
                  for (int d = 1; d < G; d <<= 1) {
                    const uint32_t o = __shfl_up_sync(FULL, v, d * LPR);
                    if (g >= d) v &= o;
                  }
                  v &= alive[x];
                  alive[x] = __shfl_sync(FULL, v, (G - 1) * LPR + t);
                } else {
                  v &= alive[x];
                  alive[x] = v;
                }
                w[x][qi] = v;
              }
            }
          }
#pragma unroll
          for (int x = 0; x < VEC; ++x) {
            // membership rows are sparse: most 32-endpoint words of a batch are zero for every lane,
            // and adding zeros is a no-op — skip the carry-save tree then (warp-uniform branch)
            uint32_t any = 0;
#pragma unroll
            for (int qi = 0; qi < BATCH; ++qi) any |= w[x][qi];
            if (__any_sync(FULL, any != 0)) bc_add<BATCH>(cnt[x], w[x]);
          }
          matched_rows = w0 + min(m_rows, b0 + BATCH * G);
          if (LPM) {  // every local endpoint already dropped out: nothing more can match
            bool any = false;
#pragma unroll
            for (int x = 0; x < VEC; ++x) any |= alive[x] != 0;
            if (!__ballot_sync(FULL, any)) return true;
          }
        }
        return false;
      };

      // blocks [w0, w0 + nw) are in s_chain
      uint32_t w0 = 0;
#pragma unroll 1
      for (;;) {
        const uint32_t nw = min(n - w0, (uint32_t)kWindow);
        const uint32_t m_rows = resolve_request_nodes(ix, s_chain, s_node, nw, lane, have_first, first_node);
        real_miss = m_rows < nw;
        __syncwarp();
        // the walk goes on into the next window (every block of this one is cached): stage that window instead
        const bool more = !real_miss && w0 + nw < n;
        if (more)
          stage_window(r, w0 + kWindow, s_chain_base + (size_t)(buf ^ 1) * SP);
        else
          stage_next_request();
#ifdef FI_MATCH_TIMING
        tm2 = clock64();
#endif
        const bool dead = read_rows(m_rows, w0);
        if (!more) break;
        if (LPM && dead) {  // the staged window goes unread: the next request's first window takes its buffer
          cp_async_wait_all();  // (lane u % 32 writes unit u in both stagings, so each lane orders its own copies)
          stage_next_request();
          break;
        }
        // the next window.  Its block 0 continues the run of consecutive nodes (index_device.cuh) when klog holds
        // its hash at the previous block's node + 1; else resolve_request_nodes looks it up in the table.
        const uint32_t prev = s_node[kWindow - 1];
        w0 += kWindow;
        buf ^= 1;
        s_chain = s_chain_base + (size_t)buf * SP;
        cp_async_wait_all();
        __syncwarp();  // the window is staged for every lane, and this window's s_node reads are done
        const uint64_t h = s_chain[0];
        first_node = prev + 1;
        have_first = first_node < ix.C && !key_is_special(h) && __ldg(ix.klog + first_node) == h;
      }
    }

    if (r_next < p.R && !key_is_special(pf_h)) {  // pf_h has arrived by now: fetch its home bucket, used next iteration
      pf_ok = true;
      if (lane < BUCKET_KEYS) {
        const uint64_t slot0 = (pf_h & ix.bmask) * BUCKET_KEYS + lane;
        pf_key = __ldg(ix.keys + slot0);
        pf_node = __ldg(ix.node_of + slot0);
      }
    }
#ifdef FI_MATCH_TIMING
    const long long tm3 = clock64();
#endif
    // ---- merge the lane groups' counters ---------------------------------------
    const bool nothing = matched_rows == 0;  // warp-uniform: no row was read, every counter is zero
    if (G > 1 && !nothing) {
#pragma unroll
      for (int x = 0; x < VEC; ++x) {
#pragma unroll
        for (int d = LPR; d < 32; d <<= 1) {
          BitCounter<NP> o;
#pragma unroll
          for (int pl = 0; pl < NP; ++pl) o.c[pl] = __shfl_xor_sync(FULL, cnt[x].c[pl], d);
          bc_merge(cnt[x], o);
        }
      }
    }
    if constexpr (COUNTS && LISTS) lists_slot<VEC, G, NP>(p, cnt, r, nothing, lane, t, g);
    else if constexpr (COUNTS) counts_row<VEC, G, NP>(p, cnt, r, nothing, s_row, lane, t, g);

    // ---- 4./5. score candidates, argmax, PD rule ---------------------------------
    TieRot tr;
    tr.E = p.E_global;
    tr.ep_begin = p.ep_begin;
    tr.start = tie_start(tie_seed(n, WIN ? h_first : (n ? s_chain[0] : 0ull), n ? 0ull : p.h0[r], p.r_base + r), p.E_global);
    uint32_t dec_e = FI_NO_ENDPOINT, dec_m = 0;
#pragma unroll
    for (int pi = 0; pi < (int)FI_EPP_MAX_PROFILES; ++pi) {
      if (pi < (int)P) {
        if constexpr (RANKED) {
          ranked_profile<VEC, G, SUBSET, NP>(p, (uint32_t)pi, cnt, sub, tr, n, r, lane, t, g, dec_e, dec_m);
          continue;
        }
        const ProfileDev& pr = p.st.prof[pi];
        const double* sc_p = p.st.sc + (uint64_t)pi * FI_EPP_MAX_SCORERS * p.st.Epad;
        Best b;
        b.score = -1.0;
        b.e = FI_NO_ENDPOINT;
        b.m = 0;
        b.k = 0xFFFFFFFFu;
        if (LORA) {
          // The lora-affinity score depends on the request's adapter, so there is no per-batch
          // zero-match best: score every eligible endpoint.  After the merge every lane group holds the
          // full counters, so group g takes bits [g*32/G, (g+1)*32/G) of its lanes' words.
          const uint64_t adapter = p.adapters ? p.adapters[r] : 0;
          constexpr uint32_t BPG = 32 / G;
          const uint32_t gmask_bits = (BPG >= 32 ? 0xFFFFFFFFu : ((1u << BPG) - 1u)) << (g * BPG);
#pragma unroll
          for (int x = 0; x < VEC; ++x) {
            const uint32_t wi = t * VEC + x;
            uint32_t cand = p.st.elig[(uint64_t)pi * ix.W + wi] & gmask_bits;
            while (cand) {
              const uint32_t bit = __ffs(cand) - 1;
              cand &= cand - 1;
              const uint32_t e = wi * 32 + bit;
              const uint32_t m = bc_get(cnt[x], bit);
              const double s = total_score(pr, sc_p, p.st.Epad, e, m, n, lora_score(p.st.lora[e], adapter));
              const uint32_t k = tr.key(e);
              if (better(s, k, b)) {
                b.score = s;
                b.e = e;
                b.m = m;
                b.k = k;
              }
            }
          }
        } else if (g == 0 && !nothing) {
#pragma unroll
          for (int x = 0; x < VEC; ++x) {
            const uint32_t wi = t * VEC + x;
            uint32_t cand = bc_nonzero(cnt[x]) & p.st.elig[(uint64_t)pi * ix.W + wi];
            while (cand) {
              const uint32_t bit = __ffs(cand) - 1;
              cand &= cand - 1;
              const uint32_t e = wi * 32 + bit;
              const uint32_t m = bc_get(cnt[x], bit);
              const double s = total_score(pr, sc_p, p.st.Epad, e, m, n);
              const uint32_t k = tr.key(e);
              if (better(s, k, b)) {
                b.score = s;
                b.e = e;
                b.m = m;
                b.k = k;
              }
            }
          }
        }
        if (!nothing || LORA) {
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) {
            const double os = __shfl_xor_sync(FULL, b.score, d);
            const uint32_t oe = __shfl_xor_sync(FULL, b.e, d);
            const uint32_t om = __shfl_xor_sync(FULL, b.m, d);
            const uint32_t ok = __shfl_xor_sync(FULL, b.k, d);
            if (better(os, ok, b)) {
              b.score = os;
              b.e = oe;
              b.m = om;
              b.k = ok;
            }
          }
        }
        // Endpoints without a matched block share the per-batch zero-match total; which of the endpoints
        // attaining it comes first depends on this request's rotation.  (Skipped when a matched candidate
        // already beats that total: every scorer weight is >= 0.)
        const ZeroBest zb = p.st.zero[pi];
        if (!LORA && zb.any && !(b.score > zb.score)) {
          const uint32_t ez = tie_first_local(p.st.ztie + (uint64_t)pi * ix.W, ix.W, tr, p.ep_count, lane);
          if (ez != FI_NO_ENDPOINT) {
            const uint32_t kz = tr.key(ez);
            if (better(zb.score, kz, b)) {
              b.score = zb.score;
              b.e = ez;
              b.m = 0;
              b.k = kz;
            }
          }
        }
        if (pi == (int)p.pd_decode) {
          dec_e = b.e;
          dec_m = b.m;
        }
        const bool none = b.e == FI_NO_ENDPOINT;
        if (p.px.enabled) {
          // sharded: this rank's pick goes straight into every rank's gather slot as four tagged words
          // (every lane holds the same b after the butterfly; lane i stores word i%4 to rank i/4)
          const unsigned long long sb = (unsigned long long)__double_as_longlong(none ? 0.0 : b.score);
          for (uint32_t i = lane; i < p.px.world * 4; i += 32) {
            const uint32_t k = i >> 2, wsel = i & 3;
            const uint32_t val = wsel == 0   ? (none ? FI_NO_ENDPOINT : b.e + p.ep_begin)
                                 : wsel == 1 ? (none ? 0u : b.m)
                                 : wsel == 2 ? (uint32_t)sb
                                             : (uint32_t)(sb >> 32);
            uint64_t* dst = reinterpret_cast<uint64_t*>(p.px.base[k] + p.px.off_pick[p.px.step & 1u]) +
                            (((uint64_t)p.px.rank * p.R + r) * P + pi) * 4 + wsel;
            ll_store(dst, val, p.px.step);
          }
        } else if (lane == 0) {
          fi_pick pk;
          pk.endpoint = none ? FI_NO_ENDPOINT : b.e + p.ep_begin;
          pk.match_blocks = none ? 0 : (uint16_t)b.m;
          pk.n_blocks = (uint16_t)n;
          pk.score = none ? 0.0 : b.score;
          p.out[(uint64_t)r * P + pi] = pk;
        }
      }
    }
    if (lane == 0) {
      if (!COUNTS && p.apply_pd) {  // pd-profile-handler: the prefill pick stands only if the threshold test passes
        const uint64_t len = p.offsets[r + 1] - p.offsets[r];
        if (!pd_prefill_runs(dec_e, dec_m, n, len, p.pd_threshold)) {
          fi_pick pk;
          pk.endpoint = FI_NO_ENDPOINT;
          pk.match_blocks = 0;
          pk.n_blocks = (uint16_t)n;
          pk.score = 0.0;
          if constexpr (RANKED) {  // the prefill profile's whole list
            for (uint32_t j = 0; j < p.k; ++j) p.out[((uint64_t)r * P + p.pd_prefill) * p.k + j] = pk;
          } else {
            p.out[(uint64_t)r * P + p.pd_prefill] = pk;
          }
        }
      }
      if (p.probed_blocks) atomicAdd(p.probed_blocks, (unsigned long long)(matched_rows + (real_miss ? 1 : 0)));
#ifdef FI_MATCH_TIMING
      if (p.probed_blocks) {  // per-phase cycle sums behind the N_probe counter (debug build only)
        const long long tm4 = clock64();
        atomicAdd(p.probed_blocks + 1, (unsigned long long)(tm1 - tm0));
        atomicAdd(p.probed_blocks + 2, (unsigned long long)(tm2 - tm1));
        atomicAdd(p.probed_blocks + 3, (unsigned long long)(tm3 - tm2));
        atomicAdd(p.probed_blocks + 4, (unsigned long long)(tm4 - tm3));
        atomicAdd(p.probed_blocks + 5, 1ull);
      }
#endif
    }
    buf ^= 1;
    __syncwarp();  // this request's s_chain / s_node reads are done before the buffers are written again
  }
}

#undef SP

template <int LPR, int VEC, bool LPM, bool LORA, bool RANKED, bool SUBSET = false, bool COUNTS = false, bool LISTS = false>
__global__ void __launch_bounds__(kWarps * 32, (VEC >= 4 || RANKED ? FI_MATCH_MIN_BLOCKS : FI_MATCH_MIN_BLOCKS + 1))
    match_pick_kernel(const MatchParams p) {
  match_pick_body<LPR, VEC, LPM, LORA, RANKED, SUBSET, COUNTS, LISTS, false>(p);
}

// chains longer than one window (max_blocks > 1023): the same CTA shape, warps and shared memory per warp as
// match_pick_kernel at MP = kWindow
template <int LPR, int VEC, bool LPM, bool LORA, bool RANKED, bool SUBSET = false, bool COUNTS = false, bool LISTS = false>
__global__ void __launch_bounds__(kWarps * 32, (VEC >= 4 || RANKED ? FI_MATCH_MIN_BLOCKS : FI_MATCH_MIN_BLOCKS + 1))
    match_window_kernel(const MatchParams p) {
  match_pick_body<LPR, VEC, LPM, LORA, RANKED, SUBSET, COUNTS, LISTS, true>(p);
}

// multi-GPU: reduce the ranks' local picks (score desc, then the request's tie rotation), then the PD rule
__global__ void __launch_bounds__(256) merge_picks_kernel(const MergeParams p) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.R) return;
  const uint32_t n = p.nblocks[r];
  const uint32_t ts = tie_start(tie_seed(n, n ? p.chain[(uint64_t)r * p.MP] : 0ull, n ? 0ull : p.h0[r], r), p.E_global);
  fi_pick best[FI_EPP_MAX_PROFILES];
  for (uint32_t pi = 0; pi < p.P; ++pi) {
    fi_pick b;
    b.endpoint = FI_NO_ENDPOINT;
    b.match_blocks = 0;
    b.n_blocks = (uint16_t)n;
    b.score = 0.0;
    uint32_t bk = 0xFFFFFFFFu;
    for (uint32_t rk = 0; rk < p.ranks; ++rk) {
      fi_pick c;
      if (p.px.enabled) {  // four tagged words per pick, valid when all carry this step's tag
        const uint64_t* src = reinterpret_cast<const uint64_t*>(p.gathered) + (((uint64_t)rk * p.R + r) * p.P + pi) * 4;
        uint64_t v0, v1, v2, v3;
        const long long t0 = clock64();
        for (;;) {
          v0 = ll_load(src);
          v1 = ll_load(src + 1);
          v2 = ll_load(src + 2);
          v3 = ll_load(src + 3);
          const uint32_t tg = p.px.step;
          if ((uint32_t)(v0 >> 32) == tg && (uint32_t)(v1 >> 32) == tg && (uint32_t)(v2 >> 32) == tg && (uint32_t)(v3 >> 32) == tg) break;
          if (clock64() - t0 > kPollTimeoutCycles) {
            *p.px.err = 1;
            break;
          }
          __nanosleep(64);
        }
        c.endpoint = (uint32_t)v0;
        c.match_blocks = (uint16_t)v1;
        c.n_blocks = (uint16_t)n;
        c.score = __longlong_as_double((long long)((v3 << 32) | (v2 & 0xFFFFFFFFull)));
      } else {
        c = p.gathered[((uint64_t)rk * p.R + r) * p.P + pi];
      }
      if (c.endpoint == FI_NO_ENDPOINT) continue;
      const uint32_t ck = tie_rot(c.endpoint, ts, p.E_global);
      if (b.endpoint == FI_NO_ENDPOINT || c.score > b.score || (c.score == b.score && ck < bk)) {
        b = c;
        bk = ck;
      }
    }
    best[pi] = b;
  }
  if (p.apply_pd) {
    const fi_pick d = best[p.pd_decode];
    const uint64_t len = p.offsets[r + 1] - p.offsets[r];
    if (!pd_prefill_runs(d.endpoint, d.match_blocks, n, len, p.pd_threshold)) {
      best[p.pd_prefill].endpoint = FI_NO_ENDPOINT;
      best[p.pd_prefill].match_blocks = 0;
      best[p.pd_prefill].score = 0.0;
    }
  }
  for (uint32_t pi = 0; pi < p.P; ++pi) p.out[(uint64_t)r * p.P + pi] = best[pi];
}

// Per-batch constants of the non-prefix scorers (SURVEY.md Appendix A.4): eligibility
// words, clamp01'd kv / queue scores of the local endpoints, the best total of each profile when
// nothing matches, and the local endpoints that attain it (the tie set).  One CTA.
__global__ void __launch_bounds__(1024) prepare_endpoints_kernel(const EndpointDev* __restrict__ eps, uint32_t E_global,
                                                                 uint32_t ep_begin, uint32_t ep_count, ScoreTables st,
                                                                 double* __restrict__ sc, uint32_t* __restrict__ elig,
                                                                 ZeroBest* __restrict__ zero, uint32_t* __restrict__ ztie) {
  __shared__ int s_min[32], s_max[32];
  __shared__ double s_bs[32];
  __shared__ int s_minq, s_maxq;
  __shared__ double s_best;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t W = st.Epad / 32;
  for (uint32_t pi = 0; pi < st.n_profiles; ++pi) {
    const ProfileDev pr = st.prof[pi];
    // queue min/max over the eligible endpoints of the WHOLE pool
    int mn = INT_MAX, mx = INT_MIN;
    for (uint32_t e = tid; e < E_global; e += blockDim.x) {
      const EndpointDev s = eps[e];
      if (profile_admits(pr, s.flags, s.role_mask)) {
        mn = min(mn, s.queue_depth);
        mx = max(mx, s.queue_depth);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      mn = min(mn, __shfl_xor_sync(FULL, mn, d));
      mx = max(mx, __shfl_xor_sync(FULL, mx, d));
    }
    if (lane == 0) {
      s_min[warp] = mn;
      s_max[warp] = mx;
    }
    __syncthreads();
    if (tid == 0) {
      int a = INT_MAX, b = INT_MIN;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
        a = min(a, s_min[w]);
        b = max(b, s_max[w]);
      }
      s_minq = a;
      s_maxq = b;
    }
    __syncthreads();
    const int minq = s_minq, maxq = s_maxq;
    double* sc_p = sc + (uint64_t)pi * FI_EPP_MAX_SCORERS * st.Epad;
    // zero-match total of one local endpoint (the prefix scorer contributes 0·w); also fills the tables
    auto zero_total = [&](uint32_t e, bool* ok_out, bool store) -> double {
      bool ok = false;
      EndpointDev s;
      s.kv_util = 0.0;
      s.queue_depth = 0;
      s.role_mask = 0;
      s.flags = 0;
      if (e < ep_count) {
        s = eps[ep_begin + e];
        ok = profile_admits(pr, s.flags, s.role_mask);
      }
      double tot = 0.0;
      for (uint32_t k = 0; k < pr.n_scorers; ++k) {
        double v = 0.0;
        if (pr.kind[k] == FI_SCORER_KV_UTIL) {
          v = __dsub_rn(1.0, s.kv_util);
        } else if (pr.kind[k] == FI_SCORER_QUEUE) {
          v = (maxq == minq) ? 1.0
                             : __ddiv_rn((double)((long long)maxq - (long long)s.queue_depth),
                                         (double)((long long)maxq - (long long)minq));
        }
        v = v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v);
        if (!ok) v = 0.0;
        if (store) sc_p[(uint64_t)k * st.Epad + e] = v;
        tot = __dadd_rn(tot, __dmul_rn(v, pr.weight[k]));
      }
      *ok_out = ok;
      return tot;
    };
    double best = -1.0;  // totals are >= 0
    for (uint32_t e = tid; e < st.Epad; e += blockDim.x) {  // blockDim multiple of 32, Epad multiple of 32
      bool ok;
      const double tot = zero_total(e, &ok, true);
      const unsigned word = __ballot_sync(FULL, ok);
      if (lane == 0) elig[(uint64_t)pi * W + e / 32] = word;
      if (ok && tot > best) best = tot;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) best = fmax(best, __shfl_xor_sync(FULL, best, d));
    if (lane == 0) s_bs[warp] = best;
    __syncthreads();
    if (tid == 0) {
      double z = -1.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) z = fmax(z, s_bs[w]);
      s_best = z;
      ZeroBest zb;
      zb.any = z >= 0.0 ? 1u : 0u;
      zb.score = zb.any ? z : 0.0;
      zb.pad = 0;
      zero[pi] = zb;
    }
    __syncthreads();
    const double zbest = s_best;
    for (uint32_t e = tid; e < st.Epad; e += blockDim.x) {  // the tie set: same arithmetic, same bits
      bool ok;
      const double tot = zero_total(e, &ok, false);
      const unsigned word = __ballot_sync(FULL, ok && tot == zbest);
      if (lane == 0) ztie[(uint64_t)pi * W + e / 32] = word;
    }
    __syncthreads();
  }
}

// Handles on one device share the match variants, and different handles may launch from different threads at once
// (each handle's mutex covers only itself), so the variants' launch state is process-wide, under this one mutex.
std::mutex g_match_launch_mu;

// One instantiation per kernel variant: the shared-memory opt-in (cudaFuncSetAttribute) applies to one function
// only, and occupancy differs between variants, so each variant keeps its own state, per device.
template <bool WIN, int LPR, int VEC, bool LPM, bool LORA, bool RANKED, bool SUBSET = false, bool COUNTS = false,
          bool LISTS = false>
cudaError_t launch_match_variant(const MatchParams& p, int sm_count, cudaStream_t s) {
  const auto kern = WIN ? match_window_kernel<LPR, VEC, LPM, LORA, RANKED, SUBSET, COUNTS, LISTS>
                        : match_pick_kernel<LPR, VEC, LPM, LORA, RANKED, SUBSET, COUNTS, LISTS>;
  const size_t sp = WIN ? (size_t)kWindow : p.MP;  // entries per staging buffer
  size_t smem = (size_t)kWarps * sp * (2 * sizeof(uint64_t) + sizeof(uint32_t));  // 2 chain buffers + nodes
  if (COUNTS && !LISTS) smem += (size_t)kWarps * (p.st.Epad + 16) * sizeof(uint16_t);  // + the staging rows
  static std::map<int, size_t> opted_in;                // device -> the variant's max dynamic smem attribute
  static std::map<std::pair<int, size_t>, int> per_sm;  // (device, smem) -> resident CTAs per SM
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  int ctas_per_sm = 1;
  {
    std::lock_guard<std::mutex> lk(g_match_launch_mu);
    // The attribute is only ever raised: another handle may be launching this variant, on another thread, with the
    // larger size it opted in to, and lowering it under that launch would make the launch fail.
    size_t& attr = opted_in[dev];
    if (smem > 48 * 1024 && smem > attr) {
      e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      attr = smem;
    }
    auto it = per_sm.find({dev, smem});
    if (it == per_sm.end()) {
      int n = 0;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kWarps * 32, smem);
      if (e != cudaSuccess) return e;
      it = per_sm.emplace(std::make_pair(dev, smem), n < 1 ? 1 : n).first;
    }
    ctas_per_sm = it->second;
  }
  uint32_t grid = (p.R + kWarps - 1) / kWarps;
  const uint32_t cap = (uint32_t)sm_count * (uint32_t)ctas_per_sm;
  if (grid > cap) grid = cap;
  if (grid == 0) grid = 1;
  e = cudaMemsetAsync(p.work_counter, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  kern<<<grid, kWarps * 32, smem, s>>>(p);
  return cudaGetLastError();
}

template <int LPR, int VEC, bool WIN>
cudaError_t launch_match_t(const MatchParams& p, int sm_count, cudaStream_t s) {
  const bool lpm = p.lpm == FI_MATCH_LPM;
  if (p.lists)  // match lists (S.3b): the counts' walk, the lists' epilogue
    return lpm ? launch_match_variant<WIN, LPR, VEC, true, false, false, false, true, true>(p, sm_count, s)
               : launch_match_variant<WIN, LPR, VEC, false, false, false, false, true, true>(p, sm_count, s);
  if (p.counts)  // match counts (S.3a): no profile is scored
    return lpm ? launch_match_variant<WIN, LPR, VEC, true, false, false, false, true>(p, sm_count, s)
               : launch_match_variant<WIN, LPR, VEC, false, false, false, false, true>(p, sm_count, s);
  if (p.k && p.subsets)  // ranked pick over per-request candidate subsets
    return lpm ? launch_match_variant<WIN, LPR, VEC, true, false, true, true>(p, sm_count, s)
               : launch_match_variant<WIN, LPR, VEC, false, false, true, true>(p, sm_count, s);
  if (p.k)  // ranked pick: the LoRA scorer is handled at run time inside the variant
    return lpm ? launch_match_variant<WIN, LPR, VEC, true, false, true>(p, sm_count, s)
               : launch_match_variant<WIN, LPR, VEC, false, false, true>(p, sm_count, s);
  if (p.st.has_lora)
    return lpm ? launch_match_variant<WIN, LPR, VEC, true, true, false>(p, sm_count, s)
               : launch_match_variant<WIN, LPR, VEC, false, true, false>(p, sm_count, s);
  return lpm ? launch_match_variant<WIN, LPR, VEC, true, false, false>(p, sm_count, s)
             : launch_match_variant<WIN, LPR, VEC, false, false, false>(p, sm_count, s);
}

template <bool WIN>
cudaError_t launch_match_w(const MatchParams& p, int sm_count, cudaStream_t s) {
  // Words per row = LPR * VEC.  Two words per lane (half the counter registers of VEC = 4 -> three CTAs
  // = 24 warps per SM instead of 16): the kernel is bound by per-warp instruction latency and wants warps, not
  // wide loads (E = 1024, cfg 3 on one H100 SXM, 700 W: match_pick 74.5 us with two words per lane vs 98.1-98.4 us
  // with four, two runs each).
  switch (p.ix.W) {
    case 1: return launch_match_t<1, 1, WIN>(p, sm_count, s);
    case 2: return launch_match_t<1, 2, WIN>(p, sm_count, s);
    case 4: return launch_match_t<2, 2, WIN>(p, sm_count, s);
    case 8: return launch_match_t<4, 2, WIN>(p, sm_count, s);
    case 16: return launch_match_t<8, 2, WIN>(p, sm_count, s);
    case 32: return launch_match_t<16, 2, WIN>(p, sm_count, s);
    case 64: return launch_match_t<32, 2, WIN>(p, sm_count, s);
    case 128: return launch_match_t<32, 4, WIN>(p, sm_count, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t launch_match_pick(const MatchParams& p, int sm_count, cudaStream_t s) {
  if (p.R == 0) return cudaSuccess;
  // A handle whose chains can be longer than 1023 blocks runs the windowed variant: a count of 1024 or more needs
  // its 12 bit-planes, and a longer chain does not fit one staging buffer (DESIGN.md §4.9).
  if (p.max_blocks > (1u << NPLANES) - 1) return launch_match_w<true>(p, sm_count, s);
  return launch_match_w<false>(p, sm_count, s);
}

cudaError_t launch_merge_picks(const MergeParams& p, cudaStream_t s) {
  if (p.R == 0) return cudaSuccess;
  merge_picks_kernel<<<(p.R + 255) / 256, 256, 0, s>>>(p);
  return cudaGetLastError();
}

namespace {

// ---- the pack step of match lists (docs/SPEC.md S.3b), on the stream of the match launches it follows ------------------
// offsets[0] = 0, offsets[r + 1] = offsets[r] + nnz[r] in u64.  One CTA walks the requests in tiles of kScanPer per
// thread (16 384 requests per tile: one tile at cfg 3): each thread reads its kScanPer consecutive counts with 16-byte
// loads, all issued before any is used, a two-level shuffle scan over the CTA gives each thread its base, and each
// thread writes its run of offsets (nnz is 16-byte aligned).
constexpr int kScanPer = 16;
__global__ void __launch_bounds__(1024) list_scan_kernel(const uint32_t* __restrict__ nnz, uint32_t R,
                                                         uint64_t* __restrict__ offsets) {
  __shared__ uint64_t s_warp[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint64_t carry = 0;
  if (tid == 0) offsets[0] = 0;
  for (uint32_t base = 0; base < R; base += kScanPer * blockDim.x) {
    const uint32_t r = base + kScanPer * tid;
    uint32_t v[kScanPer];
#pragma unroll
    for (int q = 0; q < kScanPer; q += 4) {
      if (r + q + 3 < R) {
        const uint4 w = *reinterpret_cast<const uint4*>(nnz + r + q);
        v[q] = w.x;
        v[q + 1] = w.y;
        v[q + 2] = w.z;
        v[q + 3] = w.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[q + i] = r + q + i < R ? nnz[r + q + i] : 0u;
      }
    }
    uint64_t sum = 0;
#pragma unroll
    for (int i = 0; i < kScanPer; ++i) sum += v[i];
    uint64_t x = sum;  // inclusive scan over the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t o = __shfl_up_sync(FULL, x, d);
      if ((int)lane >= d) x += o;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint64_t w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint64_t o = __shfl_up_sync(FULL, w, d);
        if ((int)lane >= d) w += o;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    uint64_t at = carry + (warp ? s_warp[warp - 1] : 0) + x - sum;
#pragma unroll
    for (int i = 0; i < kScanPer; ++i) {
      at += v[i];
      if (r + i < R) offsets[r + i + 1] = at;
    }
    carry += s_warp[31];
    __syncthreads();  // s_warp is read above before the next tile writes it
  }
}

// One warp per request: the entries of its slot at list positions [offsets[r], offsets[r + 1]) within [lo, hi) go to
// out[position - lo], widened to fi_match_entry with the global endpoint.  Positions past hi are not written.
__global__ void __launch_bounds__(256) list_copy_kernel(const uint32_t* __restrict__ lists, uint32_t pitch,
                                                        const uint64_t* __restrict__ offsets, uint32_t R, uint32_t ep_begin,
                                                        uint64_t lo, uint64_t hi, fi_match_entry* __restrict__ out) {
  const uint32_t r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  const uint64_t a = offsets[r], b = offsets[r + 1];
  const uint64_t e = b < hi ? b : hi;
  const uint32_t* src = lists + (uint64_t)r * pitch;
  for (uint64_t pos = (a > lo ? a : lo) + lane; pos < e; pos += 32) {
    const uint32_t v = src[pos - a];
    fi_match_entry m;
    m.endpoint = ep_begin + (v >> 12);
    m.match_blocks = (uint16_t)(v & 0xFFFu);
    m.reserved = 0;
    out[pos - lo] = m;
  }
}

}  // namespace

cudaError_t launch_list_scan(const uint32_t* nnz, uint32_t R, uint64_t* offsets, cudaStream_t s) {
  list_scan_kernel<<<1, 1024, 0, s>>>(nnz, R, offsets);
  return cudaGetLastError();
}

cudaError_t launch_list_copy(const uint32_t* lists, uint32_t pitch, const uint64_t* offsets, uint32_t R, uint32_t ep_begin,
                             uint64_t lo, uint64_t hi, fi_match_entry* out, cudaStream_t s) {
  if (R == 0 || hi <= lo) return cudaSuccess;
  list_copy_kernel<<<(R + 7) / 8, 256, 0, s>>>(lists, pitch, offsets, R, ep_begin, lo, hi, out);
  return cudaGetLastError();
}

cudaError_t launch_prepare_endpoints(const EndpointDev* eps, uint32_t E_global, uint32_t ep_begin, uint32_t ep_count,
                                     ScoreTables st, double* sc, uint32_t* elig, ZeroBest* zero, uint32_t* ztie,
                                     cudaStream_t s) {
  prepare_endpoints_kernel<<<1, 1024, 0, s>>>(eps, E_global, ep_begin, ep_count, st, sc, elig, zero, ztie);
  return cudaGetLastError();
}

}  // namespace fi
