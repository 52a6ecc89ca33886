// lru_plan.h — host-side planning of one batch of indexer.Add calls for the DEVICE-resident LRU
// (lru_kernels.cu).  Pure C++ (unit-tested on the CPU through hostcheck.cpp).
//
// Upstream's PreRequest step is indexer.Add(chain_r, pod_r) for every routed request, in request order
// (SURVEY.md Appendix A.2; capacity lruCapacityPerServer, /root/reference/pkg/router/strategy.go:59,149).
// The device LRU applies a whole SUB-BATCH of those at once, which is exact as long as an endpoint's LRU
// never receives more than `cap_per_endpoint` touches within one sub-batch (then nothing touched in the
// sub-batch can be evicted before its end: an LRU of capacity C always holds the C most recently touched
// distinct keys).  The planner cuts the request stream — in request order — into such sub-batches and lays out,
// per sub-batch, what the kernels need:
//   req_id[k]    index of the k-th kept request in the caller's arrays (ascending)
//   req_ep[k]    its LOCAL endpoint
//   req_n[k]     its block count
//   req_off[k]   exclusive prefix sum of req_n within the sub-batch (position of its first touch)
//   ep_start[e] .. ep_start[e+1]  range of ep_list holding the k's of local endpoint e, ascending
//   inc[e]       touches endpoint e receives in the sub-batch (upper bound of its new log records)
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

namespace fi {

// Touches one endpoint may receive in a sub-batch so that the touch kernel can never find its table full: the bound
// fi_epp_index_add_submitted plans with (it has no overflow readback).  Per endpoint, with `add` touches in the
// sub-batch (so at most `add` new keys, and at most `add` slot reservations outstanding at any time), table size TS,
// capacity C and used = regular slots taken (entries + tombstones), lru_maintain_kernel (lru_kernels.cu) leaves
//   either the table as it is, only if (used + min(add, C)) * 10 <= 6 TS, i.e. used <= calm - min(add, C),
//   or a table rebuilt from the live entries: used = count <= C (evict ran at the end of the previous sub-batch),
// and a new key is inserted only while used < limit = TS * 85 / 100 (integer division, as alloc_dev_lru computes it;
// calm = TS * 6 / 10 likewise).  The touch kernel cannot overflow iff used + add <= limit:
//   add <= C:  calm <= limit, and C + add <= 2 C <= limit (TS >= 4 C): always;
//   add > C:   add <= limit - calm + C (table kept) and add <= limit - C (table rebuilt).
// The bound is the smaller of the two, >= 2 C since TS >= 4 C, so every chain (at most C blocks) fits.
// C is the uniform lru_capacity even when endpoints have capacities of their own (fi_epp_set_lru_capacities): every
// c_e <= C, and the argument only uses C as an upper bound on an endpoint's entries (count <= c_e <= C after a
// rebuild), so it holds unchanged.  Resize evictions only turn entries into tombstones, which `used` already counts.
inline uint32_t lru_touch_bound(uint32_t TS, uint32_t C) {
  const uint64_t limit = (uint64_t)TS * 85 / 100, calm = (uint64_t)TS * 6 / 10;
  return (uint32_t)std::min<uint64_t>(limit - calm + C, limit - C);
}

struct LruSubBatch {
  uint32_t k_begin = 0, k_end = 0;  // range of the kept-request arrays
  uint64_t touches = 0;             // sum of req_n over the range
};

struct LruPlan {
  std::vector<uint32_t> req_id, req_ep, req_n, req_off;  // [K]   (req_off restarts at 0 in every sub-batch)
  std::vector<uint32_t> ep_list;                         // [K]   k relative to the sub-batch's k_begin
  std::vector<uint32_t> ep_start;                        // [nsub][EL + 1]
  std::vector<uint32_t> inc;                             // [nsub][EL]
  std::vector<LruSubBatch> subs;
};

// endpoints[r] is a GLOBAL endpoint index (or any value outside [ep_begin, ep_begin + EL): skipped, like
// FI_NO_ENDPOINT and requests with no blocks).  A request with more than cap_per_endpoint blocks cannot be
// planned (the caller rejects it first).  cap_touches / cap_requests bound a sub-batch by the size of the
// device scratch arrays.
inline void lru_plan_batch(const uint32_t* endpoints, const uint32_t* nblocks, uint32_t R, uint32_t ep_begin, uint32_t EL,
                           uint32_t cap_per_endpoint, uint64_t cap_touches, uint32_t cap_requests, LruPlan* out) {
  LruPlan& p = *out;
  p.req_id.clear();
  p.req_ep.clear();
  p.req_n.clear();
  p.req_off.clear();
  p.ep_list.clear();
  p.ep_start.clear();
  p.inc.clear();
  p.subs.clear();
  std::vector<uint32_t> acc(EL, 0);
  std::vector<uint32_t> touched;  // endpoints with acc != 0 in the open sub-batch
  LruSubBatch cur;
  auto close = [&]() {
    if (cur.k_end == cur.k_begin) return;
    // bucket the sub-batch's requests by endpoint (counting sort keeps k ascending within an endpoint)
    const size_t s0 = p.ep_start.size();
    p.ep_start.resize(s0 + EL + 1, 0);
    uint32_t* st = p.ep_start.data() + s0;
    for (uint32_t k = cur.k_begin; k < cur.k_end; ++k) st[p.req_ep[k] + 1]++;
    for (uint32_t e = 0; e < EL; ++e) st[e + 1] += st[e];
    const size_t l0 = p.ep_list.size();
    p.ep_list.resize(l0 + (cur.k_end - cur.k_begin));
    std::vector<uint32_t> fill(st, st + EL);
    for (uint32_t k = cur.k_begin; k < cur.k_end; ++k) p.ep_list[l0 + fill[p.req_ep[k]]++] = k - cur.k_begin;
    const size_t i0 = p.inc.size();
    p.inc.resize(i0 + EL, 0);
    for (uint32_t e : touched) {
      p.inc[i0 + e] = acc[e];
      acc[e] = 0;
    }
    touched.clear();
    p.subs.push_back(cur);
    cur.k_begin = cur.k_end;
    cur.touches = 0;
  };
  for (uint32_t r = 0; r < R; ++r) {
    const uint32_t e = endpoints[r] - ep_begin;
    const uint32_t n = nblocks[r];
    if (e >= EL || n == 0) continue;
    if (acc[e] + (uint64_t)n > cap_per_endpoint || cur.touches + n > cap_touches || cur.k_end - cur.k_begin >= cap_requests)
      close();
    if (acc[e] == 0) touched.push_back(e);
    acc[e] += n;
    p.req_id.push_back(r);
    p.req_ep.push_back(e);
    p.req_n.push_back(n);
    p.req_off.push_back((uint32_t)cur.touches);
    cur.touches += n;
    cur.k_end++;
  }
  close();
}

// The plan as the LRU kernels read it: one u32 array (one H2D copy per call), the vectors of LruPlan back to back,
//   req_id[K] | req_ep[K] | req_n[K] | req_off[K] | ep_list[K] | ep_start[nsub][EL + 1] | inc[nsub][EL]
inline size_t lru_plan_words(const LruPlan& p, uint32_t EL) {
  return 5 * p.req_id.size() + p.subs.size() * ((size_t)2 * EL + 1);
}

// dst: lru_plan_words(p, EL) words (an empty plan writes none).  Packing the vectors back to back gives the layout
// above because lru_plan_batch sizes ep_start [nsub][EL + 1] and inc [nsub][EL] (fihc_lru_plan_pack_check holds the
// packer and lru_plan_offsets to each other).
inline void lru_plan_pack(const LruPlan& p, uint32_t* dst) {
  for (const std::vector<uint32_t>* v : {&p.req_id, &p.req_ep, &p.req_n, &p.req_off, &p.ep_list, &p.ep_start, &p.inc}) {
    if (v->empty()) continue;
    std::memcpy(dst, v->data(), v->size() * sizeof(uint32_t));
    dst += v->size();
  }
}

// where sub-batch sb's arrays start in the packed plan, in words
struct LruPlanOffsets {
  size_t req_id, req_ep, req_n, req_off, ep_list, ep_start, inc;
};

inline LruPlanOffsets lru_plan_offsets(const LruPlan& p, uint32_t EL, size_t sb) {
  const size_t K = p.req_id.size(), nsub = p.subs.size(), k0 = p.subs[sb].k_begin;
  LruPlanOffsets o;
  o.req_id = k0;
  o.req_ep = K + k0;
  o.req_n = 2 * K + k0;
  o.req_off = 3 * K + k0;
  o.ep_list = 4 * K + k0;
  o.ep_start = 5 * K + sb * ((size_t)EL + 1);
  o.inc = 5 * K + nsub * ((size_t)EL + 1) + sb * EL;
  return o;
}

}  // namespace fi
