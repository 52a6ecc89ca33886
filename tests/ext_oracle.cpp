// ext_oracle.cpp — the CPU oracle's test-side extension, test infrastructure only.
//
// It compiles the CPU oracle (oracle/epp_oracle.cpp) into the same translation unit and adds, from the oracle's own
// hashing, index, eligibility, scoring and tie-rotation pieces:
//   * the ranked pick (docs/SPEC.md S.6a), over each request's candidate subset (S.5a) when one is given;
//   * per-endpoint LRU capacities (S.2b): a capacity c_e per endpoint, an indexer.Add that evicts against it, the
//     resize of fi_epp_set_lru_capacities, and the LRU's content for comparisons;
//   * the shard view (S.2e): a handle over endpoints [lo, lo + cnt) of the pool.  Its Adds and capacity changes skip
//     the other endpoints, and its ranked pick ranks only its own endpoints, with the queue scorer's min / max still
//     taken over the whole pool.  (Index ops addressed elsewhere are dropped by the wrapper, tests/ext_oracle.py.)
//   * the match counts of fi_epp_match_counts (S.3a), from the ranked pick's own walk;
//   * the per-endpoint part of fi_epp_resize_pool (S.2c);
//   * the state of an index snapshot (S.2d), read and written whole: the pair set, every endpoint's capacity and,
//     with the LRU lists of epx_lru_dump, epx_load_state, which replaces all three.
// The handle is the oracle's own plus the capacities, so every epo_* function of the oracle works on it too.  The
// oracle itself is left as it is: its single pick stays the yardstick of fi_epp_pick_batch.
#include "../oracle/epp_oracle.cpp"

namespace {

struct ExtOracle : Oracle {
  std::vector<uint32_t> cap;  // [num_endpoints] c_e, lru_capacity until set
  uint32_t lo = 0, cnt = 0;   // the shard [lo, lo + cnt): the whole pool unless epx_set_shard narrowed it
  bool mine(uint32_t e) const { return e - lo < cnt; }
};

inline ExtOracle* ext_of(void* h) { return static_cast<ExtOracle*>(static_cast<Oracle*>(h)); }

struct Ranked {
  double total;
  uint32_t dist;  // tie rotation distance (smaller first among equal totals)
  uint32_t e;
  uint32_t match;
};

inline bool in_subset(const uint32_t* row, uint32_t e) { return !row || ((row[e >> 5] >> (e & 31)) & 1u); }

// One request: hash → match (A.3) over the WHOLE index, exactly as pick_one does (the walk stops at the first block
// no endpoint of the index holds, whatever the subset; a shard view's index holds its own endpoints only).  Then per
// profile: the eligible endpoints of the subset (of the pool when row is NULL), the queue scorer's min / max over them
// (S.4 per request; make_ctx's set without a row), the totals (A.4) of those inside the shard, partially sorted by
// (total desc, rotation distance asc), the order whose first element is pick_one's pick, and the PD rule on the
// decode profile's entry 0 (A.6) applied to the prefill profile's whole list.
void rank_one(const ExtOracle& o, const uint8_t* prompt, uint64_t len, uint64_t h0, uint64_t adapter, const uint32_t* row,
              uint32_t r, uint32_t k, fi_pick* out, Scratch& sc, std::vector<Ranked>& cand) {
  const fi_epp_config& cfg = o.cfg;
  const uint32_t E = cfg.num_endpoints;
  sc.chain.resize(cfg.max_blocks);
  const uint32_t n = hash_prompt(prompt, len, h0, cfg.block_bytes, cfg.max_blocks, sc.chain.data(), sc.tmp);
  if (sc.match.size() != E) sc.match.assign(E, 0);
  sc.touched.clear();
  if (cfg.match_mode == FI_MATCH_UPSTREAM) {
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t* m = nullptr;
      const uint32_t cnt = o.index.get(sc.chain[i], &m);
      if (cnt == 0) break;
      for (uint32_t j = 0; j < cnt; ++j)
        if (sc.match[m[j]]++ == 0) sc.touched.push_back(m[j]);
    }
  } else {
    sc.alive.clear();
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t* m = nullptr;
      const uint32_t cnt = o.index.get(sc.chain[i], &m);
      if (cnt == 0) break;
      if (i == 0) {
        sc.alive.assign(m, m + cnt);
      } else {
        sc.alive2.clear();
        for (uint32_t a : sc.alive)
          if (std::find(m, m + cnt, a) != m + cnt) sc.alive2.push_back(a);
        sc.alive.swap(sc.alive2);
      }
      if (sc.alive.empty()) break;
      for (uint32_t a : sc.alive)
        if (sc.match[a]++ == 0) sc.touched.push_back(a);
    }
  }

  const uint32_t start = tie_rotation_start(n, n ? sc.chain[0] : 0, h0, r, E);
  for (uint32_t p = 0; p < cfg.n_profiles; ++p) {
    const fi_profile& prof = cfg.profiles[p];
    ProfileCtx ctx;  // make_ctx over the request's eligible candidates
    cand.clear();
    for (uint32_t e = 0; e < E; ++e) {
      if (!eligible(o.eps[e], prof) || !in_subset(row, e)) continue;
      const int32_t q = o.eps[e].queue_depth;
      ctx.min_q = ctx.any ? std::min(ctx.min_q, q) : q;
      ctx.max_q = ctx.any ? std::max(ctx.max_q, q) : q;
      ctx.any = true;
      if (o.mine(e)) cand.push_back({0.0, tie_distance(e, start, E), e, sc.match[e]});
    }
    for (Ranked& c : cand) c.total = total_score(prof, ctx, o.eps[c.e], c.match, n, adapter);
    const size_t kk = std::min<size_t>(k, cand.size());
    std::partial_sort(cand.begin(), cand.begin() + kk, cand.end(), [](const Ranked& a, const Ranked& b) {
      return a.total > b.total || (a.total == b.total && a.dist < b.dist);
    });
    for (uint32_t j = 0; j < k; ++j) {
      fi_pick& pk = out[(size_t)p * k + j];
      pk.n_blocks = (uint16_t)n;
      if (j < kk) {
        pk.endpoint = cand[j].e;
        pk.match_blocks = (uint16_t)cand[j].match;
        pk.score = cand[j].total;
      } else {
        pk.endpoint = FI_NO_ENDPOINT;
        pk.match_blocks = 0;
        pk.score = 0.0;
      }
    }
  }
  if (cfg.pd_enabled) {
    const fi_pick& d = out[(size_t)cfg.pd_decode_profile * k];
    const double hit = (d.endpoint != FI_NO_ENDPOINT && n) ? (double)d.match_blocks / (double)n : 0.0;
    const double miss_bytes = (1.0 - hit) * (double)len;
    if (!(miss_bytes >= cfg.pd_threshold)) {
      for (uint32_t j = 0; j < k; ++j) {
        fi_pick& pf = out[(size_t)cfg.pd_prefill_profile * k + j];
        pf.endpoint = FI_NO_ENDPOINT;
        pf.match_blocks = 0;
        pf.score = 0.0;
      }
    }
  }
  for (uint32_t e : sc.touched) sc.match[e] = 0;
}

// evict e's least recently used keys until it holds at most c_e, CLEARing each pair; emit(hash) oldest first
template <class Emit>
void shrink_to_cap(ExtOracle* o, uint32_t e, Emit&& emit) {
  PodLRU& l = o->lrus[e];
  while (l.order.size() > o->cap[e]) {
    const uint64_t old = l.order.back();
    l.order.pop_back();
    l.pos.erase(old);
    o->index.clear(old, e);
    emit(old);
  }
}

// The oracle's index keeps its slots private.  An explicit instantiation may name a private member, which lets the pair
// enumeration read them without changing the oracle.
using SlotsMember = std::vector<Slot> PodIndex::*;
SlotsMember slots_member();
template <SlotsMember M>
struct SlotsAccess {
  friend SlotsMember slots_member() { return M; }
};
template struct SlotsAccess<&PodIndex::slots_>;

template <class Visit>
void for_each_pair(const ExtOracle& o, Visit&& visit) {
  for (const Slot& s : o.index.*slots_member()) {
    if (!s.used) continue;
    const uint32_t* m = s.ext ? s.ext->data() : s.inl;
    for (uint32_t j = 0; j < s.n; ++j) visit(s.key, m[j]);
  }
}

// a resize or a load needs a handle over the whole pool (the product's check_whole_pool)
inline bool whole_pool(const ExtOracle& o) { return o.lo == 0 && o.cnt == o.cfg.num_endpoints; }

}  // namespace

extern "C" {

// epo_create's handle plus c_e = lru_capacity for every endpoint.  lru_capacity = 0 is accepted, as epo_create
// accepts it (the pick tests use such configurations); the capacity calls below return FI_ERR_STATE on that handle.
void* epx_create(const fi_epp_config* cfg) {
  std::string err;
  if (!cfg || !validate(*cfg, err)) {
    std::fprintf(stderr, "epx_create: %s\n", err.c_str());
    return nullptr;
  }
  ExtOracle* o = new ExtOracle();
  o->cfg = *cfg;
  o->eps.assign(cfg->num_endpoints, EpState{});
  if (cfg->lru_capacity) o->lrus.resize(cfg->num_endpoints);
  o->cap.assign(cfg->num_endpoints, cfg->lru_capacity);
  o->cnt = cfg->num_endpoints;
  return static_cast<Oracle*>(o);
}

void epx_destroy(void* h) { delete ext_of(h); }

// Narrow a fresh handle to the shard view over endpoints [begin, begin + count) (docs/SPEC.md S.2e).  FI_ERR_INVALID
// for a range that is empty or leaves the pool.
int epx_set_shard(void* h, uint32_t begin, uint32_t count) {
  ExtOracle* o = ext_of(h);
  if (count == 0 || (uint64_t)begin + count > o->cfg.num_endpoints) return FI_ERR_INVALID;
  o->lo = begin;
  o->cnt = count;
  return FI_OK;
}

// subsets: R rows of ceil(num_endpoints / 32) words (bit e of row r: e is a candidate of request r), or NULL (every
// request ranks the whole pool).  out: R*n_profiles*k picks, out[(r*n_profiles + p)*k + j] = rank j of profile p;
// adapters may be NULL (id 0).
int epx_pick_batch_ranked(void* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                          const uint64_t* adapters, const uint32_t* subsets, uint32_t R, uint32_t k, fi_pick* out) {
  if (!h || k == 0) return FI_ERR_INVALID;
  const ExtOracle* o = ext_of(h);
  const uint32_t P = o->cfg.n_profiles;
  const size_t pitch = (o->cfg.num_endpoints + 31) / 32;
  Scratch sc;
  std::vector<Ranked> cand;
  for (uint32_t r = 0; r < R; ++r)
    rank_one(*o, prompts + offsets[r], offsets[r + 1] - offsets[r], h0[r], adapters ? adapters[r] : 0,
             subsets ? subsets + r * pitch : nullptr, r, k, out + (size_t)r * P * k, sc, cand);
  return FI_OK;
}

// upstream indexer.Add(hashes, pod) against the pod's own capacity (S.2 with c_e, S.2b): epo_index_add_chain with
// lru_capacity replaced by c_e, so with every c_e at lru_capacity it makes the same changes step for step.  An Add
// to an endpoint outside the shard changes nothing.
int epx_add_chain(void* h, uint32_t endpoint, const uint64_t* hashes, uint32_t n) {
  ExtOracle* o = ext_of(h);
  if (!o->cfg.lru_capacity) return FI_ERR_STATE;
  if (endpoint >= o->cfg.num_endpoints) return FI_ERR_INVALID;
  if (!o->mine(endpoint)) return FI_OK;
  PodLRU& l = o->lrus[endpoint];
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t k = hashes[i];
    auto it = l.pos.find(k);
    if (it != l.pos.end()) {
      l.order.splice(l.order.begin(), l.order, it->second);
      continue;
    }
    l.order.push_front(k);
    l.pos[k] = l.order.begin();
    o->index.set(k, endpoint);
    if (l.order.size() > o->cap[endpoint]) {
      const uint64_t old = l.order.back();
      l.order.pop_back();
      l.pos.erase(old);
      o->index.clear(old, endpoint);
    }
  }
  return FI_OK;
}

// a batch of decisions, sequentially in request order
int epx_add_chains(void* h, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch, const uint32_t* nblocks,
                   uint32_t R) {
  if (!ext_of(h)->cfg.lru_capacity) return FI_ERR_STATE;
  for (uint32_t r = 0; r < R; ++r) {
    if (endpoints[r] == FI_NO_ENDPOINT || nblocks[r] == 0) continue;
    const int rc = epx_add_chain(h, endpoints[r], chains + (size_t)r * pitch, nblocks[r]);
    if (rc != FI_OK) return rc;
  }
  return FI_OK;
}

// fi_epp_set_lru_capacities (S.2b): c_e = capacities[i] (0: lru_capacity; the last entry of an endpoint wins), then
// each listed endpoint, in order of first appearance, evicts down to c_e.  The evicted pairs are written to
// ev_hash / ev_ep (at most ev_cap), oldest first per endpoint; *n_evicted = how many.  FI_ERR_INVALID (nothing
// changes) for an endpoint >= num_endpoints, a capacity above lru_capacity or one in (0, max_blocks).  Endpoints
// outside the shard are checked, then ignored.
int epx_set_lru_capacities(void* h, const uint32_t* endpoints, const uint32_t* capacities, uint32_t n,
                           uint64_t* ev_hash, uint32_t* ev_ep, uint64_t ev_cap, uint64_t* n_evicted) {
  ExtOracle* o = ext_of(h);
  const uint32_t C = o->cfg.lru_capacity;
  *n_evicted = 0;
  if (!C) return FI_ERR_STATE;
  for (uint32_t i = 0; i < n; ++i)
    if (endpoints[i] >= o->cfg.num_endpoints || capacities[i] > C || (capacities[i] && capacities[i] < o->cfg.max_blocks))
      return FI_ERR_INVALID;
  std::vector<uint32_t> order;
  std::vector<uint8_t> listed(o->cfg.num_endpoints, 0);
  for (uint32_t i = 0; i < n; ++i) {
    if (!o->mine(endpoints[i])) continue;
    o->cap[endpoints[i]] = capacities[i] ? capacities[i] : C;
    if (!listed[endpoints[i]]) {
      listed[endpoints[i]] = 1;
      order.push_back(endpoints[i]);
    }
  }
  uint64_t m = 0;
  for (uint32_t e : order)
    shrink_to_cap(o, e, [&](uint64_t k) {
      if (m < ev_cap) {
        ev_hash[m] = k;
        ev_ep[m] = e;
      }
      ++m;
    });
  *n_evicted = m;
  return FI_OK;
}

// e's LRU, least recently used first (at most cap written); returns its size (0 on a handle without LRUs)
uint32_t epx_lru_dump(void* h, uint32_t e, uint64_t* out, uint32_t cap) {
  const ExtOracle* o = ext_of(h);
  if (e >= o->lrus.size()) return 0;
  const PodLRU& l = o->lrus[e];
  uint32_t i = 0;
  for (auto it = l.order.rbegin(); it != l.order.rend(); ++it, ++i)
    if (i < cap) out[i] = *it;
  return (uint32_t)l.order.size();
}

// the LRU part of upstream indexer.RemovePod (S.2a): e's LRU becomes empty, its capacity stays
int epx_lru_clear(void* h, uint32_t e) {
  ExtOracle* o = ext_of(h);
  if (!o->cfg.lru_capacity) return FI_ERR_STATE;
  if (e >= o->cfg.num_endpoints) return FI_ERR_INVALID;
  o->lrus[e].order.clear();
  o->lrus[e].pos.clear();
  return FI_OK;
}

// fi_epp_match_counts (S.3a): counts[r * cnt + j] = match[lo + j] of request r, nblocks[r] = N.  For the call the
// handle's configuration is one profile without filters or PD and its endpoints are all alive, so rank_one's one
// list holds every endpoint of the shard; configuration and states are restored before the call returns.  The count
// reads neither, as S.3a says.  A probe that makes every endpoint a candidate and ranks all of the shard's endpoints
// reports each one's match_blocks, so the walk of S.3 is the one the ranked and subset tests already check.
int epx_match_counts(void* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                     uint16_t* counts, uint32_t* nblocks) {
  if (!h) return FI_ERR_INVALID;
  ExtOracle* o = ext_of(h);
  const fi_epp_config saved_cfg = o->cfg;
  std::vector<EpState> saved_eps;
  saved_eps.swap(o->eps);
  o->eps.assign(saved_cfg.num_endpoints, EpState{});
  for (EpState& s : o->eps) s.flags = FI_ENDPOINT_ALIVE;
  fi_profile probe{};
  probe.n_scorers = 1;
  probe.scorers[0].kind = FI_SCORER_PREFIX;
  probe.scorers[0].weight = 1;
  o->cfg.n_profiles = 1;
  o->cfg.profiles[0] = probe;
  o->cfg.pd_enabled = 0;
  Scratch sc;
  std::vector<Ranked> cand;
  std::vector<fi_pick> list(o->cnt);
  for (uint32_t r = 0; r < R; ++r) {
    rank_one(*o, prompts + offsets[r], offsets[r + 1] - offsets[r], h0[r], 0, nullptr, r, o->cnt, list.data(), sc, cand);
    for (const fi_pick& pk : list) counts[(size_t)r * o->cnt + (pk.endpoint - o->lo)] = pk.match_blocks;
    nblocks[r] = list[0].n_blocks;
  }
  o->cfg = saved_cfg;
  o->eps.swap(saved_eps);
  return FI_OK;
}

// fi_epp_resize_pool (S.2c) on the oracle's per-endpoint state: endpoints [E', E) are truncated away, [E, E') are
// appended fresh (not alive, no adapters, an empty LRU of capacity lru_capacity), and E becomes E'.  A shrink's index
// pairs are the caller's to remove first (ExtOracle.resize: remove_endpoints of the tail).  FI_ERR_STATE on a shard
// view, as the product refuses a handle over part of the pool.
int epx_resize(void* h, uint32_t num_endpoints) {
  ExtOracle* o = ext_of(h);
  if (!whole_pool(*o)) return FI_ERR_STATE;
  if (num_endpoints == 0 || num_endpoints > 4096) return FI_ERR_INVALID;
  const uint32_t keep = std::min(o->cfg.num_endpoints, num_endpoints);
  o->eps.resize(keep);
  o->eps.resize(num_endpoints, EpState{});
  if (o->cfg.lru_capacity) {
    o->lrus.resize(keep);
    o->lrus.resize(num_endpoints);
  }
  o->cap.resize(keep);
  o->cap.resize(num_endpoints, o->cfg.lru_capacity);
  o->cfg.num_endpoints = o->cfg.endpoint_count = num_endpoints;
  o->cnt = num_endpoints;  // (a resized handle covers the whole pool: lo is 0)
  return FI_OK;
}

// the pair set: (hashes[i], endpoints[i]) for i < the returned count (at most cap written), in no particular order
uint64_t epx_index_pairs(void* h, uint64_t* hashes, uint32_t* endpoints, uint64_t cap) {
  uint64_t n = 0;
  for_each_pair(*ext_of(h), [&](uint64_t key, uint32_t e) {
    if (n < cap) {
      hashes[n] = key;
      endpoints[n] = e;
    }
    ++n;
  });
  return n;
}

// every endpoint's LRU capacity c_e (0 without an LRU)
int epx_lru_capacities(void* h, uint32_t* out) {
  ExtOracle* o = ext_of(h);
  for (uint32_t e = 0; e < o->cfg.num_endpoints; ++e) out[e] = o->cfg.lru_capacity ? o->cap[e] : 0;
  return FI_OK;
}

// Replace the state of S.2d: the pair set becomes the n pairs (hashes[i], endpoints[i]); endpoint e's LRU becomes its
// lens[e] keys, least recently used first, taken in endpoint order from `keys`; its capacity becomes caps[e].
// Endpoint states and adapters are left as they are.  FI_ERR_STATE on a shard view, as for epx_resize.
int epx_load_state(void* h, uint64_t n, const uint64_t* hashes, const uint32_t* endpoints, const uint32_t* lens,
                   const uint64_t* keys, const uint32_t* caps) {
  ExtOracle* o = ext_of(h);
  if (!whole_pool(*o)) return FI_ERR_STATE;
  const uint32_t E = o->cfg.num_endpoints;
  for (uint64_t i = 0; i < n; ++i)
    if (endpoints[i] >= E) return FI_ERR_INVALID;
  std::vector<std::pair<uint64_t, uint32_t>> old;
  for_each_pair(*o, [&](uint64_t key, uint32_t e) { old.emplace_back(key, e); });
  for (const auto& p : old) o->index.clear(p.first, p.second);
  for (uint64_t i = 0; i < n; ++i) o->index.set(hashes[i], endpoints[i]);
  if (!o->cfg.lru_capacity) return FI_OK;
  for (uint32_t e = 0; e < E; ++e) {
    PodLRU& l = o->lrus[e];
    l.order.clear();
    l.pos.clear();
    for (uint32_t j = 0; j < lens[e]; ++j) {  // oldest first: each key goes in front of the older ones
      l.order.push_front(*keys++);
      l.pos[l.order.front()] = l.order.begin();
    }
    o->cap[e] = caps[e];
  }
  return FI_OK;
}

}  // extern "C"
