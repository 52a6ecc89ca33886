// capacity_oracle.cpp — CPU reference of per-endpoint LRU capacities (docs/SPEC.md S.2b), test infrastructure only.
//
// It compiles the CPU oracle (oracle/epp_oracle.cpp) into the same translation unit and adds what S.2b needs: every
// endpoint's LRU capacity c_e (CapOracle), an indexer.Add that evicts against c_e, the resize of
// fi_epp_set_lru_capacities, and the LRU's content for comparisons.  The Add is the oracle's epo_index_add_chain with
// lru_capacity replaced by c_e, so with every c_e at lru_capacity it makes the same changes step for step.  The handle
// is the oracle's own, so every epo_* function of the oracle (picks, index ops, membership) works on it.  The oracle
// itself is left as it is.
#include "../oracle/epp_oracle.cpp"

namespace {

struct CapOracle : Oracle {
  std::vector<uint32_t> cap;  // [num_endpoints] c_e
};

inline CapOracle* cap_of(void* h) { return static_cast<CapOracle*>(static_cast<Oracle*>(h)); }

// evict e's least recently used keys until it holds at most c_e, CLEARing each pair; emit(hash) oldest first
template <class Emit>
void shrink_to_cap(CapOracle* o, uint32_t e, Emit&& emit) {
  PodLRU& l = o->lrus[e];
  while (l.order.size() > o->cap[e]) {
    const uint64_t old = l.order.back();
    l.order.pop_back();
    l.pos.erase(old);
    o->index.clear(old, e);
    emit(old);
  }
}

}  // namespace

extern "C" {

void* epo_cap_create(const fi_epp_config* cfg) {
  std::string err;
  if (!cfg || !validate(*cfg, err) || !cfg->lru_capacity) {
    std::fprintf(stderr, "epo_cap_create: %s\n", err.empty() ? "lru_capacity is 0" : err.c_str());
    return nullptr;
  }
  CapOracle* o = new CapOracle();
  o->cfg = *cfg;
  o->eps.assign(cfg->num_endpoints, EpState{});
  o->lrus.resize(cfg->num_endpoints);
  o->cap.assign(cfg->num_endpoints, cfg->lru_capacity);
  return static_cast<Oracle*>(o);
}

void epo_cap_destroy(void* h) { delete cap_of(h); }

// upstream indexer.Add(hashes, pod) against the pod's own capacity (S.2 with c_e, S.2b)
int epo_cap_add_chain(void* h, uint32_t endpoint, const uint64_t* hashes, uint32_t n) {
  CapOracle* o = cap_of(h);
  if (endpoint >= o->cfg.num_endpoints) return FI_ERR_INVALID;
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
int epo_cap_add_chains(void* h, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch, const uint32_t* nblocks,
                       uint32_t R) {
  for (uint32_t r = 0; r < R; ++r) {
    if (endpoints[r] == FI_NO_ENDPOINT || nblocks[r] == 0) continue;
    const int rc = epo_cap_add_chain(h, endpoints[r], chains + (size_t)r * pitch, nblocks[r]);
    if (rc != FI_OK) return rc;
  }
  return FI_OK;
}

// fi_epp_set_lru_capacities (S.2b): c_e = capacities[i] (0: lru_capacity; the last entry of an endpoint wins), then
// each listed endpoint, in order of first appearance, evicts down to c_e.  The evicted pairs are written to
// ev_hash / ev_ep (at most ev_cap), oldest first per endpoint; *n_evicted = how many.  FI_ERR_INVALID (nothing
// changes) for an endpoint >= num_endpoints, a capacity above lru_capacity or one in (0, max_blocks).
int epo_cap_set_lru_capacities(void* h, const uint32_t* endpoints, const uint32_t* capacities, uint32_t n,
                               uint64_t* ev_hash, uint32_t* ev_ep, uint64_t ev_cap, uint64_t* n_evicted) {
  CapOracle* o = cap_of(h);
  const uint32_t C = o->cfg.lru_capacity;
  *n_evicted = 0;
  for (uint32_t i = 0; i < n; ++i)
    if (endpoints[i] >= o->cfg.num_endpoints || capacities[i] > C || (capacities[i] && capacities[i] < o->cfg.max_blocks))
      return FI_ERR_INVALID;
  std::vector<uint32_t> order;
  std::vector<uint8_t> listed(o->cfg.num_endpoints, 0);
  for (uint32_t i = 0; i < n; ++i) {
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

// e's LRU, least recently used first (at most cap written); returns its size
uint32_t epo_cap_lru_dump(void* h, uint32_t e, uint64_t* out, uint32_t cap) {
  const PodLRU& l = cap_of(h)->lrus[e];
  uint32_t i = 0;
  for (auto it = l.order.rbegin(); it != l.order.rend(); ++it, ++i)
    if (i < cap) out[i] = *it;
  return (uint32_t)l.order.size();
}

// the LRU part of upstream indexer.RemovePod (S.2a): e's LRU becomes empty, its capacity stays
void epo_cap_lru_clear(void* h, uint32_t e) {
  PodLRU& l = cap_of(h)->lrus[e];
  l.order.clear();
  l.pos.clear();
}

}  // extern "C"
