// snapshot_oracle.cpp — the CPU oracle's extension (tests/resize_oracle.cpp) with the state of an index snapshot
// (docs/SPEC.md S.2d), test infrastructure only.
//
// It compiles the resize extension (and through it tests/ext_oracle.cpp and oracle/epp_oracle.cpp) into the same
// translation unit and adds the three parts of S.2d's state, read and written whole: the pair set (epx_index_pairs),
// every endpoint's LRU capacity (epx_lru_capacities) and, with the LRU lists of epx_lru_dump, epx_load_state, which
// replaces all three.  Every epo_* and epx_* function works on its handles.
#include "resize_oracle.cpp"

namespace {

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

}  // namespace

extern "C" {

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
// Endpoint states and adapters are left as they are.
int epx_load_state(void* h, uint64_t n, const uint64_t* hashes, const uint32_t* endpoints, const uint32_t* lens,
                   const uint64_t* keys, const uint32_t* caps) {
  ExtOracle* o = ext_of(h);
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
