// resize_oracle.cpp — the CPU oracle's extension (tests/ext_oracle.cpp) with a pool resize, test infrastructure only.
//
// It compiles the extension (and through it oracle/epp_oracle.cpp) into the same translation unit and adds the
// per-endpoint part of fi_epp_resize_pool (docs/SPEC.md S.2c).  Every epo_* and epx_* function works on its handles.
#include "ext_oracle.cpp"

extern "C" {

// fi_epp_resize_pool (S.2c) on the oracle's per-endpoint state: endpoints [E', E) are truncated away, [E, E') are
// appended fresh (not alive, no adapters, an empty LRU of capacity lru_capacity), and E becomes E'.  A shrink's index
// pairs are the caller's to remove first (ResizeOracle.resize: remove_endpoints of the tail).
int epx_resize(void* h, uint32_t num_endpoints) {
  ExtOracle* o = ext_of(h);
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
  return FI_OK;
}

}  // extern "C"
