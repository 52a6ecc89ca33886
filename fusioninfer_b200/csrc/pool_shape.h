// pool_shape.h — the shape of a handle's prefix index as a function of its pool: words per membership row and index
// slots.  fi_epp_create and fi_epp_resize_pool (engine.cu) both derive it from here.  Pure C++ (unit-tested on the CPU
// through hostcheck.cpp).
#pragma once
#include <cstdint>

namespace fi {

// Words per membership row over `endpoint_count` local endpoints: ceil(E / 32) rounded up to a power of two (the row
// index is node << logW, and match_pick has one variant per power of two).
inline uint32_t pool_row_words(uint32_t endpoint_count) {
  const uint32_t words = (endpoint_count + 31) / 32;
  uint32_t w = 1;
  while (w < words) w <<= 1;
  return w;
}

// The index slots of a handle created with index_slots = 0: room for every LRU entry of the pool at load <= 0.5
// (1 024 entries per endpoint without an LRU), at least 4 096, at most 2^31, a power of two.  An endpoint-range shard
// is a directory of the WHOLE pool's keys, so the pool size counts, not the shard's.
inline uint64_t pool_default_slots(uint32_t num_endpoints, uint32_t lru_capacity) {
  uint64_t want = 2ull * num_endpoints * (lru_capacity ? lru_capacity : 1024);
  if (want < 4096) want = 4096;
  uint64_t p = 1;
  while (p < want) p <<= 1;
  return p > 0x80000000ull ? 0x80000000ull : p;
}

// The index slots of a pool resized to num_endpoints: the create-time index_slots if one was given (`pinned` != 0),
// else the default for the new pool, doubled until `live_keys` are at most 60% of it — the share above which
// check_counters reports a full index — since direct SETs can hold more keys than the LRUs allow.
inline uint64_t pool_resized_slots(uint64_t pinned, uint32_t num_endpoints, uint32_t lru_capacity, uint64_t live_keys) {
  if (pinned) return pinned;
  uint64_t slots = pool_default_slots(num_endpoints, lru_capacity);
  while (live_keys * 10 > slots * 6) slots <<= 1;
  return slots;
}

// A resize rebuilds the index exactly when the row width or the slot count changes; otherwise the rows stay where they
// are (a removed endpoint's bits are cleared in place, a new endpoint's bits are zero already).
inline bool pool_needs_rebuild(uint32_t W, uint64_t slots, uint32_t new_W, uint64_t new_slots) {
  return W != new_W || slots != new_slots;
}

}  // namespace fi
