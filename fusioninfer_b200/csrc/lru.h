// lru.h — host-side per-endpoint LRU of block hashes.
//
// Mirrors upstream's podToLRU (SURVEY.md Appendix A.2; capacity =
// lruCapacityPerServer, /root/reference/pkg/router/strategy.go:59,149) with
// hashicorp/golang-lru semantics: adding an existing key moves it to the front;
// adding a new key pushes it to the front and, if the set is full, evicts the
// oldest.  The LRU *order* is pointer-chasing and stays on the host; only the
// resulting membership changes (SET / CLEAR) are streamed to the GPU index.
//
// Flat arrays + an open-addressed key→node map (16-byte slots: one cache line per probe) with
// backward-shift deletion: 48 bytes per entry, cut from a huge-page arena on an endpoint's first use.  A pool of 1 024
// endpoints x 31 250 entries is 1.5 GB of host memory touched at random, i.e. every touch is a few DRAM
// misses; touch_chain() therefore runs a chain of hashes through the LRU with the map slots prefetched a few
// keys ahead and the next eviction victims' slots prefetched as soon as they are known.
#pragma once
#include <sys/mman.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>

namespace fi {

// Backing store of a pool's LRUs: ONE anonymous mapping, advised to use transparent huge pages (the tables of
// a 1 024 x 31 250-entry pool are 1.5 GB touched at random — with 4 KiB pages every touch is a TLB miss too),
// carved up by a lock-free bump pointer (an endpoint's tables are cut on its first use, from whichever worker
// thread gets there).  Physical pages appear on first touch.
class LruArena {
 public:
  LruArena() = default;
  LruArena(const LruArena&) = delete;
  LruArena& operator=(const LruArena&) = delete;
  ~LruArena() { release(); }
  bool reserve(size_t bytes) {
    release();
    bytes = (bytes + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
    void* p = mmap(nullptr, bytes + (2u << 20), PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) return false;
    raw_ = p;
    raw_bytes_ = bytes + (2u << 20);
    base_ = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + (2u << 20) - 1) & ~(uintptr_t)((2u << 20) - 1));
    size_ = bytes;
#ifdef MADV_HUGEPAGE
    madvise(base_, size_, MADV_HUGEPAGE);
#endif
    next_.store(0);
    return true;
  }
  void* take(size_t bytes) {  // 64-byte aligned; nullptr when exhausted
    bytes = (bytes + 63) & ~(size_t)63;
    const size_t off = next_.fetch_add(bytes, std::memory_order_relaxed);
    return off + bytes <= size_ ? base_ + off : nullptr;
  }
  void release() {
    if (raw_) munmap(raw_, raw_bytes_);
    raw_ = nullptr;
    base_ = nullptr;
    size_ = raw_bytes_ = 0;
  }

 private:
  void* raw_ = nullptr;
  char* base_ = nullptr;
  size_t size_ = 0, raw_bytes_ = 0;
  std::atomic<size_t> next_{0};
};

// One endpoint's LRU.  Over-aligned: head / tail / size change on every touch, and the LRUs of neighbouring
// endpoints are walked by different threads at the same time (false sharing otherwise).
class alignas(128) LruSet {
 public:
  explicit LruSet(uint32_t capacity = 0, LruArena* arena = nullptr) : cap_(capacity), limit_(capacity), arena_(arena) {}
  LruSet(const LruSet& o) : cap_(o.cap_), limit_(o.limit_), arena_(o.arena_) {}  // copies are made only of fresh, empty sets
  LruSet& operator=(const LruSet&) = delete;
  ~LruSet() {
    if (owned_) std::free(owned_);
  }
  static size_t bytes_needed(uint32_t capacity) {
    uint64_t m = 16;
    while (m < (uint64_t)capacity * 2) m <<= 1;
    return (((size_t)capacity * sizeof(Node) + 63) & ~(size_t)63) + (size_t)m * sizeof(Slot) + 128;
  }

  uint32_t size() const { return size_; }
  uint32_t capacity() const { return cap_; }
  // the run-time capacity (fi_epp_set_lru_capacities): at most `capacity`, the size the memory is cut for
  uint32_t limit() const { return limit_; }

  // Touch `key`.  Returns true if it was newly inserted; *evicted/ *did_evict
  // report the key pushed out to make room.
  bool touch(uint64_t key, uint64_t* evicted, bool* did_evict) {
    *did_evict = false;
    if (cap_ == 0) return false;
    if (!nodes_) init();
    uint32_t slot = find_slot(key);
    if (map_[slot].idx != kNone) {  // hit: move to front
      move_front(map_[slot].idx);
      return false;
    }
    uint32_t node;
    if (size_ >= limit_) {  // evict the tail, reuse its node
      node = tail_;
      *evicted = nodes_[node].key;
      *did_evict = true;
      unlink(node);
      map_erase(nodes_[node].key);
      --size_;
      slot = find_slot(key);  // the erase may have shifted entries
      // the next victims are known now: bring their map slots in before the next insertion needs them
      if (tail_ != kNone) {
        prefetch_slot(nodes_[tail_].key);
        const uint32_t t2 = nodes_[tail_].prev;
        if (t2 != kNone) prefetch_slot(nodes_[t2].key);
      }
    } else if (free_ != kNone) {  // a node a shrink gave back
      node = free_;
      free_ = nodes_[node].next;
    } else {
      node = fresh_++;  // nodes are handed out densely until full
    }
    nodes_[node].key = key;
    link_front(node);
    map_[slot].key = key;
    map_[slot].idx = node;
    ++size_;
    return true;
  }

  // indexer.Add(chain): touch keys[0..n) in order; emit(key, inserted, did_evict, evicted) after each touch
  // that changed the set.  Same result as n touch() calls.
  template <class Emit>
  void touch_chain(const uint64_t* keys, uint32_t n, Emit&& emit) {
    if (cap_ == 0 || n == 0) return;
    if (!nodes_) init();
    constexpr uint32_t kAhead = 12;
    for (uint32_t i = 0; i < n && i < kAhead; ++i) prefetch_slot(keys[i]);
    for (uint32_t i = 0; i < n; ++i) {
      if (i + kAhead < n) prefetch_slot(keys[i + kAhead]);
      uint64_t ev = 0;
      bool did = false;
      const bool inserted = touch(keys[i], &ev, &did);
      if (inserted || did) emit(keys[i], inserted, did, ev);
    }
  }

  bool contains(uint64_t key) const {
    if (!nodes_) return false;
    return map_[find_slot(key)].idx != kNone;
  }

  // Forget every entry.  The node and map memory stay with the set: the arena is a bump allocator and never
  // takes memory back.
  void clear() {
    if (!nodes_) return;
    for (uint64_t i = 0; i <= mask_; ++i) map_[i] = Slot{0, kNone, 0};
    size_ = 0;
    head_ = tail_ = kNone;
    free_ = kNone;
    fresh_ = 0;
  }

  // Set the run-time capacity to `limit` (<= capacity()) and evict the least recently used keys until the set holds
  // at most `limit`: emit(key) for each, oldest first, as touch reports an eviction.  Raising the limit evicts nothing.
  template <class Emit>
  void shrink(uint32_t limit, Emit&& emit) {
    limit_ = limit < cap_ ? limit : cap_;
    while (size_ > limit_) {
      const uint32_t node = tail_;
      const uint64_t key = nodes_[node].key;
      unlink(node);
      map_erase(key);
      nodes_[node].next = free_;
      free_ = node;
      --size_;
      emit(key);
    }
  }

  // the keys, least recently used first (diagnostics)
  template <class Visit>
  void for_each_oldest_first(Visit&& visit) const {
    for (uint32_t n = tail_; n != kNone; n = nodes_[n].prev) visit(nodes_[n].key);
  }

 private:
  static constexpr uint32_t kNone = 0xFFFFFFFFu;
  struct Node {
    uint64_t key;
    uint32_t prev, next;
  };
  struct Slot {
    uint64_t key;
    uint32_t idx;  // kNone: empty
    uint32_t pad;
  };

  void init() {
    uint64_t m = 16;
    while (m < (uint64_t)cap_ * 2) m <<= 1;
    mask_ = (uint32_t)(m - 1);
    const size_t node_bytes = ((size_t)cap_ * sizeof(Node) + 63) & ~(size_t)63;
    const size_t total = node_bytes + (size_t)m * sizeof(Slot);
    char* mem = arena_ ? static_cast<char*>(arena_->take(total)) : nullptr;
    if (!mem) {  // no arena (tests, tiny pools) or arena exhausted
      if (posix_memalign(&owned_, 64, total) != 0) throw std::bad_alloc();
      mem = static_cast<char*>(owned_);
    }
    nodes_ = reinterpret_cast<Node*>(mem);
    map_ = reinterpret_cast<Slot*>(mem + node_bytes);
    for (uint64_t i = 0; i < m; ++i) map_[i] = Slot{0, kNone, 0};
    head_ = tail_ = kNone;
  }
  static inline uint64_t mix(uint64_t h) {
    h ^= h >> 31;
    h *= 0x9E3779B97F4A7C15ULL;
    return h ^ (h >> 29);
  }
  void prefetch_slot(uint64_t key) const { __builtin_prefetch(&map_[(uint32_t)mix(key) & mask_], 1, 1); }
  uint32_t find_slot(uint64_t key) const {
    uint32_t i = (uint32_t)mix(key) & mask_;
    while (map_[i].idx != kNone && map_[i].key != key) i = (i + 1) & mask_;
    return i;
  }
  void map_erase(uint64_t key) {
    uint32_t i = find_slot(key);
    if (map_[i].idx == kNone) return;
    // backward-shift deletion keeps probe sequences intact without tombstones
    uint32_t j = i;
    for (;;) {
      j = (j + 1) & mask_;
      if (map_[j].idx == kNone) break;
      uint32_t home = (uint32_t)mix(map_[j].key) & mask_;
      // can entry j move into hole i?  yes iff home is not in (i, j] cyclically
      bool in_range = (i <= j) ? (home > i && home <= j) : (home > i || home <= j);
      if (!in_range) {
        map_[i] = map_[j];
        i = j;
      }
    }
    map_[i].idx = kNone;
  }
  void unlink(uint32_t n) {
    Node& x = nodes_[n];
    if (x.prev != kNone) nodes_[x.prev].next = x.next; else head_ = x.next;
    if (x.next != kNone) nodes_[x.next].prev = x.prev; else tail_ = x.prev;
  }
  void link_front(uint32_t n) {
    nodes_[n].prev = kNone;
    nodes_[n].next = head_;
    if (head_ != kNone) nodes_[head_].prev = n;
    head_ = n;
    if (tail_ == kNone) tail_ = n;
  }
  void move_front(uint32_t n) {
    if (head_ == n) return;
    unlink(n);
    link_front(n);
  }

  uint32_t cap_;
  uint32_t limit_;
  uint32_t size_ = 0;
  uint32_t head_ = kNone, tail_ = kNone;
  uint32_t free_ = kNone;  // nodes given back by shrink, linked through `next`
  uint32_t fresh_ = 0;     // nodes [fresh_, cap_) have never been handed out
  uint32_t mask_ = 0;
  Node* nodes_ = nullptr;
  Slot* map_ = nullptr;
  LruArena* arena_ = nullptr;
  void* owned_ = nullptr;
};

}  // namespace fi
