// lru_batch.h — host side of fi_epp_index_add_chains: upstream's PreRequest step, indexer.Add(chain, picked pod),
// for a whole batch of routing decisions (SURVEY.md Appendix A.2; capacity = lruCapacityPerServer,
// /root/reference/pkg/router/strategy.go:59,149).
//
// The endpoints' LRUs are independent, so they are walked in parallel: requests are bucketed by endpoint
// (request order kept), one endpoint is one task of a persistent worker pool, and every worker appends the
// resulting membership changes to its own op lists.  The GPU applies a group of ops as "all SETs, then all
// CLEARs"; that equals the sequential order except when a hash is re-added after its own eviction inside the same
// batch — then the endpoint's later ops go to the next SEGMENT (segments are applied one after the other), which
// keeps "last op wins" exact.  Every set evicts against its own limit() (fi_epp_set_lru_capacities).  Host-only
// code (no CUDA): tests/test_host_logic.py and tests/test_lru_capacity_cpu.py run it against a sequential LRU, and
// tests/test_add_staging_cpu.py checks the staging plan (plan_staging).
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/fi_epp.h"
#include "lru.h"

namespace fi {

// Persistent worker threads for the host LRU (fi_epp_index_add_chains): run(n, fn) calls fn(task, worker)
// for task = 0..n-1, tasks handed out dynamically; the caller is worker 0.
class WorkerPool {
 public:
  explicit WorkerPool(unsigned workers) : n_(workers < 1 ? 1 : workers) {
    for (unsigned w = 1; w < n_; ++w) th_.emplace_back([this, w] { loop(w); });
  }
  ~WorkerPool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
      ++gen_;
    }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  unsigned size() const { return n_; }
  void run(uint32_t ntasks, const std::function<void(uint32_t, unsigned)>& fn) {
    if (ntasks == 0) return;
    {
      std::lock_guard<std::mutex> lk(mu_);
      fn_ = &fn;
      ntasks_ = ntasks;
      next_.store(0, std::memory_order_relaxed);
      busy_ = n_ - 1;
      ++gen_;
    }
    cv_.notify_all();
    work(0);
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [this] { return busy_ == 0; });
    fn_ = nullptr;
  }

 private:
  void work(unsigned w) {
    for (;;) {
      const uint32_t t = next_.fetch_add(1, std::memory_order_relaxed);
      if (t >= ntasks_) break;
      (*fn_)(t, w);
    }
  }
  void loop(unsigned w) {
    uint64_t seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
      }
      work(w);
      std::lock_guard<std::mutex> lk(mu_);
      if (--busy_ == 0) done_.notify_one();
    }
  }
  unsigned n_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  const std::function<void(uint32_t, unsigned)>* fn_ = nullptr;
  uint32_t ntasks_ = 0;
  std::atomic<uint32_t> next_{0};
  unsigned busy_ = 0;
  uint64_t gen_ = 0;
  bool stop_ = false;
};


// open-addressed set of 64-bit keys, emptied in O(1) (generation stamps): the hashes one endpoint evicted
// during the current fi_epp_index_add_chains call
struct StampSet {
  std::vector<uint64_t> key;
  std::vector<uint32_t> gen;
  uint32_t cur = 0, mask = 0, used = 0;
  void reset() {
    if (key.empty()) {
      key.assign(1u << 12, 0);
      gen.assign(1u << 12, 0);
      mask = (1u << 12) - 1;
    }
    ++cur;
    used = 0;
    if (cur == 0) {  // stamp wrapped
      std::fill(gen.begin(), gen.end(), 0u);
      cur = 1;
    }
  }
  static uint32_t mix(uint64_t h) {
    h ^= h >> 29;
    h *= 0x9E3779B97F4A7C15ULL;
    return (uint32_t)(h >> 32);
  }
  bool contains(uint64_t k) const {
    for (uint32_t i = mix(k) & mask;; i = (i + 1) & mask) {
      if (gen[i] != cur) return false;
      if (key[i] == k) return true;
    }
  }
  void insert(uint64_t k) {
    if ((used + 1) * 2 > mask + 1) grow();
    for (uint32_t i = mix(k) & mask;; i = (i + 1) & mask) {
      if (gen[i] != cur) {
        gen[i] = cur;
        key[i] = k;
        ++used;
        return;
      }
      if (key[i] == k) return;
    }
  }
  void grow() {
    std::vector<uint64_t> ok;
    ok.reserve(used);
    for (uint32_t i = 0; i <= mask; ++i)
      if (gen[i] == cur) ok.push_back(key[i]);
    const uint32_t n = (mask + 1) * 2;
    key.assign(n, 0);
    gen.assign(n, 0);
    mask = n - 1;
    cur = 1;
    used = 0;
    for (uint64_t k : ok) insert(k);
  }
};

// ops one worker produced, by segment: within a segment SETs run before CLEARs; a SET that follows a CLEAR of
// the same (hash, endpoint) pair opens the endpoint's next segment.  The vectors keep their capacity from call
// to call (a batch is ~5 M ops = 77 MB: growing fresh vectors every call costs more than the LRU walk).
struct WorkerOps {
  std::vector<std::vector<fi_index_op>> sets, clears;
  size_t nseg = 0;  // segments used by the current batch
  StampSet evicted;
  void begin_batch() {
    for (size_t s = 0; s < nseg; ++s) {
      sets[s].clear();
      clears[s].clear();
    }
    nseg = 0;
  }
  void need(size_t seg) {
    if (sets.size() <= seg) {
      sets.resize(seg + 1);
      clears.resize(seg + 1);
    }
    if (nseg <= seg) nseg = seg + 1;
  }
  std::vector<fi_index_op>& sets_of(size_t seg) {
    need(seg);
    return sets[seg];
  }
  std::vector<fi_index_op>& clears_of(size_t seg) {
    need(seg);
    return clears[seg];
  }
};

// Walk the LRUs for one batch.  endpoints[r]: global endpoint (FI_NO_ENDPOINT or outside [lo, lo+EL): skipped);
// chains: R rows of `pitch` hashes, nblocks[r] valid.  outs[w] receives worker w's ops (cleared first, capacity
// kept from earlier calls).  Returns the number of segments.
inline size_t lru_walk_batch(std::vector<LruSet>& lrus, uint32_t lo, uint32_t EL, const uint32_t* endpoints,
                             const uint64_t* chains, uint32_t pitch, const uint32_t* nblocks, uint32_t R, WorkerPool& pool,
                             std::vector<WorkerOps>& outs) {
  // requests of every local endpoint, in request order (counting sort)
  std::vector<uint32_t> first(EL + 1, 0), order, active;
  for (uint32_t r = 0; r < R; ++r) {
    const uint32_t e = endpoints[r] - lo;
    if (endpoints[r] != FI_NO_ENDPOINT && e < EL && nblocks[r]) first[e + 1]++;
  }
  for (uint32_t e = 0; e < EL; ++e) {
    if (first[e + 1]) active.push_back(e);
    first[e + 1] += first[e];
  }
  order.resize(first[EL]);
  {
    std::vector<uint32_t> fill(first.begin(), first.end() - 1);
    for (uint32_t r = 0; r < R; ++r) {
      const uint32_t e = endpoints[r] - lo;
      if (endpoints[r] != FI_NO_ENDPOINT && e < EL && nblocks[r]) order[fill[e]++] = r;
    }
  }
  // endpoints with the most requests first: the dynamic hand-out then ends with the short ones
  std::stable_sort(active.begin(), active.end(),
                   [&](uint32_t a, uint32_t b) { return first[a + 1] - first[a] > first[b + 1] - first[b]; });
  if (outs.size() != pool.size()) outs.resize(pool.size());
  for (auto& o : outs) o.begin_batch();
  pool.run((uint32_t)active.size(), [&](uint32_t task, unsigned w) {
    const uint32_t e = active[task];
    LruSet& l = lrus[e];
    WorkerOps& o = outs[w];
    o.evicted.reset();
    size_t seg = 0;
    bool any_evicted = false;
    const uint32_t eg = e + lo;
    for (uint32_t k = first[e]; k < first[e + 1]; ++k) {
      const uint32_t r = order[k];
      l.touch_chain(chains + (size_t)r * pitch, nblocks[r], [&](uint64_t key, bool inserted, bool did, uint64_t ev) {
        if (did) {
          o.clears_of(seg).push_back(fi_index_op{ev, eg, FI_OP_CLEAR});
          o.evicted.insert(ev);
          any_evicted = true;
        }
        if (inserted) {
          if (any_evicted && o.evicted.contains(key)) {  // re-added after its eviction in this call
            ++seg;
            o.evicted.reset();
            any_evicted = false;
          }
          o.sets_of(seg).push_back(fi_index_op{key, eg, FI_OP_SET});
        }
      });
    }
  });
  size_t nseg = 0;
  for (auto& o : outs) nseg = std::max(nseg, o.nseg);
  return nseg;
}

// One copy of a staging plan: ops [src, src + n) of outs[worker].sets[seg] (or .clears[seg]) go to offset dst of the
// group's SET (or CLEAR) buffer.
struct StagePiece {
  uint32_t worker, seg;
  bool clear;
  size_t src, n;
  uint64_t dst;
};
struct StageGroup {
  std::vector<StagePiece> pieces;
  uint64_t n_sets = 0, n_clears = 0;  // the group's fill once its pieces are copied
};

// Where the ops of one walk are staged (fi_epp_index_add_chains).  The open group already holds ns0 SETs and nc0
// CLEARs; the walk's ops follow segment by segment, a segment's SETs before its CLEARs, worker by worker.  A group is
// closed (flushed) when a buffer of `chunk` ops is full, and at a segment boundary when anything is staged.  The ops
// staged before the call count as a segment of their own: when they include CLEARs the plan begins with a flush, so
// that no SET of this call shares a group with them.  Every group but the last (the tail) ends with a flush.  Counts
// and offsets only: the ops themselves are not read.
inline std::vector<StageGroup> plan_staging(const std::vector<WorkerOps>& outs, size_t nseg, uint64_t ns0, uint64_t nc0,
                                            uint64_t chunk) {
  std::vector<StageGroup> groups(1);
  groups[0].n_sets = ns0;
  groups[0].n_clears = nc0;
  if (nc0) groups.emplace_back();
  for (size_t seg = 0; seg < nseg; ++seg) {
    for (int kind = 0; kind < 2; ++kind)
      for (uint32_t w = 0; w < outs.size(); ++w) {
        if (outs[w].nseg <= seg) continue;
        const size_t n = (kind ? outs[w].clears[seg] : outs[w].sets[seg]).size();
        for (size_t done = 0; done < n;) {
          StageGroup& g = groups.back();
          uint64_t& fill = kind ? g.n_clears : g.n_sets;
          const size_t take = std::min<uint64_t>(chunk - fill, n - done);
          g.pieces.push_back(StagePiece{w, (uint32_t)seg, kind == 1, done, take, fill});
          fill += take;
          done += take;
          if (fill == chunk) groups.emplace_back();
        }
      }
    // the next segment's SETs must run after these CLEARs
    if (seg + 1 < nseg && (groups.back().n_sets || groups.back().n_clears)) groups.emplace_back();
  }
  return groups;
}

}  // namespace fi
