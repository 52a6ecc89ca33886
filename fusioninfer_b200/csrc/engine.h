// engine.h — private to the host sources of libfi_epp (engine*.cu): the handle, the types it owns, and the helpers
// and functions the sources share.  Each source holds one concern:
//   engine.cu           the handle's lifetime, options, endpoint tables, statistics and pool resize;
//   engine_index.cu     the ordering rule of index updates, op staging and the index entry points;
//   engine_lru.cu       the host and device LRUs and every indexer.Add;
//   engine_pick.cu      the pick paths and the pipelined submit;
//   engine_snapshot.cu  index snapshots and captures;
//   engine_comm.cu      the NCCL / peer-memory communicator of endpoint-range sharded pools.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include <sched.h>

#include "../../include/fi_epp.h"
#include "cuda_owned.h"
#include "kernels.cuh"
#include "lru.h"
#include "lru_batch.h"
#include "lru_device.cuh"
#include "lru_plan.h"
#include "pool_shape.h"

namespace fi::engine {

typedef struct ncclComm* ncclComm_t;

struct PairKey {
  uint64_t hash;
  uint32_t endpoint;
  bool operator==(const PairKey& o) const { return hash == o.hash && endpoint == o.endpoint; }
};
struct PairHash {
  size_t operator()(const PairKey& k) const {
    uint64_t x = k.hash ^ ((uint64_t)k.endpoint * 0x9E3779B97F4A7C15ULL);
    x ^= x >> 29;
    return (size_t)(x * 0xBF58476D1CE4E5B9ULL);
  }
};

constexpr uint64_t kOpChunk = 1ull << 20;  // ops per pinned staging buffer
constexpr uint64_t kListChunk = 1ull << 20;  // entries per copy of the host match-lists call (8 MiB)

enum KernelKind { K_HASH = 0, K_MATCH = 1, K_INDEX = 2, K_OTHER = 3, K_KINDS = 4 };

// host cores this process may really use: the affinity mask capped by the cgroup CPU quota (more runnable
// threads than quota only get the group throttled)
inline unsigned usable_cores() {
  unsigned n = std::thread::hardware_concurrency();
  cpu_set_t set;
  CPU_ZERO(&set);
  if (sched_getaffinity(0, sizeof(set), &set) == 0 && CPU_COUNT(&set) > 0) n = (unsigned)CPU_COUNT(&set);
  if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {  // cgroup v2: "<quota|max> <period>"
    char q[64] = {0};
    long long period = 0;
    if (std::fscanf(f, "%63s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0 && period > 0) {
      const long long quota = std::atoll(q);
      if (quota > 0) n = std::min<unsigned>(n, (unsigned)std::max<long long>(1, (quota + period - 1) / period));
    }
    std::fclose(f);
  }
  return n ? n : 1u;
}

// A device staging buffer and its pinned host mirror (h stays null for a device-only buffer), grown by grow_staging
template <typename T>
struct Staging {
  DevPtr<T> d;
  PinnedPtr<T> h;
  size_t cap = 0;  // elements
};

// The six arrays behind one IndexView, and the view (filled by alloc_index)
struct IndexTables {
  IndexView v{};
  DevPtr<uint64_t> keys, klog;
  DevPtr<uint32_t> node_of, rows, cnt, rmask;
};

// The device tables sized by the pool (filled by alloc_endpoint_tables; the ScoreTables of a handle point into them)
struct EndpointTables {
  DevPtr<EndpointDev> eps;      // [num_endpoints]
  DevPtr<double> sc;            // [FI_EPP_MAX_PROFILES][FI_EPP_MAX_SCORERS][Epad]
  DevPtr<uint32_t> elig, ztie;  // [FI_EPP_MAX_PROFILES][W]
  DevPtr<LoraDev> lora;         // [Epad] local endpoints' adapter residency
};

// The device-resident LRU of a handle (lru_kernels.cu), allocated whole by ensure_dev_lru at the first Add
struct DevLruStore {
  DevLru v{};  // points into slots, log, state and ctr
  DevPtr<LruSlot> slots;
  DevPtr<uint64_t> log;
  DevPtr<uint32_t> state;             // head | tail | count | used | hold | dcount | ovf | any_ovf | error | cap
  DevPtr<unsigned long long> ctr;     // [0] SETs emitted, [1] endpoints maintained, [2] CLEARs of the running sub-batch,
                                      // [3] CLEARs total, [4] doomed winners
  struct HostStat {
    uint32_t error, any_ovf;  // (any_ovf: the touch kernel's overflow flag of the running sub-batch)
    unsigned long long n_sets, n_maintained, n_clears_cur, n_clears, n_doomed;
    uint32_t planned_ovf;     // the touch kernel's overflow flag after a fi_epp_index_add_submitted call (must stay 0)
  };
  PinnedPtr<HostStat> stat;           // pinned copy, refreshed after every call
  // per-sub-batch scratch, for touch_cap touches
  DevPtr<uint32_t> slot_of, wcount, base;
  DevPtr<fi_index_op> sets, clears;
  uint64_t touch_cap = 0;
  Event ev;                           // the previous call's staging has been consumed
  Event ev_ovf;                       // the touch kernel's overflow flag has reached the host
};

// Sharded mode (fi_epp_comm_init): the communicator and the buffers of the cross-rank merge and directory gossip
struct ShardState {
  ncclComm_t comm = nullptr;
  DevPtr<fi_pick> d_local;   // [R][P] this rank's picks
  DevPtr<fi_pick> d_gather;  // [world][R][P]
  // directory gossip (index_kernels.cu): this rank's transition log of the current round and the buffers the ranks'
  // logs are gathered into
  DevPtr<unsigned long long> d_glog_n;  // [2] appear / vanish counts
  DevPtr<uint64_t> d_glog_a;            // [kOpChunk]
  DevPtr<uint64_t> d_glog_v;            // [kOpChunk]
  DevPtr<unsigned long long> d_ghdr;    // [world + 1][2] gathered counts
  PinnedPtr<unsigned long long> h_ghdr; // pinned copy
  DevPtr<uint64_t> d_ggather;           // [world][kOpChunk]
  // peer-memory exchange (kernels.cuh PeerXchg)
  DevPtr<uint8_t> d_xchg;               // this rank's exchange buffer
  PinnedPtr<volatile uint32_t> h_xerr;  // poll-timeout flag of the exchange (mapped pinned host word the kernels set)
  void* peer_ipc[FI_MAX_RANKS] = {};    // mappings opened with cudaIpcOpenMemHandle
  ~ShardState();  // engine_comm.cu
};

}  // namespace fi::engine

// (a private header: every engine source works in these names)
using namespace fi;
using namespace fi::engine;

struct fi_epp {
  // declared first so that they are destroyed last, after every buffer and event the work on them used
  Stream s_main, s_index;  // compute; index maintenance (side stream)
  // host-buffer picks feed the prompts in slices: the copy engine runs ahead on s_copy while s_main hashes,
  // walks and matches the slices that have landed (the step is PCIe-bound: only the last slice's work is exposed)
  Stream s_copy;
  // Pipelined device path (fi_epp_pick_submit / fi_epp_pick_wait): stage A (block hashing + chain walk) of
  // batch k+1 runs on s_a while stage B (match + pick) of batch k runs on s_main; the chain / block-count
  // buffers are double-buffered (slot = batch parity).
  Stream s_a;

  fi_epp_config cfg;
  std::mutex mu;
  std::string err;
  int sm_count = 132;
  uint32_t MP = 0;  // chain pitch
  uint32_t W = 0;   // words per index row
  uint32_t P = 0;   // profiles
  bool fast_hash = false;

  static constexpr int kMaxFeedSlices = 16;
  Event ev_copy[kMaxFeedSlices];
  uint32_t feed_slices = 8;  // FI_EPP_FEED_SLICES (1: one copy, then the whole batch)
  // slot 1's chain and block-count buffers, allocated together by the first pipelined submit that needs them
  DevPtr<uint64_t> d_chain2;
  DevPtr<uint32_t> d_nblocks2;
  Event ev_in, ev_a[2], ev_b[2];
  Event ev_pick;   // completion of the most recent pick of any kind (recorded on s_main)
  Event ev_plain;  // completion of the most recent stream-ordered (not pipelined) pick
  uint64_t pipe_seq = 0;          // batches submitted
  // Tickets (fi_epp_pick_submit_ex / fi_epp_pick_wait_batch / fi_epp_index_add_submitted): every submit, pipelined or
  // not, takes the next number; ev_ticket[t % kTicketRing] is recorded on s_main when batch t is complete.
  static constexpr int kTicketRing = 8;
  Event ev_ticket[kTicketRing];
  uint64_t tickets = 0;
  uint64_t slot_ticket[2] = {~0ull, ~0ull};  // ticket whose chains slot s still holds (~0: none)
  uint32_t slot_R[2] = {0, 0};
  Event ev_slot_read[2];          // the last copy of slot s's chains for fi_epp_index_add_submitted
  Event ev_index, ev_user, ev_done, ev_ctr;

  // request buffers (device)
  DevPtr<uint8_t> d_prompts;
  DevPtr<uint64_t> d_offsets;
  DevPtr<uint64_t> d_h0;
  DevPtr<uint64_t> d_chain;
  DevPtr<uint32_t> d_nblocks;
  DevPtr<fi_pick> d_picks;      // [R][P] final
  Staging<fi_pick> ranked;      // [R][P][k] of the host ranked pick: allocated by the first such call, grown with k
  Staging<uint32_t> subsets;    // [max_batch][ceil(E/32)] staging of fi_epp_pick_batch_subset: allocated by its first call
  Staging<uint16_t> counts;     // [max_batch][endpoint_count] of fi_epp_match_counts: allocated by its first call
  // fi_epp_match_lists (docs/SPEC.md S.3b): every request's slot of (column << 12) | count entries and the entry
  // counts the match kernel writes, allocated together by the first lists call for max_batch requests of the pool as
  // it is (alloc_list_scratch), and freed by a resize
  struct ListScratch {
    DevPtr<uint32_t> slots;  // [max_batch][endpoint_count]
    DevPtr<uint32_t> nnz;    // [max_batch]
    size_t cap = 0;          // entries of slots
  } lists;
  Staging<uint64_t> list_offsets;       // [max_batch + 1] of the host lists call: allocated by its first call
  Staging<fi_match_entry> list_chunk;   // the host lists call's entries, copied out kListChunk at most at a time
  std::unique_ptr<ShardState> shard;  // sharded mode only
  PeerXchg px{};                 // px.enabled == 0: NCCL all-gathers are used
  // sharded mode: every rank hashes every prompt (the default: hashing 16 KiB from local HBM is expected to cost
  // less than receiving 2 KiB of chain over NVLink; not measured on H100s, bench.py --gpus N times both); FI_EPP_SHARD_HASH=
  // split / option "shard_hash" = 1: every rank hashes R/world requests and the chains are all-gathered
  bool split_hash = false;
  uint32_t chain_rows = 0;  // rows allocated in d_chain / d_nblocks (max_batch padded for the gather)
  DevPtr<unsigned long long> d_probed;
  DevPtr<uint32_t> d_work;  // [16] dynamic work-queue counters of in-flight match launches
  // pinned host mirrors
  PinnedPtr<fi_pick> h_picks;
  PinnedPtr<uint64_t> h_offsets;
  PinnedPtr<uint64_t> h_h0;
  PinnedPtr<uint32_t> h_nblocks;

  // index
  IndexTables ix;
  uint64_t index_slots_given = 0;  // index_slots as passed to fi_epp_create (0: the default for the pool, pool_shape.h)
  std::unique_ptr<IndexTables> ix_spare;  // rebuild target, allocated at the first rebuild and reused alternately
  DevPtr<IndexCounters> d_ctr;
  PinnedPtr<IndexCounters> h_ctr;
  bool ctr_pending = false;
  // the last counters read (`used`) and how many new keys the updates queued since then can add at most (one per
  // SET or LRU touch): check_counters_lagged decides from these when the pending counters are not in yet
  uint64_t ctr_used_known = 0, ctr_unchecked = 0;
  uint64_t rebuilds = 0, ops_applied = 0;
  PinnedPtr<fi_index_op> h_sets[2], h_clears[2];
  DevPtr<fi_index_op> d_sets[2], d_clears[2];
  Event ev_buf[2];
  // the open op group (submit_op states the rule that keeps it exact)
  int cur_buf = 0;
  uint64_t n_sets = 0, n_clears = 0;
  std::unordered_set<PairKey, PairHash> cleared;
  bool clears_untracked = false;
  // fi_epp_index_remove_endpoints: [0] pairs removed, then (u32) the local endpoints whose device LRU is reset.
  // Allocated at the first call.
  DevPtr<unsigned long long> d_rm;
  LruArena lru_arena;  // backing store of the LRUs (one huge-page mapping)
  std::vector<LruSet> lrus;
  // [endpoint_count] every local endpoint's LRU capacity (fi_epp_set_lru_capacities; lru_capacity until set): the
  // host copy of DevLru::cap and of the host LRU's limits, kept whichever LRU serves the handle
  std::vector<uint32_t> lru_caps;
  Staging<uint32_t> lru_resize;  // a device resize's rounds: local endpoints | eviction quotas
  std::unique_ptr<WorkerPool> pool;  // host LRU workers (fi_epp_index_add_chains), created on first use
  std::vector<WorkerOps> lru_outs;   // their op lists (capacity kept from batch to batch)
  bool verbose = false;              // FI_EPP_VERBOSE
  // device-resident LRU (lru_kernels.cu): the default for single-rank handles whose lru_capacity holds a whole
  // chain; option "device_lru" / FI_EPP_DEVICE_LRU=0 selects the host LRU instead.  Allocated at the first Add;
  // the two are never mixed on one handle.
  int lru_mode = -1;  // -1: not chosen yet, 0: host LRU, 1: device LRU
  int lru_want = -1;  // option / environment override (-1: automatic)
  uint32_t lru_table_slots = 0;  // option "lru_table_slots": slots per endpoint table of the device LRU (0: sized by free HBM)
  std::unique_ptr<DevLruStore> dlru;  // null until the first device-LRU Add
  // fi_epp_index_add_submitted: double-buffered plan and chain staging (Add j uses padd[j & 1]; ev_done: consumed).
  // d_chains and ev_done are allocated together by the buffer's first Add.
  struct PipeAdd {
    Staging<uint32_t> plan;      // the packed plan (lru_plan.h)
    DevPtr<uint64_t> d_chains;   // [max_batch][MP]
    Event ev_done;
  };
  PipeAdd padd[2];
  uint64_t padd_seq = 0;
  uint64_t lru_deferred = 0, lru_sub_batches = 0;  // host-side totals
  Staging<uint32_t> lru_plan_buf;            // the packed plan of the current call (lru_plan.h)
  Staging<uint64_t> lru_chains;              // staging of host chains (device only)
  uint32_t last_plain_R = 0;                 // rows of d_chain the most recent stream-ordered pick wrote
  LruPlan lru_plan;
  unsigned lru_threads = 0;          // 0: FI_EPP_LRU_THREADS, else min(usable cores, 64)

  // endpoints / score tables
  std::vector<EndpointDev> eps;  // global pool
  bool eps_dirty = true;
  EndpointTables ept;
  DevPtr<ZeroBest> d_zero;
  std::vector<LoraDev> lora;   // local endpoints' adapter residency (lora-affinity-scorer)
  bool lora_dirty = false;
  DevPtr<uint64_t> d_adapters;    // staging of the host path's per-request adapter ids
  PinnedPtr<uint64_t> h_adapters;
  ScoreTables st{};

  // multi-GPU (fi_epp_comm_init)
  uint32_t rank = 0, world = 1;

  // stats / profiling
  fi_epp_stats stats{};
  bool profiling = false;
  bool tracing = false;       // FI_EPP_TRACE=<call index>: print that call's kernel timeline to stderr
  long trace_call = -1;
  Event ev_trace0;
  struct Ev {
    Event a, b;
    int kind;
  };
  std::vector<Ev> pending_ev;
  std::vector<Event> ev_pool;
};

namespace fi::engine {

#define FI_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e__ = (call);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e__);                     \
      return FI_ERR_CUDA;                                                               \
    }                                                                                   \
  } while (0)

inline int fail(fi_epp* h, int code, const std::string& m) {
  h->err = m;
  return code;
}

// The status of a failed allocation (or of a chain of them): FI_ERR_NOMEM when memory ran out, else FI_ERR_CUDA.
// The error is cleared, so that later calls do not report it.
inline int alloc_status(cudaError_t e) {
  cudaGetLastError();
  return e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA;
}

// Make `s` hold at least n elements: a smaller one is replaced by `alloc` (>= n) elements, its pinned mirror too if
// `pinned`.  On failure nothing of it stays allocated (cap 0) and the call fails with FI_ERR_NOMEM.
template <typename T>
int grow_staging(fi_epp* h, Staging<T>& s, size_t n, size_t alloc, bool pinned) {
  if (n <= s.cap) return FI_OK;
  s = Staging<T>{};
  Staging<T> t;
  if (cuda_alloc(t.d, alloc) != cudaSuccess || (pinned && cuda_alloc(t.h, alloc) != cudaSuccess)) {
    cudaGetLastError();
    return fail(h, FI_ERR_NOMEM, "cannot allocate a staging buffer of " + std::to_string(alloc * sizeof(T)) + " bytes");
  }
  t.cap = alloc;
  s = std::move(t);
  return FI_OK;
}

inline Event get_event(fi_epp* h) {
  Event e;
  if (!h->ev_pool.empty()) {
    e = std::move(h->ev_pool.back());
    h->ev_pool.pop_back();
  } else {
    cuda_create(e, cudaEventDefault);
  }
  return e;
}

// wraps one kernel launch: counts it and, when profiling, brackets it with events
struct LaunchScope {
  fi_epp* h;
  cudaStream_t s;
  int kind;
  Event a, b;
  LaunchScope(fi_epp* h_, cudaStream_t s_, int kind_) : h(h_), s(s_), kind(kind_) {
    h->stats.kernel_launches++;
    if (h->profiling || h->tracing) {
      a = get_event(h);
      b = get_event(h);
      cudaEventRecord(a.get(), s);
    }
  }
  ~LaunchScope() {
    if (h->profiling || h->tracing) {
      cudaEventRecord(b.get(), s);
      h->pending_ev.push_back({std::move(a), std::move(b), kind});
    }
  }
};

// ---- the ordering rule of index updates -------------------------------------------------------------------------
// Every change to the GPU index or to the device LRU runs on s_index as one update, between update_begin and
// update_end:
//  1. the ops staged earlier (fi_epp_index_apply, the host LRU) are flushed first;
//  2. the counters of the previous update are checked, which may rebuild the index or report it full;
//  3. s_index waits for ev_pick: a pick sees the index as it was when it was called, so an update queued after a pick
//     must not overtake it on the GPU;
//  -- the update's work --
//  4. the index counters are copied back for the next rebuild decision, and the device LRU's status too when the work
//     ran LRU kernels that count or flag errors;
//  5. ev_index is recorded, so that every later pick waits for this update.
// A missing step is a silent race between the streams.  A pick takes steps 1 and 2 (settle_updates) before it reads
// the index.  Settle says which of steps 1 and 2 update_begin takes: both (kLagged: with check_counters_lagged(h,
// extra)), step 2 only (flush_ops, which is the flush) or neither (the callers say why); Readback what step 4 copies.
enum class Settle { kAll, kLagged, kCheck, kNone };
enum class Readback { kIndex, kIndexAndLru, kNone };

// engine_index.cu
int alloc_index(fi_epp* h, uint64_t slots, uint32_t W, IndexTables& out);
int read_counters(fi_epp* h);
int settle_updates(fi_epp* h, bool lagged = false, uint64_t extra = 0);
int update_begin(fi_epp* h, Settle settle = Settle::kAll, uint64_t extra = 0);
int update_end(fi_epp* h, Readback rb = Readback::kIndex, cudaEvent_t done = nullptr);
int check_counters(fi_epp* h);
int check_counters_lagged(fi_epp* h, uint64_t extra);
GossipLog gossip_log(fi_epp* h);
int flush_ops(fi_epp* h);
int run_rounds(fi_epp* h, uint64_t mine, int my_err, const std::function<int(uint64_t)>& step);
int submit_op(fi_epp* h, uint64_t hash, uint32_t endpoint, uint32_t op);
int remove_local_endpoints(fi_epp* h, const std::vector<uint32_t>& local, uint64_t* pairs_removed);

// engine_lru.cu
int choose_lru_mode(fi_epp* h);
int size_dev_lru(fi_epp* h, uint32_t* TS, uint32_t* L);
int alloc_dev_lru(fi_epp* h, DevLruStore& s, uint32_t EL, uint32_t TS, uint32_t L, const uint32_t* caps);

// engine_comm.cu
int nccl_allgather_on(fi_epp* h, ncclComm_t comm, const void* send, void* recv, size_t bytes, cudaStream_t s);
int nccl_allgather(fi_epp* h, const void* send, void* recv, size_t bytes);

// engine.cu
void dump_trace(fi_epp* h, uint32_t R);
int sync_all_streams(fi_epp* h);
int check_whole_pool(fi_epp* h, const char* what);
int replace_begin(fi_epp* h);
int replace_commit(fi_epp* h, IndexTables* nix, std::unique_ptr<DevLruStore>& nlru, std::vector<uint32_t>& caps);

}  // namespace fi::engine
