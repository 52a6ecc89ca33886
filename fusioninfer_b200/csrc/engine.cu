// engine.cu — host side of libfi_epp: the C ABI of include/fi_epp.h.
//
// Owns the device buffers, two CUDA streams (compute, index maintenance),
// the pinned op ring that keeps the GPU index live (async H2D on the side stream,
// ordered before the next pick), the host LRU, the per-batch score tables, and the
// optional NCCL communicator for endpoint-range sharded pools.  No CPU fallback:
// creation fails without a CUDA device.
#include <cuda_runtime.h>
#include <unistd.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
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
#include "snapshot_format.h"
#include "xxh64.cuh"

using namespace fi;

namespace {

// ---- minimal NCCL binding through dlopen (the torch-bundled or the system libnccl.so.2) ----
typedef struct ncclComm* ncclComm_t;
typedef struct {
  char internal[128];
} ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1 };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool load(std::string* err) {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) {
      *err = std::string("dlopen libnccl.so.2 failed: ") + dlerror();
      return false;
    }
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllGather) {
      *err = "libnccl is missing a required symbol";
      return false;
    }
    return true;
  }
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

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

enum KernelKind { K_HASH = 0, K_MATCH = 1, K_INDEX = 2, K_OTHER = 3, K_KINDS = 4 };

uint32_t pow2_ceil32(uint32_t v) {
  uint32_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

// host cores this process may really use: the affinity mask capped by the cgroup CPU quota (more runnable
// threads than quota only get the group throttled)
unsigned usable_cores() {
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
  ~ShardState() {
    for (void* m : peer_ipc)
      if (m) cudaIpcCloseMemHandle(m);
    if (comm) g_nccl.CommDestroy(comm);
  }
};

}  // namespace

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
  DevPtr<EndpointDev> d_eps;
  DevPtr<double> d_sc;
  DevPtr<uint32_t> d_elig;
  DevPtr<ZeroBest> d_zero;
  DevPtr<uint32_t> d_ztie;
  std::vector<LoraDev> lora;   // local endpoints' adapter residency (lora-affinity-scorer)
  bool lora_dirty = false;
  DevPtr<LoraDev> d_lora;
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

namespace {

#define FI_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e__ = (call);                                                           \
    if (e__ != cudaSuccess) {                                                           \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e__);                     \
      return FI_ERR_CUDA;                                                               \
    }                                                                                   \
  } while (0)

int fail(fi_epp* h, int code, const std::string& m) {
  h->err = m;
  return code;
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

Event get_event(fi_epp* h) {
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

void drain_profile(fi_epp* h) {
  for (auto& e : h->pending_ev) {
    float ms = 0.f;
    if (cudaEventSynchronize(e.b.get()) == cudaSuccess && cudaEventElapsedTime(&ms, e.a.get(), e.b.get()) == cudaSuccess) {
      switch (e.kind) {
        case K_HASH: h->stats.ms_hash_blocks += ms; h->stats.n_hash_blocks++; break;
        case K_MATCH: h->stats.ms_match_pick += ms; h->stats.n_match_pick++; break;
        case K_INDEX: h->stats.ms_index_apply += ms; h->stats.n_index_apply++; break;
        default: h->stats.ms_other += ms; h->stats.n_other++; break;
      }
    }
    h->ev_pool.push_back(std::move(e.a));
    h->ev_pool.push_back(std::move(e.b));
  }
  h->pending_ev.clear();
}

size_t index_bytes(uint64_t slots, uint32_t W) {
  const uint64_t total = slots + 3;
  return total * (sizeof(uint64_t) * 2 + sizeof(uint32_t) * 3 + (size_t)W * sizeof(uint32_t));
}

// queue the clears that make `v` an empty index (on the index stream)
int clear_index(fi_epp* h, IndexView& v) {
  const uint64_t total = v.C + 3;
  FI_CUDA(cudaMemsetAsync(v.keys, 0, total * sizeof(uint64_t), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(v.node_of, 0xFF, total * sizeof(uint32_t), h->s_index.get()));  // NODE_INVALID
  FI_CUDA(cudaMemsetAsync(v.klog, 0, total * sizeof(uint64_t), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(v.rows, 0, total * v.W * sizeof(uint32_t), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(v.cnt, 0, total * sizeof(uint32_t), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(v.rmask, 0, total * sizeof(uint32_t), h->s_index.get()));
  return FI_OK;
}

// empty index tables of `slots` slots and rows of W words into `out`, which is left as it was on failure
int alloc_index(fi_epp* h, uint64_t slots, uint32_t W, IndexTables& out) {
  IndexTables t;
  IndexView& v = t.v;
  v.C = slots;
  v.bmask = slots / BUCKET_KEYS - 1;
  v.W = W;
  v.logW = 0;
  while ((1u << v.logW) < v.W) ++v.logW;
  const uint64_t total = slots + 3;  // + slots for hash 0, hash ~0, and a permanently-zero row
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && index_bytes(slots, v.W) + (256ull << 20) > free_b) {
    h->err = "index of " + std::to_string(index_bytes(slots, v.W) >> 20) + " MiB does not fit in the " +
             std::to_string(free_b >> 20) + " MiB of free device memory";
    return FI_ERR_NOMEM;
  }
  cudaError_t e = cuda_alloc(t.keys, total);
  if (e == cudaSuccess) e = cuda_alloc(t.node_of, total);
  if (e == cudaSuccess) e = cuda_alloc(t.klog, total);
  if (e == cudaSuccess) e = cuda_alloc(t.rows, total * v.W);
  if (e == cudaSuccess) e = cuda_alloc(t.cnt, total);
  if (e == cudaSuccess) e = cuda_alloc(t.rmask, total);
  if (e != cudaSuccess) {
    cudaGetLastError();
    h->err = std::string("index allocation: ") + cudaGetErrorString(e);
    return e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA;
  }
  v.keys = t.keys.get();
  v.node_of = t.node_of.get();
  v.klog = t.klog.get();
  v.rows = t.rows.get();
  v.cnt = t.cnt.get();
  v.rmask = t.rmask.get();
  int rc = clear_index(h, v);
  if (rc != FI_OK) return rc;
  out = std::move(t);
  return FI_OK;
}

// Compact the live nodes into the spare table and swap.  Everything is queued on the index stream — no host
// synchronisation: picks submitted later wait for ev_index and are launched with the new view; picks already in
// flight keep reading the old tables, which are not touched again before the NEXT rebuild, and that one is ordered
// behind them (the rebuild is an update: update_begin).
// The spare is allocated once, at the first rebuild (the only point where memory doubles), and then reused.
int rebuild_index(fi_epp* h) {
  if (!h->ix_spare) {
    auto spare = std::make_unique<IndexTables>();
    int rc = alloc_index(h, h->ix.v.C, h->ix.v.W, *spare);  // clears it too
    if (rc != FI_OK) return rc;
    h->ix_spare = std::move(spare);
  } else {
    int rc = clear_index(h, h->ix_spare->v);
    if (rc != FI_OK) return rc;
  }
  FI_CUDA(cudaMemsetAsync(h->d_ctr.get(), 0, sizeof(IndexCounters), h->s_index.get()));
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_rebuild(h->ix.v, h->ix_spare->v, h->d_ctr.get(), h->s_index.get()));
  }
  std::swap(h->ix, *h->ix_spare);  // owners and views together
  h->rebuilds++;
  return FI_OK;
}

// queue the copy of the index counters that the next check_counters reads
int read_counters(fi_epp* h) {
  FI_CUDA(cudaMemcpyAsync(h->h_ctr.get(), h->d_ctr.get(), sizeof(IndexCounters), cudaMemcpyDeviceToHost, h->s_index.get()));
  FI_CUDA(cudaEventRecord(h->ev_ctr.get(), h->s_index.get()));
  h->ctr_pending = true;
  return FI_OK;
}

int check_counters(fi_epp* h);
int check_counters_lagged(fi_epp* h, uint64_t extra);
int flush_ops(fi_epp* h);

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

int settle_updates(fi_epp* h, bool lagged = false, uint64_t extra = 0) {
  int rc = flush_ops(h);
  if (rc != FI_OK) return rc;
  return lagged ? check_counters_lagged(h, extra) : check_counters(h);
}

int update_begin(fi_epp* h, Settle settle = Settle::kAll, uint64_t extra = 0) {
  int rc = FI_OK;
  if (settle == Settle::kAll || settle == Settle::kLagged) rc = settle_updates(h, settle == Settle::kLagged, extra);
  if (settle == Settle::kCheck) rc = check_counters(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamWaitEvent(h->s_index.get(), h->ev_pick.get(), 0));
  return FI_OK;
}

// done (optional) is recorded behind the update's work and copies, before ev_index
int update_end(fi_epp* h, Readback rb = Readback::kIndex, cudaEvent_t done = nullptr) {
  cudaStream_t si = h->s_index.get();
  if (rb == Readback::kIndexAndLru) {
    FI_CUDA(cudaMemcpyAsync(&h->dlru->stat->error, h->dlru->v.error, sizeof(uint32_t), cudaMemcpyDeviceToHost, si));
    FI_CUDA(cudaMemcpyAsync(&h->dlru->stat->n_sets, h->dlru->ctr.get(), 5 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, si));
  }
  const int rc = rb == Readback::kNone ? FI_OK : read_counters(h);  // (ev_ctr covers the status copies too)
  if (rc != FI_OK) return rc;
  if (done) FI_CUDA(cudaEventRecord(done, si));
  FI_CUDA(cudaEventRecord(h->ev_index.get(), si));
  return FI_OK;
}

// look at the counters copied back after the previous flush; rebuild if the table is
// clogged with tombstones, fail if it is genuinely full
int check_counters(fi_epp* h) {
  if (!h->ctr_pending) return FI_OK;
  FI_CUDA(cudaEventSynchronize(h->ev_ctr.get()));
  h->ctr_pending = false;
  h->ctr_used_known = h->h_ctr->used;
  h->ctr_unchecked = 0;
  if (h->dlru && h->dlru->stat->error)
    return fail(h, FI_ERR_STATE, "device LRU: invariant " + std::to_string(h->dlru->stat->error) + " broken");
  if (h->dlru && h->dlru->stat->planned_ovf)
    return fail(h, FI_ERR_STATE, "device LRU: a table overflowed in a sub-batch planned not to (broken invariant)");
  if (h->h_ctr->overflow) return fail(h, FI_ERR_CAPACITY, "index full: raise index_slots");
  const uint64_t used = h->h_ctr->used, tomb = h->h_ctr->tombstones;
  if (used * 10 > h->ix.v.C * 7) {
    if ((used - tomb) * 10 > h->ix.v.C * 6) return fail(h, FI_ERR_CAPACITY, "index above 60% live keys: raise index_slots");
    int rc = update_begin(h, Settle::kNone);  // (inside the check already)
    if (rc == FI_OK) rc = rebuild_index(h);
    if (rc != FI_OK) return rc;
    return update_end(h, Readback::kNone);  // (a rebuild leaves the table below the rebuild threshold)
  }
  return FI_OK;
}

// check_counters without its host wait where the wait cannot change anything (the pipelined calls): the counters of
// the previous update are not in yet, but the last ones read leave room below the rebuild threshold for every key the
// unchecked updates and `extra` more touches can add (at most one each), so they cannot ask for a rebuild (or report
// a full index) yet.  Counters that are in are checked as always, and so are the device LRU's error flags.
int check_counters_lagged(fi_epp* h, uint64_t extra) {
  if (h->ctr_pending && h->world == 1) {
    const cudaError_t q = cudaEventQuery(h->ev_ctr.get());
    if (q == cudaErrorNotReady && (h->ctr_used_known + h->ctr_unchecked + extra) * 10 <= h->ix.v.C * 7) return FI_OK;
    if (q != cudaSuccess && q != cudaErrorNotReady) FI_CUDA(q);
  }
  return check_counters(h);
}

GossipLog gossip_log(fi_epp* h) {
  GossipLog g{};
  if (h->world > 1) {
    g.n_appear = h->shard->d_glog_n.get();
    g.n_vanish = h->shard->d_glog_n.get() + 1;
    g.appear = h->shard->d_glog_a.get();
    g.vanish = h->shard->d_glog_v.get();
    g.cap = kOpChunk;
  }
  return g;
}

// launch the staged SET then CLEAR ops of the current group on the index stream.
// Asynchronous: the only waits are for the *previous* group's counters (rebuild /
// overflow decisions lag one group) and for the staging buffer being reused.
int flush_ops(fi_epp* h) {
  if (h->n_sets == 0 && h->n_clears == 0) return FI_OK;
  int rc = update_begin(h, Settle::kCheck);  // may rebuild (swaps tables) — only ever between groups
  if (rc != FI_OK) return rc;
  const int b = h->cur_buf;
  const GossipLog gl = gossip_log(h);
  if (h->n_sets) {
    FI_CUDA(cudaMemcpyAsync(h->d_sets[b].get(), h->h_sets[b].get(), h->n_sets * sizeof(fi_index_op), cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += h->n_sets * sizeof(fi_index_op);
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_set(h->ix.v, h->d_ctr.get(), h->d_sets[b].get(), h->n_sets, h->cfg.endpoint_begin, h->cfg.endpoint_count, h->rank,
                             gl, h->s_index.get()));
  }
  if (h->n_clears) {
    FI_CUDA(cudaMemcpyAsync(h->d_clears[b].get(), h->h_clears[b].get(), h->n_clears * sizeof(fi_index_op), cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += h->n_clears * sizeof(fi_index_op);
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_clear(h->ix.v, h->d_ctr.get(), h->d_clears[b].get(), h->n_clears, h->cfg.endpoint_begin, h->cfg.endpoint_count,
                               h->rank, gl, h->s_index.get()));
  }
  h->ops_applied += h->n_sets + h->n_clears;
  h->ctr_unchecked += h->n_sets;
  FI_CUDA(cudaEventRecord(h->ev_buf[b].get(), h->s_index.get()));
  rc = update_end(h);
  if (rc != FI_OK) return rc;
  h->n_sets = h->n_clears = 0;
  h->cleared.clear();
  h->clears_untracked = false;
  h->cur_buf ^= 1;
  // the buffer we are about to fill must have been consumed
  FI_CUDA(cudaEventSynchronize(h->ev_buf[h->cur_buf].get()));
  return FI_OK;
}

int nccl_allgather_on(fi_epp* h, ncclComm_t comm, const void* send, void* recv, size_t bytes, cudaStream_t s);

// Sharded pools, one gossip round (collective: every rank calls it the same number of times): exchange the
// transition logs written by this round's SET / CLEAR kernels and replay the other ranks' into the local
// directory — all APPEARs before all VANISHes, like the SETs and CLEARs that produced them.
int gossip_round(fi_epp* h) {
  if (h->world <= 1) return FI_OK;
  ShardState& sh = *h->shard;
  const unsigned long long* hdr = sh.h_ghdr.get();
  const uint32_t Wd = h->world;
  int rc = update_begin(h, Settle::kNone);  // (a check could fail this rank before the collectives, or make it wait)
  if (rc != FI_OK) return rc;
  rc = nccl_allgather_on(h, sh.comm, sh.d_glog_n.get(), sh.d_ghdr.get(), 2 * sizeof(unsigned long long), h->s_index.get());
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaMemcpyAsync(sh.h_ghdr.get(), sh.d_ghdr.get(), (size_t)Wd * 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->s_index.get()));
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  uint64_t na = 0, nv = 0;
  for (uint32_t g = 0; g < Wd; ++g) {
    na = std::max<uint64_t>(na, hdr[2 * g]);
    nv = std::max<uint64_t>(nv, hdr[2 * g + 1]);
  }
  if (na > kOpChunk || nv > kOpChunk) return fail(h, FI_ERR_STATE, "gossip log overflow");
  if (na) {
    rc = nccl_allgather_on(h, sh.comm, sh.d_glog_a.get(), sh.d_ggather.get(), na * sizeof(uint64_t), h->s_index.get());
    if (rc != FI_OK) return rc;
    for (uint32_t g = 0; g < Wd; ++g) {
      if (g == h->rank || hdr[2 * g] == 0) continue;
      LaunchScope ls(h, h->s_index.get(), K_INDEX);
      FI_CUDA(launch_index_remote_appear(h->ix.v, h->d_ctr.get(), sh.d_ggather.get() + (size_t)g * na, hdr[2 * g], g, h->s_index.get()));
    }
  }
  if (nv) {
    rc = nccl_allgather_on(h, sh.comm, sh.d_glog_v.get(), sh.d_ggather.get(), nv * sizeof(uint64_t), h->s_index.get());
    if (rc != FI_OK) return rc;
    for (uint32_t g = 0; g < Wd; ++g) {
      if (g == h->rank || hdr[2 * g + 1] == 0) continue;
      LaunchScope ls(h, h->s_index.get(), K_INDEX);
      FI_CUDA(launch_index_remote_vanish(h->ix.v, h->d_ctr.get(), sh.d_ggather.get() + (size_t)g * nv, hdr[2 * g + 1], g, h->s_index.get()));
    }
  }
  FI_CUDA(cudaMemsetAsync(sh.d_glog_n.get(), 0, 2 * sizeof(unsigned long long), h->s_index.get()));
  return update_end(h, na || nv ? Readback::kIndex : Readback::kNone);  // (only the replays change the counters)
}

// One collective index update of a sharded pool = `rounds` gossip rounds on every rank: the ranks agree on the
// largest of their round counts `mine`, and `step(i)` stages and flushes this rank's share of round i (nothing if it
// has fewer).  A rank whose arguments were rejected (my_err) still takes part, with zero rounds, so that the others do
// not hang.  Single rank: just the steps.
int run_rounds(fi_epp* h, uint64_t mine, int my_err, const std::function<int(uint64_t)>& step) {
  if (my_err != FI_OK) {
    if (h->world <= 1) return my_err;
    mine = 0;
  }
  uint64_t rounds = mine;
  if (h->world > 1) {
    ShardState& sh = *h->shard;
    unsigned long long v[2] = {mine, 0};
    FI_CUDA(cudaMemcpyAsync(sh.d_ghdr.get() + 2 * (size_t)h->world, v, sizeof(v), cudaMemcpyHostToDevice, h->s_index.get()));
    int rc = nccl_allgather_on(h, sh.comm, sh.d_ghdr.get() + 2 * (size_t)h->world, sh.d_ghdr.get(), sizeof(v), h->s_index.get());
    if (rc != FI_OK) return rc;
    FI_CUDA(cudaMemcpyAsync(sh.h_ghdr.get(), sh.d_ghdr.get(), (size_t)h->world * sizeof(v), cudaMemcpyDeviceToHost, h->s_index.get()));
    FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
    for (uint32_t g = 0; g < h->world; ++g) rounds = std::max<uint64_t>(rounds, sh.h_ghdr.get()[2 * g]);
  }
  for (uint64_t i = 0; i < rounds; ++i) {
    int rc = i < mine ? step(i) : FI_OK;
    if (rc == FI_OK) rc = gossip_round(h);
    if (rc != FI_OK) return rc;
  }
  return my_err;
}

// Stage one op (already filtered to this shard) in the open group.  The GPU applies a group as all its SETs, then all
// its CLEARs, so a SET that follows a CLEAR of the same pair starts a new group.  `cleared` holds the pairs CLEARed in
// the group, unless clears_untracked: fi_epp_index_add_chains stages its CLEARs in bulk without recording them, and
// until the next flush every SET then counts as following a CLEAR of its pair if the group holds any CLEAR.
int submit_op(fi_epp* h, uint64_t hash, uint32_t endpoint, uint32_t op) {
  if (op == FI_OP_SET) {
    if (h->n_clears && (h->clears_untracked || h->cleared.count(PairKey{hash, endpoint}))) {
      int rc = flush_ops(h);
      if (rc != FI_OK) return rc;
    }
    h->h_sets[h->cur_buf].get()[h->n_sets++] = fi_index_op{hash, endpoint, FI_OP_SET};
  } else {
    h->cleared.insert(PairKey{hash, endpoint});
    h->h_clears[h->cur_buf].get()[h->n_clears++] = fi_index_op{hash, endpoint, FI_OP_CLEAR};
  }
  if (h->n_sets == kOpChunk || h->n_clears == kOpChunk) return flush_ops(h);
  return FI_OK;
}

// ---- device-resident LRU (lru_kernels.cu) --------------------------------------------------------------
// Which LRU serves this handle's indexer.Add calls: decided at the first one.
int choose_lru_mode(fi_epp* h) {
  if (h->lru_mode >= 0) return FI_OK;
  int want = h->lru_want;
  if (want < 0) {
    if (const char* e = std::getenv("FI_EPP_DEVICE_LRU")) want = std::strtol(e, nullptr, 10) != 0;
  }
  const bool possible = h->cfg.lru_capacity >= h->cfg.max_blocks && h->cfg.lru_capacity <= (1u << 28);
  if (want == 1 && !possible) return fail(h, FI_ERR_STATE, "device_lru needs lru_capacity >= max_blocks");
  h->lru_mode = (want < 0 ? possible : want == 1) ? 1 : 0;
  return FI_OK;
}

// the per-request arguments of a batched Add: every endpoint in range or FI_NO_ENDPOINT, every chain at most
// max_nblocks long (`bound` names that limit)
int check_add_requests(fi_epp* h, const uint32_t* endpoints, const uint32_t* nblocks, uint32_t R, uint32_t max_nblocks,
                       const char* bound) {
  for (uint32_t r = 0; r < R; ++r) {
    if (endpoints[r] != FI_NO_ENDPOINT && endpoints[r] >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint out of range");
    if (nblocks[r] > max_nblocks) return fail(h, FI_ERR_INVALID, std::string("nblocks[r] larger than ") + bound);
  }
  return FI_OK;
}

// The device LRU's table size TS and log size L, chosen at its first Add and kept for its life (fi_epp_resize_pool
// keeps them too).
int size_dev_lru(fi_epp* h, uint32_t* TS, uint32_t* L) {
  const uint32_t EL = h->cfg.endpoint_count, C = h->cfg.lru_capacity;
  size_t free_b = 0, total_b = 0;
  FI_CUDA(cudaMemGetInfo(&free_b, &total_b));
  // Log: at least 4 C records (a sub-batch appends at most C; more room = rarer compaction).  Table: at least 4 C slots (C entries + C new keys of a
  // conservative sub-batch + tombstones); a table takes a batch's DISTINCT keys on top of its entries, and an
  // endpoint that attracts a popular prefix can receive a large share of a batch — so the tables get as much as
  // a quarter of the free HBM buys, up to 32 C slots (1 Mi slots = 16 MiB per endpoint at lruCapacityPerServer
  // 31 250: 17 GB for 1 024 endpoints, a fifth of an H100's 80).  Option "lru_table_slots" / FI_EPP_LRU_TABLE_SLOTS pins it.
  const uint32_t log_min = std::max<uint32_t>(pow2_ceil32(4u * C), 64u);
  const uint32_t ts_min = log_min;
  uint32_t ts = pow2_ceil32(32u * C);
  while (ts > ts_min && (size_t)EL * (ts + 2) * sizeof(LruSlot) > free_b / 4) ts >>= 1;
  uint32_t want = h->lru_table_slots;
  if (!want)
    if (const char* ev = std::getenv("FI_EPP_LRU_TABLE_SLOTS")) want = (uint32_t)std::strtoul(ev, nullptr, 10);
  if (want) ts = std::max(ts_min, pow2_ceil32(want));
  *TS = ts;
  *L = std::max(log_min, ts / 4);
  return FI_OK;
}

// the device LRU's buffers for EL local endpoints, tables of TS slots and logs of L records, all or nothing: `s` is
// filled only as far as it got when a step fails.  Every LRU starts empty, endpoint e with capacity caps[e] (a
// pageable host array: taken when the call returns).
int alloc_dev_lru(fi_epp* h, DevLruStore& s, uint32_t EL, uint32_t TS, uint32_t L, const uint32_t* caps) {
  DevLru& d = s.v;
  d.EL = EL;
  d.capacity = h->cfg.lru_capacity;
  d.TS = TS;
  d.L = L;
  d.insert_limit = (uint32_t)((uint64_t)d.TS * 85 / 100);
  size_t free_b = 0, total_b = 0;
  FI_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const size_t slots = (size_t)EL * (d.TS + 2), log_records = (size_t)EL * d.L;
  s.touch_cap = std::max<uint64_t>((uint64_t)h->cfg.max_batch * h->MP, 1u << 16);
  const size_t scratch = (size_t)s.touch_cap * (sizeof(uint32_t) + 3 * sizeof(fi_index_op));
  if (slots * sizeof(LruSlot) + log_records * sizeof(uint64_t) + scratch + (256u << 20) > free_b)
    return fail(h, FI_ERR_NOMEM, "device LRU does not fit in free HBM (option device_lru = 0 selects the host LRU)");
  const size_t state_words = (size_t)8 * EL + 2;
  FI_CUDA(cuda_alloc(s.slots, slots));
  FI_CUDA(cuda_alloc(s.log, log_records));
  FI_CUDA(cuda_alloc(s.state, state_words));
  FI_CUDA(cuda_alloc(s.ctr, 8));
  FI_CUDA(cuda_alloc(s.stat, 1));
  std::memset(s.stat.get(), 0, sizeof(DevLruStore::HostStat));
  FI_CUDA(cuda_alloc(s.slot_of, s.touch_cap));
  FI_CUDA(cuda_alloc(s.sets, s.touch_cap));
  FI_CUDA(cuda_alloc(s.clears, 2 * s.touch_cap));  // doomed keys + evictions
  FI_CUDA(cuda_alloc(s.wcount, h->cfg.max_batch));
  FI_CUDA(cuda_alloc(s.base, h->cfg.max_batch));
  FI_CUDA(cuda_create(s.ev));
  FI_CUDA(cuda_create(s.ev_ovf));
  FI_CUDA(cudaMemsetAsync(s.slots.get(), 0, slots * sizeof(LruSlot), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(s.state.get(), 0, state_words * sizeof(uint32_t), h->s_index.get()));
  FI_CUDA(cudaMemsetAsync(s.ctr.get(), 0, 8 * sizeof(unsigned long long), h->s_index.get()));
  FI_CUDA(cudaEventRecord(s.ev.get(), h->s_index.get()));
  d.slots = s.slots.get();
  d.log = s.log.get();
  d.head = s.state.get();
  d.tail = d.head + EL;
  d.count = d.tail + EL;
  d.used = d.count + EL;
  d.hold = d.used + EL;
  d.dcount = d.hold + EL;
  d.ovf = d.dcount + EL;
  d.any_ovf = d.ovf + EL;
  d.error = d.any_ovf + 1;
  d.cap = d.error + 1;
  FI_CUDA(cudaMemcpyAsync(d.cap, caps, (size_t)EL * sizeof(uint32_t), cudaMemcpyHostToDevice, h->s_index.get()));
  d.n_sets = s.ctr.get();
  d.n_maintained = s.ctr.get() + 1;
  d.n_clears = s.ctr.get() + 3;
  d.n_doomed = s.ctr.get() + 4;
  return FI_OK;
}

// the device LRU is allocated whole at the first Add; nothing of a failed allocation survives (a later call may
// succeed, e.g. with the host LRU freed)
int ensure_dev_lru(fi_epp* h) {
  if (h->dlru) return FI_OK;
  const uint32_t EL = h->cfg.endpoint_count;
  uint32_t TS = 0, L = 0;
  int rc = size_dev_lru(h, &TS, &L);
  if (rc != FI_OK) return rc;
  // the capacities set so far (possibly before this first Add)
  if (h->lru_caps.size() != EL) h->lru_caps.assign(EL, h->cfg.lru_capacity);
  auto s = std::make_unique<DevLruStore>();
  rc = alloc_dev_lru(h, *s, EL, TS, L, h->lru_caps.data());
  if (rc != FI_OK) {
    cudaGetLastError();
    return rc;
  }
  h->dlru = std::move(s);
  return FI_OK;
}

// One sub-batch of a planned Add (the plan packed at `dp` by lru_plan_pack): the view the LRU kernels take, and the
// kernels themselves.  Both Add paths (lru_device_add, lru_add_submitted) enqueue a sub-batch through these two.
LruBatch lru_sub_batch(fi_epp* h, const uint32_t* dp, const LruPlan& pl, size_t sb, const uint64_t* chains, uint32_t pitch,
                       const uint32_t** inc) {
  const LruPlanOffsets o = lru_plan_offsets(pl, h->cfg.endpoint_count, sb);
  LruBatch b{};
  b.req_id = dp + o.req_id;
  b.req_ep = dp + o.req_ep;
  b.req_n = dp + o.req_n;
  b.req_off = dp + o.req_off;
  b.ep_list = dp + o.ep_list;
  b.ep_start = dp + o.ep_start;
  *inc = dp + o.inc;
  b.chains = chains;
  b.pitch = pitch;
  b.K = pl.subs[sb].k_end - pl.subs[sb].k_begin;
  b.slot_of = h->dlru->slot_of.get();
  b.wcount = h->dlru->wcount.get();
  b.base = h->dlru->base.get();
  b.sets = h->dlru->sets.get();
  return b;
}

// maintain (log compaction / table rebuild) and touch of one sub-batch
int lru_enqueue_touch(fi_epp* h, const LruBatch& b, const uint32_t* inc) {
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_maintain(h->dlru->v, inc, false, h->s_index.get()));
  }
  LaunchScope ls(h, h->s_index.get(), K_INDEX);
  FI_CUDA(launch_lru_touch(h->dlru->v, b, h->s_index.get()));
  return FI_OK;
}

// the rest of one sub-batch after its touch: winners, log records, index SETs, evictions, index CLEARs (clear_ovf:
// then the overflow flags of the touch are reset); unless it is the update's last sub-batch, the index counters are
// copied back for the rebuild decision before the next one
int lru_enqueue_apply(fi_epp* h, const LruBatch& b, uint64_t touches, const GossipLog& glog, bool clear_ovf, bool last) {
  const uint32_t EL = h->cfg.endpoint_count, lo = h->cfg.endpoint_begin;
  FI_CUDA(cudaMemsetAsync(h->dlru->ctr.get() + 2, 0, sizeof(unsigned long long), h->s_index.get()));
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_count(h->dlru->v, b, h->s_index.get()));
  }
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_scan(h->dlru->v, b, h->s_index.get()));
  }
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_append(h->dlru->v, b, h->dlru->clears.get(), h->dlru->ctr.get() + 2, 2 * h->dlru->touch_cap, lo, h->s_index.get()));
  }
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_set(h->ix.v, h->d_ctr.get(), h->dlru->sets.get(), touches, lo, EL, h->rank, glog, h->s_index.get()));
  }
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_evict(h->dlru->v, h->dlru->clears.get(), h->dlru->ctr.get() + 2, 2 * h->dlru->touch_cap, lo, h->s_index.get()));
  }
  {
    // CLEARs of a sub-batch: at most one per doomed key (<= touches) and one per eviction (<= keys it added)
    const uint64_t cap = std::min<uint64_t>(2 * h->dlru->touch_cap, 2 * touches);
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_clear_counted(h->ix.v, h->d_ctr.get(), h->dlru->clears.get(), cap, h->dlru->ctr.get() + 2, lo, EL, h->rank, glog,
                                       h->s_index.get()));
  }
  if (clear_ovf) FI_CUDA(cudaMemsetAsync(h->dlru->v.ovf, 0, ((size_t)EL + 1) * sizeof(uint32_t), h->s_index.get()));  // ovf[] and any_ovf
  h->ctr_unchecked += touches;
  return last ? FI_OK : read_counters(h);
}

// What both device-LRU Adds need before they plan: the LRU exists and every local chain fits lru_capacity.
int lru_add_prepare(fi_epp* h, const uint32_t* endpoints, const uint32_t* nblocks, uint32_t R) {
  int rc = ensure_dev_lru(h);
  if (rc != FI_OK) return rc;
  for (uint32_t r = 0; r < R; ++r)
    if (nblocks[r] > h->cfg.lru_capacity && endpoints[r] - h->cfg.endpoint_begin < h->cfg.endpoint_count)
      return fail(h, FI_ERR_INVALID, "device LRU: a chain longer than lru_capacity");
  return FI_OK;
}

// Pack plan `pl` into `buf` once `done` says the device has consumed the plan staged there before, and upload it on
// the index stream.
int lru_stage_plan(fi_epp* h, Staging<uint32_t>& buf, const LruPlan& pl, cudaEvent_t done) {
  const size_t words = lru_plan_words(pl, h->cfg.endpoint_count);
  FI_CUDA(cudaEventSynchronize(done));
  int rc = grow_staging(h, buf, words, words + words / 2 + 1024, true);  // room to spare: plans vary in size
  if (rc != FI_OK) return rc;
  lru_plan_pack(pl, buf.h.get());
  if (words) FI_CUDA(cudaMemcpyAsync(buf.d.get(), buf.h.get(), words * sizeof(uint32_t), cudaMemcpyHostToDevice, h->s_index.get()));
  h->stats.h2d_bytes += words * sizeof(uint32_t);
  return FI_OK;
}

// copy the rows of host `chains` that plan `pl` keeps to the device staging; *d_chains = where they are
int lru_stage_chains(fi_epp* h, const uint64_t* chains, uint32_t pitch, uint32_t R, const LruPlan& pl, const uint64_t** d_chains) {
  const size_t K = pl.req_id.size(), cw = (size_t)R * pitch;
  int rc = grow_staging(h, h->lru_chains, cw, cw, false);
  if (rc != FI_OK) return rc;
  *d_chains = h->lru_chains.d.get();
  // whole-range copy when most rows are kept (one DMA), row copies otherwise
  if (K * 2 >= R) {
    FI_CUDA(cudaMemcpyAsync(h->lru_chains.d.get(), chains, cw * sizeof(uint64_t), cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += cw * sizeof(uint64_t);
    return FI_OK;
  }
  for (size_t k = 0; k < K; ++k) {
    const size_t r = pl.req_id[k];
    FI_CUDA(cudaMemcpyAsync(h->lru_chains.d.get() + r * pitch, chains + r * pitch, (size_t)pl.req_n[k] * sizeof(uint64_t),
                            cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += (size_t)pl.req_n[k] * sizeof(uint64_t);
  }
  return FI_OK;
}

// indexer.Add(chains[r], endpoints[r]) for r = 0..R-1 through the device LRU.  `chains` is a host pointer
// (copied to the device first) or, with on_device, memory the index stream can read.  The first pass is
// OPTIMISTIC: sub-batches are cut only by the scratch arrays' size, and an endpoint whose table cannot take the
// batch's distinct keys is rolled back and deferred; the deferred requests then run in a second, conservative pass
// (at most lru_capacity touches per endpoint and sub-batch: always fits).  On a sharded pool both passes are
// collective (one gossip round per sub-batch) and every rank takes part in both, one whose arguments were rejected
// (my_err) with no sub-batches.
int lru_device_add(fi_epp* h, const uint32_t* endpoints, const uint64_t* chains, bool on_device, uint32_t pitch,
                   const uint32_t* nblocks, uint32_t R, int my_err) {
  if (my_err == FI_OK) my_err = lru_add_prepare(h, endpoints, nblocks, R);
  const uint32_t EL = h->cfg.endpoint_count, lo = h->cfg.endpoint_begin;
  const bool sharded = h->world > 1;
  LruPlan& pl = h->lru_plan;
  std::vector<uint32_t> ep2;  // the conservative pass's endpoints: the deferred requests' (FI_NO_ENDPOINT elsewhere)
  for (const bool conservative : {false, true}) {
    const auto t0 = std::chrono::steady_clock::now();
    size_t K = 0, nsub = 0;
    if (my_err == FI_OK) {
      // sharded pool: a sub-batch's APPEAR / VANISH transitions must fit the gossip log of one round (at most one SET
      // per touch; CLEARs: evictions <= keys added, plus doomed entries <= touches)
      const uint64_t cap_touches = sharded ? std::min<uint64_t>(h->dlru->touch_cap, kOpChunk / 2) : h->dlru->touch_cap;
      lru_plan_batch(endpoints, nblocks, R, lo, EL, conservative ? h->cfg.lru_capacity : 0xFFFFFFFFu, cap_touches, h->cfg.max_batch, &pl);
      if (pl.subs.empty() && !sharded) return settle_updates(h);
      K = pl.req_id.size();
      nsub = pl.subs.size();
      my_err = update_begin(h);
      if (my_err == FI_OK) my_err = lru_stage_plan(h, h->lru_plan_buf, pl, h->dlru->ev.get());  // (dlru->ev covers the chain staging too)
    }
    if (my_err == FI_OK && !on_device && K) my_err = lru_stage_chains(h, chains, pitch, R, pl, &chains);
    if (my_err == FI_OK) h->lru_sub_batches += nsub;
    const GossipLog glog = gossip_log(h);
    std::vector<uint8_t> deferred;  // per request of this call: its endpoint overflowed in the optimistic pass
    std::vector<uint32_t> ovf_host;
    size_t n_deferred = 0;
    int rc = run_rounds(h, nsub, my_err, [&](uint64_t sb) -> int {
      if (sb) {  // the index counters of the previous sub-batch decide about a rebuild before more keys arrive
        const int rc2 = check_counters(h);
        if (rc2 != FI_OK) return rc2;
      }
      const LruSubBatch& sbt = pl.subs[sb];
      const uint32_t* inc = nullptr;
      const LruBatch b = lru_sub_batch(h, h->lru_plan_buf.d.get(), pl, sb, chains, pitch, &inc);
      const int rc2 = lru_enqueue_touch(h, b, inc);
      if (rc2 != FI_OK) return rc2;
      // did some endpoint's table refuse keys?  (one host round trip per sub-batch; everything after it is queued
      // without waiting)
      FI_CUDA(cudaMemcpyAsync(&h->dlru->stat->any_ovf, h->dlru->v.any_ovf, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_index.get()));
      FI_CUDA(cudaEventRecord(h->dlru->ev_ovf.get(), h->s_index.get()));
      FI_CUDA(cudaEventSynchronize(h->dlru->ev_ovf.get()));
      const bool any_ovf = h->dlru->stat->any_ovf != 0;
      if (any_ovf) {
        if (conservative) return fail(h, FI_ERR_STATE, "device LRU: overflow in a conservative sub-batch");
        {
          LaunchScope ls(h, h->s_index.get(), K_INDEX);
          FI_CUDA(launch_lru_untouch(h->dlru->v, b, h->s_index.get()));
        }
        ovf_host.resize(EL);
        FI_CUDA(cudaMemcpyAsync(ovf_host.data(), h->dlru->v.ovf, (size_t)EL * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_index.get()));
        FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
        if (deferred.empty()) deferred.assign(R, 0);
        for (uint32_t k = sbt.k_begin; k < sbt.k_end; ++k)
          if (ovf_host[pl.req_ep[k]]) {
            deferred[pl.req_id[k]] = 1;
            ++n_deferred;
          }
      }
      return lru_enqueue_apply(h, b, sbt.touches, glog, any_ovf, sb + 1 == nsub);
    });
    if (rc != (sharded ? my_err : FI_OK)) return rc;  // (a sharded rank with my_err goes on to the second pass)
    if (my_err != FI_OK) continue;
    rc = update_end(h, Readback::kIndexAndLru, h->dlru->ev.get());
    if (rc != FI_OK) return rc;
    if (h->verbose) {
      const auto t1 = std::chrono::steady_clock::now();
      std::fprintf(stderr, "[fi_epp] device LRU%s: %u requests (%zu kept), %zu sub-batch(es), %zu deferred, host side %.3f ms\n",
                   conservative ? " (conservative pass)" : "", R, K, nsub, n_deferred,
                   std::chrono::duration<double, std::milli>(t1 - t0).count());
    }
    h->lru_deferred += n_deferred;
    // (sharded: every rank enters the second pass, most with nothing to do)
    if (conservative || (!n_deferred && !sharded)) return FI_OK;
    ep2.assign(R, FI_NO_ENDPOINT);
    for (uint32_t r = 0; r < R; ++r)
      if (n_deferred && deferred[r]) ep2[r] = endpoints[r];
    endpoints = ep2.data();
    on_device = true;  // `chains` is in device memory now
  }
  return my_err;
}

// the index-stream part of lru_add_submitted behind the plan upload: the chain copy out of the slot, the sub-batches,
// the copy of the touch kernel's overflow flag
int lru_add_submitted_enqueue(fi_epp* h, uint32_t slot, const LruPlan& pl, fi_epp::PipeAdd& pa, uint32_t R) {
  const uint64_t* slot_chain = slot ? h->d_chain2.get() : h->d_chain.get();
  FI_CUDA(cudaStreamWaitEvent(h->s_copy.get(), h->ev_a[slot].get(), 0));  // the batch's chains are written
  FI_CUDA(cudaMemcpyAsync(pa.d_chains.get(), slot_chain, (size_t)R * h->MP * sizeof(uint64_t), cudaMemcpyDeviceToDevice, h->s_copy.get()));
  FI_CUDA(cudaEventRecord(h->ev_slot_read[slot].get(), h->s_copy.get()));
  FI_CUDA(cudaStreamWaitEvent(h->s_index.get(), h->ev_slot_read[slot].get(), 0));
  const GossipLog glog = gossip_log(h);
  h->lru_sub_batches += pl.subs.size();
  for (size_t sb = 0; sb < pl.subs.size(); ++sb) {
    const uint64_t touches = pl.subs[sb].touches;
    int rc = sb ? check_counters_lagged(h, touches) : FI_OK;  // may rebuild the index (update_begin checked the first)
    if (rc != FI_OK) return rc;
    const uint32_t* inc = nullptr;
    const LruBatch b = lru_sub_batch(h, pa.plan.d.get(), pl, sb, pa.d_chains.get(), h->MP, &inc);
    rc = lru_enqueue_touch(h, b, inc);
    if (rc != FI_OK) return rc;
    rc = lru_enqueue_apply(h, b, touches, glog, false, sb + 1 == pl.subs.size());
    if (rc != FI_OK) return rc;
  }
  FI_CUDA(cudaMemcpyAsync(&h->dlru->stat->planned_ovf, h->dlru->v.any_ovf, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_index.get()));
  return FI_OK;
}

// fi_epp_index_add_submitted: indexer.Add(chain_r, endpoints[r]) for the batch whose chains pipeline slot `slot`
// holds.  Unlike lru_device_add, which waits on the host for the device in every sub-batch:
//  - sub-batches are cut with lru_touch_bound (lru_plan.h), so no table can overflow: there is no optimistic pass,
//    no overflow readback and no deferral (the touch kernel's flag is still copied back and reported as a broken
//    invariant by the next counters check);
//  - the plan and chain staging are double-buffered: the call waits at most for the Add before the previous one;
//  - the index counters may lag (check_counters_lagged) — while the lag rule holds; when it does not (an index near
//    its rebuild threshold), the call waits for the previous update's counters as lru_device_add does;
//  - the chains are first copied out of the slot on s_copy, as soon as the batch's hashing is done, so that the submit
//    that reuses the slot waits for that copy only and not for this Add, which runs behind the picks in flight.
int lru_add_submitted(fi_epp* h, uint32_t slot, const uint32_t* endpoints, const uint32_t* nblocks, uint32_t R) {
  int rc = lru_add_prepare(h, endpoints, nblocks, R);
  if (rc != FI_OK) return rc;
  LruPlan& pl = h->lru_plan;
  lru_plan_batch(endpoints, nblocks, R, h->cfg.endpoint_begin, h->cfg.endpoint_count, lru_touch_bound(h->dlru->v.TS, h->dlru->v.capacity),
                 h->dlru->touch_cap, h->cfg.max_batch, &pl);
  if (pl.subs.empty()) return flush_ops(h);
  fi_epp::PipeAdd& pa = h->padd[h->padd_seq & 1];
  if (!pa.ev_done) {
    Event ev;
    DevPtr<uint64_t> chains;
    FI_CUDA(cuda_create(ev));
    FI_CUDA(cuda_alloc(chains, (size_t)h->cfg.max_batch * h->MP));
    pa.ev_done = std::move(ev);
    pa.d_chains = std::move(chains);
  }
  rc = update_begin(h, Settle::kLagged, pl.subs[0].touches);
  if (rc == FI_OK) rc = lru_stage_plan(h, pa.plan, pl, pa.ev_done.get());  // waits for the Add before the previous one
  if (rc != FI_OK) return rc;
  // From here on work that reads pa's buffers is queued: whatever happens, pa.ev_done marks its end (the s_index wait
  // on the chain copy makes it cover that copy too), and the next call takes the other buffers.
  rc = lru_add_submitted_enqueue(h, slot, pl, pa, R);
  if (rc == FI_OK) rc = update_end(h, Readback::kIndexAndLru, pa.ev_done.get());
  if (rc != FI_OK && cudaStreamWaitEvent(h->s_index.get(), h->ev_slot_read[slot].get(), 0) == cudaSuccess)
    cudaEventRecord(pa.ev_done.get(), h->s_index.get());
  h->padd_seq++;
  return rc;
}

// fi_epp_set_lru_capacities on the device LRU: upload the new capacities `caps`, then evict the listed local endpoints
// down to them and CLEAR the evicted pairs.  lru_shrink_kernel writes its CLEARs to the same buffer as an Add's
// evictions (2 lru_touch_cap ops) and would drop any beyond it, while a shrink can evict far more (1 024 pods halved
// from 31 250 entries: 16 M).  So the evictions run in ROUNDS of at most one buffer each, planned on the host from the
// endpoints' entry counts (a control-plane readback, which waits for the index updates queued so far); an endpoint
// with more evictions than a round takes is evicted part of the way per round, oldest first, so the rounds together
// evict exactly what one pass would.  Only a lowered capacity can evict: without one there is no readback and nothing
// blocks.  Everything that can fail without a CUDA error (the readback, the staging) happens before the capacities
// reach the device, so a failed call leaves them as they were.  *evicted += entries evicted.
int lru_device_resize(fi_epp* h, const std::vector<uint32_t>& local, const std::vector<uint32_t>& caps, uint64_t* evicted) {
  const uint32_t EL = h->cfg.endpoint_count, lo = h->cfg.endpoint_begin;
  bool lowered = false;
  for (uint32_t e : local) lowered |= caps[e] < h->lru_caps[e];
  std::vector<uint32_t> cnt;
  if (lowered) {  // the entries every endpoint holds once the Adds queued so far have run
    cnt.resize(EL);
    FI_CUDA(cudaMemcpyAsync(cnt.data(), h->dlru->v.count, (size_t)EL * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_index.get()));
    FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  }
  // rounds: (endpoint, quota) pairs, at most clears_cap evictions per round; an endpoint is listed once per round
  const uint64_t clears_cap = 2 * h->dlru->touch_cap;
  std::vector<uint32_t> r_eps, r_quota;
  std::vector<size_t> r_begin{0};
  std::vector<uint64_t> r_total;
  uint64_t fill = 0;
  for (uint32_t e : local) {
    uint64_t over = lowered && cnt[e] > caps[e] ? cnt[e] - caps[e] : 0;
    while (over) {
      const uint64_t take = std::min(over, clears_cap - fill);
      r_eps.push_back(e);
      r_quota.push_back((uint32_t)take);
      fill += take;
      over -= take;
      *evicted += take;
      if (fill == clears_cap) {
        r_begin.push_back(r_eps.size());
        r_total.push_back(fill);
        fill = 0;
      }
    }
  }
  if (fill) {
    r_begin.push_back(r_eps.size());
    r_total.push_back(fill);
  }
  const size_t pairs = r_eps.size();
  if (pairs) {
    // (the previous resize's copy out of the pinned buffer is done: the readback above synchronised s_index)
    int rc = grow_staging(h, h->lru_resize, 2 * pairs, 2 * pairs, true);
    if (rc != FI_OK) return rc;
    std::memcpy(h->lru_resize.h.get(), r_eps.data(), pairs * sizeof(uint32_t));
    std::memcpy(h->lru_resize.h.get() + pairs, r_quota.data(), pairs * sizeof(uint32_t));
  }
  int rc = update_begin(h, Settle::kNone);  // (the caller settled before the readback, which must not wait for picks)
  if (rc != FI_OK) return rc;
  // (pageable source: the copy has taken the data when cudaMemcpyAsync returns)
  FI_CUDA(cudaMemcpyAsync(h->dlru->v.cap, caps.data(), (size_t)EL * sizeof(uint32_t), cudaMemcpyHostToDevice, h->s_index.get()));
  h->stats.h2d_bytes += (size_t)EL * sizeof(uint32_t);
  if (pairs) {
    FI_CUDA(cudaMemcpyAsync(h->lru_resize.d.get(), h->lru_resize.h.get(), 2 * pairs * sizeof(uint32_t), cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += 2 * pairs * sizeof(uint32_t);
  }
  const GossipLog glog = gossip_log(h);
  for (size_t k = 0; k < r_total.size(); ++k) {
    const size_t b = r_begin[k];
    const uint32_t n = (uint32_t)(r_begin[k + 1] - b);
    FI_CUDA(cudaMemsetAsync(h->dlru->ctr.get() + 2, 0, sizeof(unsigned long long), h->s_index.get()));
    {
      LaunchScope ls(h, h->s_index.get(), K_INDEX);
      FI_CUDA(launch_lru_shrink(h->dlru->v, h->lru_resize.d.get() + b, h->lru_resize.d.get() + pairs + b, n, h->dlru->clears.get(), h->dlru->ctr.get() + 2,
                                clears_cap, lo, h->s_index.get()));
    }
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_clear_counted(h->ix.v, h->d_ctr.get(), h->dlru->clears.get(), r_total[k], h->dlru->ctr.get() + 2, lo, EL, h->rank, glog,
                                       h->s_index.get()));
  }
  return update_end(h, Readback::kIndexAndLru);
}

// Whether a pick may hash each request only up to its first block the index does not hold (hash_kernels.cu "early
// exit"): the pick reads nothing past that block, and here nothing else reads the chains either.  That needs a single
// rank (a sharded pool gathers and merges over whole chains), hash_chain (block_bytes % 32 == 0), no chains_out, and
// no LRU (lru_capacity == 0: no device-LRU Add can take the batch's chains from the handle's buffers; the index is fed
// by fi_epp_index_apply alone).  Every other batch, and fi_epp_hash_batch, hashes whole chains.
bool early_exit_hashing(const fi_epp* h, bool chains_wanted) {
  return h->world == 1 && h->fast_hash && !chains_wanted && h->cfg.lru_capacity == 0;
}

// blocks hash_chain read the prompt bytes of, while profiling (slot 6 of d_probed; 0 is N_probe, 1-5 the
// FI_MATCH_TIMING sums)
unsigned long long* hashed_counter(fi_epp* h) { return h->profiling ? h->d_probed.get() + 6 : nullptr; }

// hash kernels for the request slice [r0, r0+R): prompts → chain (device buffers), on stream s.  early: the index
// view the batch's match reads, when early_exit_hashing allows it (s must already wait for ev_index), else null
int run_hash(fi_epp* h, const uint8_t* d_prompts, const uint64_t* d_offsets, const uint64_t* d_h0, uint32_t r0,
             uint32_t R, cudaStream_t s, const IndexView* early) {
  uint64_t* chain = h->d_chain.get() + (size_t)r0 * h->MP;
  uint32_t* nb = h->d_nblocks.get() + r0;
  LaunchScope ls(h, s, K_HASH);
  if (h->fast_hash) {  // block hashing and chain walk in one kernel, no pre-states in HBM
    FI_CUDA(launch_hash_chain(d_prompts, d_offsets + r0, d_h0 + r0, R, h->cfg.block_bytes, h->cfg.max_blocks, h->MP,
                              chain, nb, h->sm_count, s, early, hashed_counter(h)));
  } else {
    FI_CUDA(launch_hash_generic(d_prompts, d_offsets + r0, d_h0 + r0, R, h->cfg.block_bytes, h->cfg.max_blocks, h->MP,
                                chain, nb, s));
  }
  return FI_OK;
}

int nccl_allgather_on(fi_epp* h, ncclComm_t comm, const void* send, void* recv, size_t bytes, cudaStream_t s) {
  int rc = g_nccl.AllGather(send, recv, bytes, ncclInt8, comm, s);
  if (rc != ncclSuccess)
    return fail(h, FI_ERR_COMM, std::string("ncclAllGather: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"));
  return FI_OK;
}
int nccl_allgather(fi_epp* h, const void* send, void* recv, size_t bytes) {
  return nccl_allgather_on(h, h->shard->comm, send, recv, bytes, h->s_main.get());
}

// Peer-memory exchange set-up (sharded mode, collective): allocate this rank's buffer in `sh`, exchange its IPC handle
// over sh's communicator, map every peer's buffer, and describe the result in *out.  Falls back to the NCCL all-gather path (px.enabled = 0)
// when FI_EPP_EXCHANGE=nccl, when there are more than FI_MAX_RANKS ranks, or when any rank cannot map a peer.
struct XchgBlob {
  cudaIpcMemHandle_t handle;
  uint64_t ptr;
  int64_t pid;
  int32_t device;
  int32_t ok;
  uint8_t pad[40];
};
static_assert(sizeof(XchgBlob) == 128, "XchgBlob size");

int setup_peer_exchange(fi_epp* h, ShardState& sh, uint32_t rank, uint32_t world, PeerXchg* out) {
  const char* mode = std::getenv("FI_EPP_EXCHANGE");
  const bool want = !(mode && std::strcmp(mode, "nccl") == 0) && world <= (uint32_t)FI_MAX_RANKS;
  const uint64_t R = h->cfg.max_batch;
  auto up = [](uint64_t v) { return (v + 255) & ~255ull; };
  PeerXchg px{};
  px.world = world;
  px.rank = rank;
  uint64_t off = 0;
  for (int par = 0; par < 2; ++par) {  // tagged 64-bit words (kernels.cuh PeerXchg)
    px.off_pick[par] = off;
    off = up(off + (uint64_t)world * R * h->P * 4 * sizeof(uint64_t));
  }
  XchgBlob mine{};
  mine.ok = 0;
  if (want && cuda_alloc(sh.d_xchg, off) == cudaSuccess && cudaMemset(sh.d_xchg.get(), 0, off) == cudaSuccess &&
      cuda_alloc(sh.h_xerr, 1, cudaHostAllocMapped) == cudaSuccess &&
      cudaIpcGetMemHandle(&mine.handle, sh.d_xchg.get()) == cudaSuccess) {
    mine.ok = 1;
  }
  cudaGetLastError();
  mine.ptr = (uint64_t)(uintptr_t)sh.d_xchg.get();
  mine.pid = (int64_t)getpid();
  mine.device = h->cfg.device;
  // round 1: handles; round 2: "I mapped every peer" votes.  Both ride the NCCL communicator.
  DevPtr<XchgBlob> blobs;
  FI_CUDA(cuda_alloc(blobs, world + 1));
  XchgBlob* d_blobs = blobs.get();
  std::vector<XchgBlob> all(world);
  auto gather = [&]() -> int {
    FI_CUDA(cudaMemcpyAsync(d_blobs + world, &mine, sizeof(mine), cudaMemcpyHostToDevice, h->s_main.get()));
    int rc = nccl_allgather_on(h, sh.comm, d_blobs + world, d_blobs, sizeof(XchgBlob), h->s_main.get());
    if (rc != FI_OK) return rc;
    FI_CUDA(cudaMemcpyAsync(all.data(), d_blobs, (size_t)world * sizeof(XchgBlob), cudaMemcpyDeviceToHost, h->s_main.get()));
    FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    return FI_OK;
  };
  int rc = gather();
  if (rc != FI_OK) return rc;
  bool ok = true;
  for (uint32_t k = 0; k < world; ++k) ok = ok && all[k].ok;
  if (ok) {
    for (uint32_t k = 0; k < world && ok; ++k) {
      if (k == rank) {
        px.base[k] = sh.d_xchg.get();
      } else if (all[k].pid == mine.pid) {  // same process: plain peer access
        int can = 0;
        if (all[k].device != h->cfg.device) {
          cudaDeviceCanAccessPeer(&can, h->cfg.device, all[k].device);
          if (can) {
            cudaError_t e = cudaDeviceEnablePeerAccess(all[k].device, 0);
            can = (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled);
            cudaGetLastError();
          }
        } else {
          can = 1;
        }
        ok = can != 0;
        px.base[k] = (uint8_t*)(uintptr_t)all[k].ptr;
      } else {
        void* m = nullptr;
        if (cudaIpcOpenMemHandle(&m, all[k].handle, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess) {
          sh.peer_ipc[k] = m;
          px.base[k] = (uint8_t*)m;
        } else {
          cudaGetLastError();
          ok = false;
        }
      }
    }
  }
  mine.ok = ok ? 1 : 0;
  rc = gather();
  if (rc != FI_OK) return rc;
  for (uint32_t k = 0; k < world; ++k) ok = ok && all[k].ok;
  if (ok) {
    px.enabled = 1;
    px.step = 0;
    *sh.h_xerr = 0;
    px.err = const_cast<uint32_t*>(sh.h_xerr.get());  // unified addressing: the host pointer is the device pointer
  }
  *out = px;
  if (std::getenv("FI_EPP_VERBOSE"))
    std::fprintf(stderr, "[fi_epp] rank %u/%u: sharded exchange over %s\n", rank, world,
                 px.enabled ? "peer memory (in-kernel tagged stores)" : "NCCL all-gather");
  return FI_OK;
}

// FI_EPP_TRACE=<call index>: print that call's kernel timeline (start/end relative to the call's start)
void dump_trace(fi_epp* h, uint32_t R) {
  if (!h->tracing) return;
  static const char* names[] = {"hash_chain", "match_pick", "index", "other"};
  cudaStreamSynchronize(h->s_main.get());
  std::fprintf(stderr, "[fi_epp trace] rank %u call %ld: R=%u\n", h->rank, h->trace_call, R);
  for (auto& e : h->pending_ev) {
    float t0 = 0.f, t1 = 0.f;
    cudaEventSynchronize(e.b.get());
    cudaEventElapsedTime(&t0, h->ev_trace0.get(), e.a.get());
    cudaEventElapsedTime(&t1, h->ev_trace0.get(), e.b.get());
    std::fprintf(stderr, "[fi_epp trace]   r%u %-15s start %8.1f us  end %8.1f us  (%6.1f us)\n", h->rank, names[e.kind],
                 t0 * 1e3, t1 * 1e3, (t1 - t0) * 1e3);
    h->ev_pool.push_back(std::move(e.a));
    h->ev_pool.push_back(std::move(e.b));
  }
  h->pending_ev.clear();
  h->tracing = false;
}

// One pick call of any variant: the single pick (k == 0), the ranked pick (k > 0, docs/SPEC.md S.6a) and the subset
// pick (subsets, S.5a), each with or without LoRA adapters.  Host or device pointers, by entry point.
struct PickCall {
  const uint8_t* prompts;
  const uint64_t* offsets;   // [R + 1]
  const uint64_t* h0;        // [R]
  const uint64_t* adapters;  // [R] adapter ids, or null
  const uint32_t* subsets;   // [R][ceil(E/32)] candidate bitsets, or null
  uint32_t R;
  uint32_t k;                // 0: out is [R][P]; else [R][P][k]
  fi_pick* out;
  uint64_t* chains_out;      // [R][max_blocks], or null
  // match counts (S.3a) instead of picks: out is null, counts [R][endpoint_count]; nblocks_out [R] or null
  uint16_t* counts;
  uint32_t* nblocks_out;
};

// the same from the untyped pointers the device entry points take
PickCall device_call(const void* p, const void* o, const void* h0, const void* a, const void* s, uint32_t R, uint32_t k,
                     void* out, void* ch) {
  return {(const uint8_t*)p, (const uint64_t*)o, (const uint64_t*)h0, (const uint64_t*)a, (const uint32_t*)s, R, k,
          (fi_pick*)out, (uint64_t*)ch};
}

// chains_out[R][max_blocks] = the chains at `chain` (pitch MP), on stream s; nothing if chains_out is null
int copy_chains_out(fi_epp* h, const uint64_t* chain, uint64_t* chains_out, uint32_t R, cudaMemcpyKind kind, cudaStream_t s) {
  if (!chains_out) return FI_OK;
  const size_t row = (size_t)h->cfg.max_blocks * sizeof(uint64_t);
  FI_CUDA(cudaMemcpy2DAsync(chains_out, row, chain, (size_t)h->MP * sizeof(uint64_t), row, R, kind, s));
  if (kind == cudaMemcpyDeviceToHost) h->stats.d2h_bytes += row * R;
  return FI_OK;
}

// Stage B's prelude, the same for the stream-ordered pick and the pipelined submit: s_main waits for every index update
// submitted so far, the endpoint and adapter tables go up if they changed, and `mp` describes the match of call `c`
// (device pointers) over the chains at chain / nb.  Sharded: the rank's picks go to d_local, and the merge applies P/D.
int prepare_match(fi_epp* h, const PickCall& c, const uint64_t* chain, const uint32_t* nb, MatchParams& mp) {
  FI_CUDA(cudaStreamWaitEvent(h->s_main.get(), h->ev_index.get(), 0));  // every submitted op is visible
  if (h->eps_dirty) {
    FI_CUDA(cudaMemcpyAsync(h->d_eps.get(), h->eps.data(), h->eps.size() * sizeof(EndpointDev), cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += h->eps.size() * sizeof(EndpointDev);
    LaunchScope ls(h, h->s_main.get(), K_OTHER);
    FI_CUDA(launch_prepare_endpoints(h->d_eps.get(), h->cfg.num_endpoints, h->cfg.endpoint_begin, h->cfg.endpoint_count, h->st,
                                     h->d_sc.get(), h->d_elig.get(), h->d_zero.get(), h->d_ztie.get(), h->s_main.get()));
    h->eps_dirty = false;  // (eps is pageable host memory: the copy has been staged by the time it returns)
  }
  if (h->lora_dirty) {
    FI_CUDA(cudaMemcpyAsync(h->d_lora.get(), h->lora.data(), h->lora.size() * sizeof(LoraDev), cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += h->lora.size() * sizeof(LoraDev);
    h->lora_dirty = false;
  }
  const bool sharded = h->world > 1;
  mp = MatchParams{};
  mp.chain = chain;
  mp.nblocks = nb;
  mp.offsets = c.offsets;
  mp.adapters = c.adapters;
  mp.R = c.R;
  mp.MP = h->MP;
  mp.max_blocks = h->cfg.max_blocks;
  mp.ix = h->ix.v;
  mp.st = h->st;
  mp.ep_begin = h->cfg.endpoint_begin;
  mp.ep_count = h->cfg.endpoint_count;
  mp.E_global = h->cfg.num_endpoints;
  mp.h0 = c.h0;
  mp.lpm = h->cfg.match_mode;
  mp.apply_pd = (h->cfg.pd_enabled && !sharded) ? 1 : 0;
  mp.pd_decode = h->cfg.pd_decode_profile;
  mp.pd_prefill = h->cfg.pd_prefill_profile;
  mp.pd_threshold = h->cfg.pd_threshold;
  mp.out = sharded ? h->shard->d_local.get() : c.out;
  mp.probed_blocks = h->profiling ? h->d_probed.get() : nullptr;
  mp.work_counter = h->d_work.get();
  mp.k = c.k;
  mp.counts = c.counts;
  if (c.subsets) {
    mp.subsets = c.subsets;
    mp.sub_pitch = (h->cfg.num_endpoints + 31) / 32;
    mp.eps = h->d_eps.get();
  }
  return FI_OK;
}

// Pipeline slot 0's chain buffer, d_chain / d_nblocks (slot 1, d_chain2 / d_nblocks2, serves odd-numbered submits only).
//   Writers: the stream-ordered pick (run_pick_impl) and fi_epp_hash_batch, on s_main;
//            stage A of an even-numbered pipelined submit (submit_pick), on s_a.
//   Readers: the match and chain copy-out of the pick or submit that wrote it, on s_main (ev_plain, ev_b[0]);
//            fi_epp_index_add_chains_device(.., NULL, ..), a device-LRU Add on s_index (ev_lru);
//            fi_epp_index_add_submitted's copy of a submitted batch's chains, on s_copy (ev_slot_read[0]).
// A stream-ordered writer calls claim_chain_slot0 before it writes: its stream waits for the last submit's stage A and
// for the readers on other streams (wait_slot_readers), and no submitted batch's chains can be taken any more.  Stage A
// of a submit waits for the same readers of its own slot, for the match of the batch two back and the last
// stream-ordered pick (submit_pick).
int wait_slot_readers(fi_epp* h, uint32_t slot, cudaStream_t s) {
  if (h->dlru) FI_CUDA(cudaStreamWaitEvent(s, h->dlru->ev.get(), 0));
  if (h->padd_seq) FI_CUDA(cudaStreamWaitEvent(s, h->ev_slot_read[slot].get(), 0));
  return FI_OK;
}

int claim_chain_slot0(fi_epp* h, cudaStream_t s) {
  if (h->pipe_seq) FI_CUDA(cudaStreamWaitEvent(s, h->ev_a[(h->pipe_seq - 1) & 1].get(), 0));
  const int rc = wait_slot_readers(h, 0, s);
  if (rc == FI_OK) h->slot_ticket[0] = h->slot_ticket[1] = ~0ull;
  return rc;
}

// the whole pick of call `c` on device buffers (out: single rank only for k > 0); feed: the same call on host buffers,
// whose prompts are still to be copied to c.prompts (in slices when it can), or null
int run_pick_impl(fi_epp* h, const PickCall& c, const PickCall* feed) {
  const uint32_t R = c.R;
  const bool sharded = h->world > 1;
  if (sharded && (h->n_sets || h->n_clears))
    return fail(h, FI_ERR_STATE, "sharded pool: index updates are collective (fi_epp_index_apply / fi_epp_index_add_chains)");
  int rc = settle_updates(h);
  if (rc != FI_OK) return rc;
  h->tracing = !h->profiling && h->trace_call >= 0 && (long)h->stats.pick_calls == h->trace_call;
  if (h->tracing) {
    if (!h->ev_trace0) cuda_create(h->ev_trace0, cudaEventDefault);
    FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    FI_CUDA(cudaEventRecord(h->ev_trace0.get(), h->s_main.get()));
  }
  MatchParams mp;
  rc = prepare_match(h, c, h->d_chain.get(), h->d_nblocks.get(), mp);
  if (rc != FI_OK) return rc;
  rc = claim_chain_slot0(h, h->s_main.get());
  if (rc != FI_OK) return rc;
  // (s_main already waits for ev_index: the hashing reads the same index view as the match)
  const IndexView* early = early_exit_hashing(h, c.chains_out || (feed && feed->chains_out)) ? &mp.ix : nullptr;

  const uint32_t S = h->feed_slices;
  if (feed && !sharded && h->fast_hash && S > 1 && R >= 64 * S && feed->offsets[R] >= (8ull << 20)) {
    // Sliced feed.  (On DEVICE-resident inputs slicing the step is slower — DESIGN.md "What did not
    // work" — but here the copy engine is the bottleneck and the kernels of slice k hide under copy k+1.)
    uint8_t* dp = const_cast<uint8_t*>(c.prompts);
    const uint32_t per = (((R + S - 1) / S) + 31) & ~31u;
    uint32_t used = 0;
    for (uint32_t k = 0; k * per < R; ++k, ++used) {
      const uint32_t r0 = k * per, r1 = std::min(R, r0 + per);
      const uint64_t b0 = feed->offsets[r0], b1 = feed->offsets[r1];
      if (b1 > b0) FI_CUDA(cudaMemcpyAsync(dp + b0, feed->prompts + b0, b1 - b0, cudaMemcpyHostToDevice, h->s_copy.get()));
      FI_CUDA(cudaEventRecord(h->ev_copy[k].get(), h->s_copy.get()));
    }
    h->stats.h2d_bytes += feed->offsets[R];
    for (uint32_t k = 0; k < used; ++k) {
      const uint32_t r0 = k * per, Rk = std::min(per, R - r0);
      FI_CUDA(cudaStreamWaitEvent(h->s_main.get(), h->ev_copy[k].get(), 0));
      rc = run_hash(h, c.prompts, c.offsets, c.h0, r0, Rk, h->s_main.get(), early);
      if (rc != FI_OK) return rc;
      MatchParams ms = mp;
      ms.chain = mp.chain + (size_t)r0 * h->MP;
      ms.nblocks = mp.nblocks + r0;
      ms.offsets = mp.offsets ? mp.offsets + r0 : nullptr;
      ms.adapters = mp.adapters ? mp.adapters + r0 : nullptr;
      ms.subsets = mp.subsets ? mp.subsets + (size_t)r0 * mp.sub_pitch : nullptr;
      ms.h0 = mp.h0 + r0;
      ms.r_base = r0;
      ms.R = Rk;
      ms.out = mp.out ? mp.out + (size_t)r0 * h->P * std::max(c.k, 1u) : nullptr;
      ms.counts = mp.counts ? mp.counts + (size_t)r0 * h->cfg.endpoint_count : nullptr;
      ms.work_counter = h->d_work.get() + k;
      LaunchScope ls(h, h->s_main.get(), K_MATCH);
      FI_CUDA(launch_match_pick(ms, h->sm_count, h->s_main.get()));
    }
    return FI_OK;
  }
  if (feed && feed->offsets[R]) {  // one copy, then the whole batch
    FI_CUDA(cudaMemcpyAsync(const_cast<uint8_t*>(c.prompts), feed->prompts, feed->offsets[R], cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += feed->offsets[R];
  }
  if (!sharded) {
    // (A sub-batch pipeline over several streams was tried and measured slower on device-resident
    // inputs — DESIGN.md "What did not work": the chain walk costs a flat serial latency at any batch
    // size and small slices pay launch/ramp overheads.)
    rc = run_hash(h, c.prompts, c.offsets, c.h0, 0, R, h->s_main.get(), early);
    if (rc != FI_OK) return rc;
    LaunchScope ls(h, h->s_main.get(), K_MATCH);
    FI_CUDA(launch_match_pick(mp, h->sm_count, h->s_main.get()));
    return FI_OK;
  }

  // ---- endpoint-range sharded pool --------------------------------------------------------------
  // Hashing: every rank needs every request's chain.  split: rank g hashes requests [g·per, (g+1)·per) and
  // the chain rows + block counts are all-gathered in place (2 KiB per request over NVLink instead of
  // re-reading 16 KiB of prompt on every rank); replicated: every rank hashes everything.
  if (h->split_hash && h->fast_hash && R >= 32 * h->world) {
    const uint32_t per = (((R + h->world - 1) / h->world) + 31) & ~31u;  // ≤ chain_rows / world
    const uint32_t r0 = std::min(R, h->rank * per), r1 = std::min(R, r0 + per);
    if (r1 > r0) {
      rc = run_hash(h, c.prompts, c.offsets, c.h0, r0, r1 - r0, h->s_main.get(), nullptr);
      if (rc != FI_OK) return rc;
    }
    rc = nccl_allgather(h, h->d_chain.get() + (size_t)h->rank * per * h->MP, h->d_chain.get(), (size_t)per * h->MP * sizeof(uint64_t));
    if (rc != FI_OK) return rc;
    rc = nccl_allgather(h, h->d_nblocks.get() + (size_t)h->rank * per, h->d_nblocks.get(), (size_t)per * sizeof(uint32_t));
    if (rc != FI_OK) return rc;
    h->stats.n_other += 2;  // two collectives of the step (not kernels of this library)
  } else {
    rc = run_hash(h, c.prompts, c.offsets, c.h0, 0, R, h->s_main.get(), nullptr);
    if (rc != FI_OK) return rc;
  }
  const bool p2p = h->px.enabled != 0;
  if (p2p) {
    // Peer-memory exchange: match_pick stores this rank's picks as tagged words into every rank's buffer and
    // merge_picks polls per request, so the reduction has no collective call, no barrier between the ranks
    // and no host round trip.  A timeout is reported once (the kernels set the mapped host word).
    if (*h->shard->h_xerr) {
      *h->shard->h_xerr = 0;
      return fail(h, FI_ERR_COMM, "peer exchange timed out waiting for another rank");
    }
    h->px.step += 1;
    if (h->px.step == 0) h->px.step = 1;  // tag 0 is the zero-initialised buffer
    mp.px = h->px;
  }
  {
    LaunchScope ls(h, h->s_main.get(), K_MATCH);
    FI_CUDA(launch_match_pick(mp, h->sm_count, h->s_main.get()));
  }
  MergeParams mg{};
  if (p2p) {
    mg.gathered = reinterpret_cast<const fi_pick*>(h->shard->d_xchg.get() + h->px.off_pick[h->px.step & 1u]);
    mg.px = h->px;
  } else {
    rc = nccl_allgather(h, h->shard->d_local.get(), h->shard->d_gather.get(), (size_t)R * h->P * sizeof(fi_pick));
    if (rc != FI_OK) return rc;
    mg.gathered = h->shard->d_gather.get();
  }
  mg.ranks = h->world;
  mg.R = R;
  mg.P = h->P;
  mg.nblocks = h->d_nblocks.get();
  mg.offsets = c.offsets;
  mg.chain = h->d_chain.get();
  mg.h0 = c.h0;
  mg.MP = h->MP;
  mg.E_global = h->cfg.num_endpoints;
  mg.apply_pd = h->cfg.pd_enabled;
  mg.pd_decode = h->cfg.pd_decode_profile;
  mg.pd_prefill = h->cfg.pd_prefill_profile;
  mg.pd_threshold = h->cfg.pd_threshold;
  mg.out = c.out;
  {
    LaunchScope ls(h, h->s_main.get(), K_OTHER);
    FI_CUDA(launch_merge_picks(mg, h->s_main.get()));
  }
  return FI_OK;
}

int run_pick(fi_epp* h, const PickCall& c, const PickCall* feed) {
  int rc = run_pick_impl(h, c, feed);
  if (rc != FI_OK) return rc;
  dump_trace(h, c.R);
  h->stats.pick_calls++;
  h->stats.requests += c.R;
  FI_CUDA(cudaEventRecord(h->ev_pick.get(), h->s_main.get()));  // index updates submitted later wait for this pick
  FI_CUDA(cudaEventRecord(h->ev_plain.get(), h->s_main.get()));
  h->last_plain_R = c.R;
  return FI_OK;
}

// the next ticket: recorded on s_main behind everything queued there so far (the batch just enqueued)
int issue_ticket(fi_epp* h, uint64_t* t) {
  FI_CUDA(cudaEventRecord(h->ev_ticket[h->tickets % fi_epp::kTicketRing].get(), h->s_main.get()));
  *t = h->tickets++;
  return FI_OK;
}

// Pipelined device path: enqueue one batch, call `c` on device buffers.  Stage A on s_a, stage B on s_main (see
// fi_epp::s_a).  lagged: the index counters may lag (check_counters_lagged, fi_epp_pick_submit_ex).
int submit_pick(fi_epp* h, const PickCall& c, cudaStream_t us, uint64_t* ticket, bool lagged) {
  const uint32_t R = c.R;
  int rc = settle_updates(h, lagged);
  if (rc != FI_OK) return rc;
  if (!h->d_chain2) {  // slot 1's buffers, both or neither
    DevPtr<uint64_t> chain;
    DevPtr<uint32_t> nb;
    FI_CUDA(cuda_alloc(chain, (size_t)h->cfg.max_batch * h->MP));
    FI_CUDA(cuda_alloc(nb, h->cfg.max_batch));
    h->d_chain2 = std::move(chain);
    h->d_nblocks2 = std::move(nb);
  }
  // FI_EPP_TRACE=<call>: timeline of three consecutive pipelined batches (printed by fi_epp_pick_wait)
  if (!h->profiling && h->trace_call >= 0 && (long)h->stats.pick_calls >= h->trace_call &&
      (long)h->stats.pick_calls < h->trace_call + 3) {
    if ((long)h->stats.pick_calls == h->trace_call) {
      if (!h->ev_trace0) cuda_create(h->ev_trace0, cudaEventDefault);
      FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
      FI_CUDA(cudaStreamSynchronize(h->s_a.get()));
      FI_CUDA(cudaEventRecord(h->ev_trace0.get(), h->s_main.get()));
      FI_CUDA(cudaStreamWaitEvent(h->s_a.get(), h->ev_trace0.get(), 0));
    }
    h->tracing = true;
  } else if (h->tracing && (long)h->stats.pick_calls >= h->trace_call + 3) {
    h->tracing = false;  // events stay queued until the dump
  }
  const uint32_t slot = (uint32_t)(h->pipe_seq & 1);
  uint64_t* chain = slot ? h->d_chain2.get() : h->d_chain.get();
  uint32_t* nb = slot ? h->d_nblocks2.get() : h->d_nblocks.get();
  // ---- stage A: inputs are ready in the caller's stream order; the slot's buffers are free once the
  // match of two batches ago is done; slot 0's d_chain / d_nblocks are free once the previous plain pick
  // (if any) is done; and the readers on other streams (claim_chain_slot0)
  FI_CUDA(cudaEventRecord(h->ev_in.get(), us));
  FI_CUDA(cudaStreamWaitEvent(h->s_a.get(), h->ev_in.get(), 0));
  if (h->pipe_seq >= 2) FI_CUDA(cudaStreamWaitEvent(h->s_a.get(), h->ev_b[slot].get(), 0));
  FI_CUDA(cudaStreamWaitEvent(h->s_a.get(), h->ev_plain.get(), 0));
  rc = wait_slot_readers(h, slot, h->s_a.get());
  if (rc != FI_OK) return rc;
  // stage B's parameters first: stage A's early exit reads the same index view (one per call: a rebuild swaps tables)
  MatchParams mp;
  rc = prepare_match(h, c, chain, nb, mp);
  if (rc != FI_OK) return rc;
  const bool early = early_exit_hashing(h, c.chains_out != nullptr);
  // Early exit reads the index in stage A: every op submitted before this batch is applied first, as for its match.
  // Updates submitted after it wait for ev_pick, which follows this batch's match and so its stage A.
  if (early) FI_CUDA(cudaStreamWaitEvent(h->s_a.get(), h->ev_index.get(), 0));
  {
    // Block hashing and chain walk in one kernel (hash_kernels.cu hash_chain).  It does not wait for the previous
    // batch's match_pick: a full batch runs half-SM CTAs, and one starts on an SM as soon as two of match's three
    // CTAs there have run out of queue (DESIGN.md §4.0; giving match fewer CTAs per SM so that the two kernels share
    // every SM for the whole step was measured slower: §7).
    LaunchScope ls(h, h->s_a.get(), K_HASH);
    FI_CUDA(launch_hash_chain(c.prompts, c.offsets, c.h0, R, h->cfg.block_bytes, h->cfg.max_blocks, h->MP, chain, nb,
                              h->sm_count, h->s_a.get(), early ? &mp.ix : nullptr, hashed_counter(h)));
  }
  FI_CUDA(cudaEventRecord(h->ev_a[slot].get(), h->s_a.get()));
  // ---- stage B
  FI_CUDA(cudaStreamWaitEvent(h->s_main.get(), h->ev_a[slot].get(), 0));
  mp.work_counter = h->d_work.get() + 8 + slot;
  {
    LaunchScope ls(h, h->s_main.get(), K_MATCH);
    FI_CUDA(launch_match_pick(mp, h->sm_count, h->s_main.get()));
  }
  rc = copy_chains_out(h, chain, c.chains_out, R, cudaMemcpyDeviceToDevice, h->s_main.get());
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaEventRecord(h->ev_b[slot].get(), h->s_main.get()));
  FI_CUDA(cudaEventRecord(h->ev_pick.get(), h->s_main.get()));
  rc = issue_ticket(h, ticket);
  if (rc != FI_OK) return rc;
  h->slot_ticket[slot] = *ticket;
  h->slot_R[slot] = R;
  h->pipe_seq++;
  h->stats.pick_calls++;
  h->stats.requests += R;
  return FI_OK;
}

// Upstream indexer.RemovePod for the distinct local endpoints `local` (fi_epp_index_remove_endpoints, and the endpoints
// a shrink of fi_epp_resize_pool drops): one sweep over the index rows clears their bits whatever put them there (LRU
// Adds or direct SETs), keys nobody holds any more are retired (tombstones, like a CLEAR), and the endpoints' LRUs
// start empty.  pairs_removed != null: wait for the sweep and write how many pairs left the index.
int remove_local_endpoints(fi_epp* h, const std::vector<uint32_t>& local, uint64_t* pairs_removed) {
  RemoveSet rs{};
  for (uint32_t e : local) rs.row[e >> 5] |= 1u << (e & 31);
  for (uint32_t w = 0; w < h->W; ++w)
    if (rs.row[w]) {
      rs.word[rs.m] = w;
      rs.bits[rs.m] = rs.row[w];
      ++rs.m;
    }
  if (!h->d_rm) FI_CUDA(cuda_alloc(h->d_rm, 1 + ((size_t)h->cfg.endpoint_count + 1) / 2));
  uint32_t* d_eps = reinterpret_cast<uint32_t*>(h->d_rm.get() + 1);
  int rc = update_begin(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaMemsetAsync(h->d_rm.get(), 0, sizeof(unsigned long long), h->s_index.get()));
  {
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_index_remove_sweep(h->ix.v, h->d_ctr.get(), rs, remove_whole_rows(rs, h->W), h->rank, h->d_rm.get(), h->sm_count, h->s_index.get()));
  }
  if (h->lru_mode == 1 && h->dlru) {
    // (pageable source: the copy has taken the data when cudaMemcpyAsync returns)
    FI_CUDA(cudaMemcpyAsync(d_eps, local.data(), local.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->s_index.get()));
    h->stats.h2d_bytes += local.size() * sizeof(uint32_t);
    LaunchScope ls(h, h->s_index.get(), K_INDEX);
    FI_CUDA(launch_lru_reset(h->dlru->v, d_eps, (uint32_t)local.size(), h->s_index.get()));
  }
  for (uint32_t e : local)
    if (e < h->lrus.size()) h->lrus[e].clear();
  rc = update_end(h);  // (the reset changes no LRU status)
  if (rc != FI_OK) return rc;
  if (pairs_removed) {
    unsigned long long c = 0;
    FI_CUDA(cudaMemcpyAsync(&c, h->d_rm.get(), sizeof(c), cudaMemcpyDeviceToHost, h->s_index.get()));
    FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
    *pairs_removed = c;
  }
  return FI_OK;
}

int validate_config(const fi_epp_config& c, std::string* err) {
  auto bad = [&](const char* m) {
    *err = m;
    return FI_ERR_INVALID;
  };
  if (c.struct_size != sizeof(fi_epp_config)) return bad("struct_size mismatch");
  if (c.abi_version != FI_EPP_ABI_VERSION) return bad("abi_version mismatch");
  if (c.block_bytes == 0 || c.block_bytes > (1u << 20)) return bad("block_bytes out of range");
  if (c.max_blocks == 0 || c.max_blocks > FI_EPP_MAX_BLOCKS) return bad("max_blocks out of range");
  if (c.num_endpoints == 0) return bad("num_endpoints == 0");
  if (c.endpoint_count == 0 || (uint64_t)c.endpoint_begin + c.endpoint_count > c.num_endpoints)
    return bad("endpoint shard out of range");
  if (c.endpoint_count > 4096) return bad("more than 4096 local endpoints: shard the pool by endpoint range");
  if (c.match_mode != FI_MATCH_UPSTREAM && c.match_mode != FI_MATCH_LPM) return bad("bad match_mode");
  if (c.max_batch == 0) return bad("max_batch == 0");
  if (c.n_profiles == 0 || c.n_profiles > FI_EPP_MAX_PROFILES) return bad("n_profiles out of range");
  for (uint32_t p = 0; p < c.n_profiles; ++p) {
    if (c.profiles[p].n_scorers > FI_EPP_MAX_SCORERS) return bad("n_scorers out of range");
    if (c.profiles[p].n_more_filters > FI_EPP_MAX_FILTERS - 1) return bad("n_more_filters out of range");
    for (uint32_t f = 0; f < c.profiles[p].n_more_filters; ++f)
      if (c.profiles[p].more_filters[f] == 0) return bad("a by-label filter without label bits admits nothing");
    for (uint32_t s = 0; s < c.profiles[p].n_scorers; ++s) {
      const uint32_t k = c.profiles[p].scorers[s].kind;
      if (k != FI_SCORER_PREFIX && k != FI_SCORER_KV_UTIL && k != FI_SCORER_QUEUE && k != FI_SCORER_LORA)
        return bad("unknown scorer kind");
      if (c.profiles[p].scorers[s].weight < 0) return bad("scorer weights must be >= 0");
    }
  }
  if (c.pd_enabled) {
    if (c.pd_decode_profile >= c.n_profiles || c.pd_prefill_profile >= c.n_profiles) return bad("pd profile index out of range");
    if (!(c.pd_threshold == c.pd_threshold)) return bad("pd_threshold is NaN");
  }
  if (c.index_slots) {
    if (c.index_slots < 64 || (c.index_slots & (c.index_slots - 1))) return bad("index_slots must be a power of two >= 64");
    if (c.index_slots > 0xFFFFFF00ull) return bad("index_slots too large");
  }
  return FI_OK;
}

}  // namespace

// =============================================================================
// C ABI
// =============================================================================
extern "C" {

uint32_t fi_epp_abi_version(void) { return FI_EPP_ABI_VERSION; }

const char* fi_epp_status_string(int s) {
  switch (s) {
    case FI_OK: return "ok";
    case FI_ERR_INVALID: return "invalid argument";
    case FI_ERR_CUDA: return "CUDA error (no CPU fallback exists)";
    case FI_ERR_NOMEM: return "out of memory";
    case FI_ERR_CAPACITY: return "capacity exceeded";
    case FI_ERR_STATE: return "invalid state";
    case FI_ERR_COMM: return "communicator error";
    case FI_ERR_CONFIG: return "EndpointPickerConfig rejected";
    default: return "unknown status";
  }
}

int fi_epp_config_default(fi_epp_config* c) {
  if (!c) return FI_ERR_INVALID;
  std::memset(c, 0, sizeof(*c));
  c->struct_size = sizeof(*c);
  c->abi_version = FI_EPP_ABI_VERSION;
  c->device = 0;
  c->block_bytes = 64;     // 16 uint32 tokens (SURVEY.md §8d); the reference YAML overrides it (strategy.go:57)
  c->max_blocks = 256;     // strategy.go:58
  c->lru_capacity = 31250; // strategy.go:59
  c->num_endpoints = 1;
  c->endpoint_begin = 0;
  c->endpoint_count = 1;
  c->match_mode = FI_MATCH_UPSTREAM;
  c->max_batch = 1024;
  c->max_prompt_bytes = 0;  // 0 = max_batch * block_bytes * max_blocks
  c->index_slots = 0;
  c->n_profiles = 1;  // generatePrefixCacheConfig: profile "default" = picker + prefix scorer weight 100
  std::snprintf(c->profiles[0].name, sizeof(c->profiles[0].name), "default");
  c->profiles[0].n_scorers = 1;
  c->profiles[0].scorers[0].kind = FI_SCORER_PREFIX;
  c->profiles[0].scorers[0].weight = 100;  // strategy.go:66
  return FI_OK;
}

int fi_epp_model_seed(const void* model, size_t model_len, const void* salt, size_t salt_len, uint64_t* h0) {
  if (!h0 || (!model && model_len) || (!salt && salt_len)) return FI_ERR_INVALID;
  if (model_len + salt_len > 0x7FFFFFFFull) return FI_ERR_INVALID;
  std::vector<uint8_t> buf(model_len + salt_len);
  if (model_len) std::memcpy(buf.data(), model, model_len);
  if (salt_len) std::memcpy(buf.data() + model_len, salt, salt_len);
  *h0 = xxh64_bytes(buf.data(), (uint32_t)buf.size());
  return FI_OK;
}

void* fi_epp_pinned_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void fi_epp_pinned_free(void* p) {
  if (p) cudaFreeHost(p);
}

const char* fi_epp_last_error(const fi_epp* h) { return h ? h->err.c_str() : "null handle"; }

// Every resource of the handle has an owner among its members; the streams, declared first, go last.
void fi_epp_destroy(fi_epp* h) {
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  for (cudaStream_t s : {h->s_main.get(), h->s_index.get(), h->s_copy.get(), h->s_a.get()}) cudaStreamSynchronize(s);
  drain_profile(h);
  delete h;
}

int fi_epp_create(const fi_epp_config* cfg, fi_epp** out) {
  if (!cfg || !out) return FI_ERR_INVALID;
  *out = nullptr;
  std::unique_ptr<fi_epp> up(new fi_epp());
  fi_epp* h = up.get();
  h->cfg = *cfg;
  {
    std::string e;
    int rc = validate_config(*cfg, &e);
    if (rc != FI_OK) {
      std::fprintf(stderr, "fi_epp_create: %s\n", e.c_str());
      return rc;
    }
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::fprintf(stderr, "fi_epp_create: no CUDA device — libfi_epp has no CPU fallback\n");
    return FI_ERR_CUDA;
  }
  if (cfg->device < 0 || cfg->device >= ndev) {
    std::fprintf(stderr, "fi_epp_create: device %d out of range (%d devices)\n", cfg->device, ndev);
    return FI_ERR_INVALID;
  }
  auto die = [&](int rc) {
    std::fprintf(stderr, "fi_epp_create: %s\n", h->err.c_str());
    return rc;  // (`up` releases whatever was created)
  };
#define FI_TRY(call)                                                    \
  do {                                                                  \
    cudaError_t e__ = (call);                                           \
    if (e__ != cudaSuccess) {                                           \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e__);     \
      return die(e__ == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA); \
    }                                                                   \
  } while (0)
  FI_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  FI_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  h->sm_count = prop.multiProcessorCount;
  h->P = cfg->n_profiles;
  h->MP = (cfg->max_blocks + 7) & ~7u;  // whole groups of 8 links for the chain walker
  h->W = pool_row_words(cfg->endpoint_count);
  h->fast_hash = (cfg->block_bytes % 32) == 0;
  if (const char* e = std::getenv("FI_EPP_TRACE")) h->trace_call = std::strtol(e, nullptr, 10);
  h->verbose = std::getenv("FI_EPP_VERBOSE") != nullptr;
  if (h->cfg.max_prompt_bytes == 0)
    h->cfg.max_prompt_bytes = (uint64_t)cfg->max_batch * cfg->block_bytes * cfg->max_blocks;
  h->index_slots_given = cfg->index_slots;
  if (h->cfg.index_slots == 0) h->cfg.index_slots = pool_default_slots(cfg->num_endpoints, cfg->lru_capacity);

  for (Stream* s : {&h->s_main, &h->s_index, &h->s_copy, &h->s_a}) FI_TRY(cuda_create(*s));
  for (Event* e : {&h->ev_in, &h->ev_a[0], &h->ev_a[1], &h->ev_b[0], &h->ev_b[1], &h->ev_pick, &h->ev_plain,
                   &h->ev_slot_read[0], &h->ev_slot_read[1]})
    FI_TRY(cuda_create(*e));
  for (Event& e : h->ev_ticket) FI_TRY(cuda_create(e));
  for (Event& e : h->ev_copy) FI_TRY(cuda_create(e));
  if (const char* e = std::getenv("FI_EPP_FEED_SLICES")) {
    const long v = std::strtol(e, nullptr, 10);
    h->feed_slices = (uint32_t)std::min<long>(std::max<long>(v, 1), fi_epp::kMaxFeedSlices);
  }
  for (Event* e : {&h->ev_index, &h->ev_user, &h->ev_done, &h->ev_ctr}) FI_TRY(cuda_create(*e));
  FI_TRY(cudaEventRecord(h->ev_index.get(), h->s_index.get()));
  const uint64_t R = cfg->max_batch;
  // rows of the per-request buffers: whole groups of 32 requests (the sliced host feed and the split-hash gather
  // cut the batch on 32-request boundaries), and — for a shard of a bigger pool — room for the in-place all-gather
  // of `world` equal slices of 32-aligned length
  h->chain_rows = (uint32_t)((R + 31) / 32 * 32);
  if (cfg->endpoint_count < cfg->num_endpoints) h->chain_rows += 32 * (FI_MAX_RANKS + 1);
  if (const char* e = std::getenv("FI_EPP_SHARD_HASH")) h->split_hash = std::strcmp(e, "split") == 0;
  FI_TRY(cuda_alloc(h->d_prompts, h->cfg.max_prompt_bytes + 64));
  FI_TRY(cuda_alloc(h->d_offsets, R + 1));
  FI_TRY(cuda_alloc(h->d_h0, R));
  FI_TRY(cuda_alloc(h->d_chain, (size_t)h->chain_rows * h->MP));
  FI_TRY(cuda_alloc(h->d_nblocks, h->chain_rows));
  FI_TRY(cuda_alloc(h->d_picks, R * h->P));
  FI_TRY(cuda_alloc(h->d_probed, 8));
  FI_TRY(cudaMemset(h->d_probed.get(), 0, 8 * sizeof(unsigned long long)));
  FI_TRY(cuda_alloc(h->d_work, 16));
  FI_TRY(cudaMemset(h->d_work.get(), 0, 16 * sizeof(uint32_t)));
  FI_TRY(cuda_alloc(h->h_picks, R * h->P));
  FI_TRY(cuda_alloc(h->h_offsets, R + 1));
  FI_TRY(cuda_alloc(h->h_h0, R));
  FI_TRY(cuda_alloc(h->h_nblocks, R));

  // index
  FI_TRY(cuda_alloc(h->d_ctr, 1));
  FI_TRY(cudaMemset(h->d_ctr.get(), 0, sizeof(IndexCounters)));
  FI_TRY(cuda_alloc(h->h_ctr, 1));
  std::memset(h->h_ctr.get(), 0, sizeof(IndexCounters));
  {
    int rc = alloc_index(h, h->cfg.index_slots, h->W, h->ix);
    if (rc != FI_OK) return die(rc);
  }
  for (int b = 0; b < 2; ++b) {
    FI_TRY(cuda_alloc(h->h_sets[b], kOpChunk));
    FI_TRY(cuda_alloc(h->h_clears[b], kOpChunk));
    FI_TRY(cuda_alloc(h->d_sets[b], kOpChunk));
    FI_TRY(cuda_alloc(h->d_clears[b], kOpChunk));
    FI_TRY(cuda_create(h->ev_buf[b]));
    FI_TRY(cudaEventRecord(h->ev_buf[b].get(), h->s_index.get()));
  }
  if (cfg->lru_capacity) {
    // virtual reservation only: an endpoint's tables become resident when it is first touched
    LruArena* arena = h->lru_arena.reserve((size_t)cfg->endpoint_count * LruSet::bytes_needed(cfg->lru_capacity)) ? &h->lru_arena : nullptr;
    h->lrus = std::vector<LruSet>(cfg->endpoint_count, LruSet(cfg->lru_capacity, arena));
    h->lru_caps.assign(cfg->endpoint_count, cfg->lru_capacity);
  }

  // endpoints + score tables
  h->eps.assign(cfg->num_endpoints, EndpointDev{0.0, 0, 0, 0, 0});
  const uint32_t Epad = h->W * 32;
  FI_TRY(cuda_alloc(h->d_eps, cfg->num_endpoints));
  FI_TRY(cuda_alloc(h->d_sc, (size_t)FI_EPP_MAX_PROFILES * FI_EPP_MAX_SCORERS * Epad));
  FI_TRY(cuda_alloc(h->d_elig, (size_t)FI_EPP_MAX_PROFILES * h->W));
  FI_TRY(cuda_alloc(h->d_zero, FI_EPP_MAX_PROFILES));
  FI_TRY(cuda_alloc(h->d_ztie, (size_t)FI_EPP_MAX_PROFILES * h->W));
  FI_TRY(cudaMemset(h->d_ztie.get(), 0, (size_t)FI_EPP_MAX_PROFILES * h->W * sizeof(uint32_t)));
  FI_TRY(cudaMemset(h->d_sc.get(), 0, (size_t)FI_EPP_MAX_PROFILES * FI_EPP_MAX_SCORERS * Epad * sizeof(double)));
  FI_TRY(cudaMemset(h->d_elig.get(), 0, (size_t)FI_EPP_MAX_PROFILES * h->W * sizeof(uint32_t)));
  h->st.n_profiles = h->P;
  h->st.Epad = Epad;
  h->st.sc = h->d_sc.get();
  h->st.elig = h->d_elig.get();
  h->st.zero = h->d_zero.get();
  h->st.ztie = h->d_ztie.get();
  h->lora.assign(Epad, LoraDev{});
  FI_TRY(cuda_alloc(h->d_lora, Epad));
  FI_TRY(cudaMemset(h->d_lora.get(), 0, (size_t)Epad * sizeof(LoraDev)));
  FI_TRY(cuda_alloc(h->d_adapters, R));
  FI_TRY(cuda_alloc(h->h_adapters, R));
  h->st.lora = h->d_lora.get();
  h->st.has_lora = 0;
  for (uint32_t p = 0; p < h->P; ++p)
    for (uint32_t s = 0; s < cfg->profiles[p].n_scorers; ++s)
      if (cfg->profiles[p].scorers[s].kind == FI_SCORER_LORA) h->st.has_lora = 1;
  for (uint32_t p = 0; p < h->P; ++p) {
    ProfileDev& d = h->st.prof[p];
    d.n_scorers = cfg->profiles[p].n_scorers;
    d.n_filters = 0;
    if (cfg->profiles[p].role_mask) d.filter[d.n_filters++] = cfg->profiles[p].role_mask;
    for (uint32_t f = 0; f < cfg->profiles[p].n_more_filters; ++f) d.filter[d.n_filters++] = cfg->profiles[p].more_filters[f];
    for (uint32_t s = 0; s < d.n_scorers; ++s) {
      d.kind[s] = cfg->profiles[p].scorers[s].kind;
      d.weight[s] = (double)cfg->profiles[p].scorers[s].weight;
    }
  }
  FI_TRY(cudaStreamSynchronize(h->s_index.get()));
  FI_TRY(cudaDeviceSynchronize());
#undef FI_TRY
  *out = up.release();
  return FI_OK;
}

int fi_epp_endpoints_update(fi_epp* h, const fi_endpoint_state* s, uint32_t n) {
  if (!h || (!s && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  for (uint32_t i = 0; i < n; ++i) {
    if (s[i].endpoint >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint index out of range");
    if (!std::isfinite(s[i].kv_util)) return fail(h, FI_ERR_INVALID, "kv_util must be finite");
  }
  for (uint32_t i = 0; i < n; ++i) {
    EndpointDev& e = h->eps[s[i].endpoint];
    e.kv_util = s[i].kv_util;
    e.queue_depth = s[i].queue_depth;
    e.role_mask = s[i].role_mask;
    e.flags = s[i].flags;
  }
  h->eps_dirty = true;
  return FI_OK;
}

int fi_epp_endpoints_lora_update(fi_epp* h, const fi_endpoint_lora* s, uint32_t n) {
  if (!h || (!s && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  for (uint32_t i = 0; i < n; ++i) {
    if (s[i].endpoint >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint index out of range");
    if (s[i].n_active > FI_EPP_MAX_LORA || s[i].n_waiting > FI_EPP_MAX_LORA)
      return fail(h, FI_ERR_INVALID, "more than FI_EPP_MAX_LORA adapters listed");
  }
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t e = s[i].endpoint - h->cfg.endpoint_begin;
    if (e >= h->cfg.endpoint_count) continue;  // another rank's shard
    LoraDev& d = h->lora[e];
    std::memset(&d, 0, sizeof(d));
    d.n_active = s[i].n_active;
    d.n_waiting = s[i].n_waiting;
    d.max_active = s[i].max_active;
    for (uint32_t k = 0; k < s[i].n_active; ++k) d.active[k] = s[i].active[k];
    for (uint32_t k = 0; k < s[i].n_waiting; ++k) d.waiting[k] = s[i].waiting[k];
  }
  h->lora_dirty = true;
  return FI_OK;
}

int fi_epp_index_apply(fi_epp* h, const fi_index_op* ops, uint64_t n) {
  if (!h || (!ops && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int err = check_counters(h);
  for (uint64_t i = 0; i < n && err == FI_OK; ++i) {
    if (ops[i].op != FI_OP_SET && ops[i].op != FI_OP_CLEAR) err = fail(h, FI_ERR_INVALID, "bad index opcode");
    else if (ops[i].endpoint >= h->cfg.num_endpoints) err = fail(h, FI_ERR_INVALID, "index op endpoint out of range");
  }
  const uint32_t lo = h->cfg.endpoint_begin, cnt = h->cfg.endpoint_count;
  // rounds of kOpChunk input ops: a round never overflows the staging buffers (or, sharded, the gossip log)
  const uint64_t rounds = (n + kOpChunk - 1) / kOpChunk;
  return run_rounds(h, rounds, err, [&](uint64_t i) -> int {
    const uint64_t i0 = i * kOpChunk, i1 = std::min(n, i0 + kOpChunk);
    for (uint64_t k = i0; k < i1; ++k) {
      const fi_index_op& op = ops[k];
      if (op.endpoint - lo >= cnt) continue;  // another rank's shard
      int rc = submit_op(h, op.hash, op.endpoint, op.op);
      if (rc != FI_OK) return rc;
    }
    return flush_ops(h);
  });
}

int fi_epp_index_remove_endpoints(fi_epp* h, const uint32_t* endpoints, uint32_t n, uint64_t* pairs_removed) {
  if (!h || (!endpoints && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (pairs_removed) *pairs_removed = 0;
  for (uint32_t i = 0; i < n; ++i)
    if (endpoints[i] >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint out of range");
  if (h->world > 1) return fail(h, FI_ERR_STATE, "sharded pool: fi_epp_index_remove_endpoints needs a single-rank handle");
  const uint32_t lo = h->cfg.endpoint_begin, EL = h->cfg.endpoint_count;
  std::vector<uint32_t> local;  // distinct local endpoints
  std::vector<uint8_t> listed(EL, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t e = endpoints[i] - lo;
    if (e >= EL || listed[e]) continue;
    listed[e] = 1;
    local.push_back(e);
  }
  if (local.empty()) return FI_OK;
  return remove_local_endpoints(h, local, pairs_removed);
}

// Resize the pool of a single-rank handle over the whole pool (docs/SPEC.md S.2c).  Blocking: every call before it
// completes against the old pool first.  Every buffer the new pool needs is allocated before anything of the handle
// changes, so FI_ERR_NOMEM leaves the handle as it was; after the allocations only a CUDA error can fail the call.  The
// old and new copies of what is reallocated are both held until the end.
int fi_epp_resize_pool(fi_epp* h, uint32_t num_endpoints, uint64_t* pairs_removed) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (pairs_removed) *pairs_removed = 0;
  const uint32_t E = h->cfg.num_endpoints, En = num_endpoints, C = h->cfg.lru_capacity;
  if (En == 0 || En > 4096) return fail(h, FI_ERR_INVALID, "num_endpoints must be in 1 .. 4096");
  if (h->world > 1) return fail(h, FI_ERR_STATE, "sharded pool: fi_epp_resize_pool needs a single-rank handle");
  if (h->cfg.endpoint_begin != 0 || h->cfg.endpoint_count != E)
    return fail(h, FI_ERR_STATE, "fi_epp_resize_pool needs a handle over the whole pool");
  if (h->lru_mode == 0) return fail(h, FI_ERR_STATE, "fi_epp_resize_pool: the host LRU serves the handle");
  if (En == E) return FI_OK;
  int rc = update_begin(h);
  if (rc != FI_OK) return rc;
  for (cudaStream_t s : {h->s_main.get(), h->s_index.get(), h->s_copy.get(), h->s_a.get()}) FI_CUDA(cudaStreamSynchronize(s));
  // The slot floor counts the live keys before a shrink's removal: an upper bound of those after it, known before
  // anything changes.
  IndexCounters ctr;
  FI_CUDA(cudaMemcpy(&ctr, h->d_ctr.get(), sizeof(ctr), cudaMemcpyDeviceToHost));
  const uint32_t Wn = pool_row_words(En), Epad = Wn * 32, keep = std::min(E, En);
  const uint64_t slots = pool_resized_slots(h->index_slots_given, En, C, ctr.used - ctr.tombstones);
  const bool rebuild = pool_needs_rebuild(h->W, h->ix.v.C, Wn, slots);

  // ---- allocations: nothing of the handle changes before all of them are in place
  IndexTables nix;
  if (rebuild) {
    rc = alloc_index(h, slots, Wn, nix);
    if (rc != FI_OK) return rc;
  }
  std::vector<uint32_t> caps;  // the new pool's LRU capacities: the kept endpoints', then lru_capacity
  if (C) {
    caps.assign(h->lru_caps.begin(), h->lru_caps.begin() + keep);
    caps.resize(En, C);
  }
  std::unique_ptr<DevLruStore> nlru;
  if (h->dlru) {
    nlru = std::make_unique<DevLruStore>();
    rc = alloc_dev_lru(h, *nlru, En, h->dlru->v.TS, h->dlru->v.L, caps.data());
    if (rc != FI_OK) {
      cudaGetLastError();
      return rc;
    }
  }
  DevPtr<EndpointDev> d_eps;
  DevPtr<double> d_sc;
  DevPtr<uint32_t> d_elig, d_ztie;
  DevPtr<LoraDev> d_lora;
  const size_t n_sc = (size_t)FI_EPP_MAX_PROFILES * FI_EPP_MAX_SCORERS * Epad, n_bits = (size_t)FI_EPP_MAX_PROFILES * Wn;
  cudaError_t e = cuda_alloc(d_eps, En);
  if (e == cudaSuccess) e = cuda_alloc(d_sc, n_sc);
  if (e == cudaSuccess) e = cuda_alloc(d_elig, n_bits);
  if (e == cudaSuccess) e = cuda_alloc(d_ztie, n_bits);
  if (e == cudaSuccess) e = cuda_alloc(d_lora, Epad);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(h, e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA, std::string("endpoint tables: ") + cudaGetErrorString(e));
  }
  cudaStream_t si = h->s_index.get();
  FI_CUDA(cudaMemsetAsync(d_sc.get(), 0, n_sc * sizeof(double), si));
  FI_CUDA(cudaMemsetAsync(d_elig.get(), 0, n_bits * sizeof(uint32_t), si));
  FI_CUDA(cudaMemsetAsync(d_ztie.get(), 0, n_bits * sizeof(uint32_t), si));

  // ---- the dropped endpoints leave the index and their LRUs, exactly as fi_epp_index_remove_endpoints removes them
  if (En < E) {
    std::vector<uint32_t> gone;
    for (uint32_t x = En; x < E; ++x) gone.push_back(x);
    rc = remove_local_endpoints(h, gone, pairs_removed);
    if (rc != FI_OK) return rc;
  }
  // ---- the index in its new shape: rebuilt only when the row width or the slot count changes
  if (rebuild) {
    FI_CUDA(cudaMemsetAsync(h->d_ctr.get(), 0, sizeof(IndexCounters), si));
    LaunchScope ls(h, si, K_INDEX);
    FI_CUDA(launch_index_rebuild(h->ix.v, nix.v, h->d_ctr.get(), si));
  }
  // ---- the device LRU: its regions are endpoint-major, so the kept endpoints move with one prefix copy per array;
  // the new ones start empty (alloc_dev_lru), and the totals carry over
  if (nlru) {
    const DevLru& o = h->dlru->v;
    const DevLru& n = nlru->v;
    FI_CUDA(cudaMemcpyAsync(n.slots, o.slots, (size_t)keep * (o.TS + 2) * sizeof(LruSlot), cudaMemcpyDeviceToDevice, si));
    FI_CUDA(cudaMemcpyAsync(n.log, o.log, (size_t)keep * o.L * sizeof(uint64_t), cudaMemcpyDeviceToDevice, si));
    const std::pair<uint32_t*, const uint32_t*> arrays[] = {{n.head, o.head}, {n.tail, o.tail},   {n.count, o.count}, {n.used, o.used},
                                                            {n.hold, o.hold}, {n.dcount, o.dcount}, {n.ovf, o.ovf}};
    for (const auto& a : arrays) FI_CUDA(cudaMemcpyAsync(a.first, a.second, (size_t)keep * sizeof(uint32_t), cudaMemcpyDeviceToDevice, si));
    FI_CUDA(cudaMemcpyAsync(n.any_ovf, o.any_ovf, 2 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, si));  // any_ovf, error
    FI_CUDA(cudaMemcpyAsync(nlru->ctr.get(), h->dlru->ctr.get(), 8 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, si));
    *nlru->stat = *h->dlru->stat;
    FI_CUDA(cudaEventRecord(nlru->ev.get(), si));
  }

  // ---- swap in the new pool (the old buffers stay allocated until the work above is done)
  if (rebuild) {
    std::swap(h->ix, nix);
    h->ix_spare.reset();  // a later rebuild allocates it in the new shape
  }
  if (nlru) std::swap(h->dlru, nlru);
  h->eps.resize(keep);
  h->eps.resize(En, EndpointDev{0.0, 0, 0, 0, 0});
  h->lora.resize(keep);
  h->lora.resize(Epad, LoraDev{});
  std::swap(h->d_eps, d_eps);
  std::swap(h->d_sc, d_sc);
  std::swap(h->d_elig, d_elig);
  std::swap(h->d_ztie, d_ztie);
  std::swap(h->d_lora, d_lora);
  h->st.Epad = Epad;
  h->st.sc = h->d_sc.get();
  h->st.elig = h->d_elig.get();
  h->st.ztie = h->d_ztie.get();
  h->st.lora = h->d_lora.get();
  h->eps_dirty = h->lora_dirty = true;
  if (C) {
    // no Add has run through the host LRUs (lru_mode != 0): they are empty and only carry the capacities
    h->lrus.clear();
    LruArena* arena = h->lru_arena.reserve((size_t)En * LruSet::bytes_needed(C)) ? &h->lru_arena : nullptr;
    h->lrus = std::vector<LruSet>(En, LruSet(C, arena));
    for (uint32_t x = 0; x < En; ++x)
      if (caps[x] != C) h->lrus[x].shrink(caps[x], [](uint64_t) {});
    h->lru_caps.swap(caps);
  }
  // lazily created buffers sized by the pool: their next use allocates them anew
  h->d_rm.reset();
  h->subsets = Staging<uint32_t>{};
  h->lru_plan_buf = Staging<uint32_t>{};
  h->lru_resize = Staging<uint32_t>{};
  for (fi_epp::PipeAdd& pa : h->padd) pa.plan = Staging<uint32_t>{};
  h->cfg.num_endpoints = h->cfg.endpoint_count = En;
  h->cfg.index_slots = h->ix.v.C;
  h->W = Wn;
  rc = update_end(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamSynchronize(si));
  return FI_OK;
}

// ---- index snapshots (docs/SPEC.md S.2d) -----------------------------------------------------------------------
namespace {

// Both directions move the blob between the caller's pageable buffer and device buffers through two pinned buffers of
// kSnapStage bytes: the copy engine fills (drains) one while the host copies the other.  Nothing larger is pinned.
constexpr uint64_t kSnapStage = 32ull << 20;

struct SnapStager {
  PinnedPtr<uint8_t> buf[2];
  Event ev[2];
  int k = 0;
  uint64_t cap = kSnapStage;  // bytes per buffer
};

cudaError_t snap_stager_alloc(SnapStager& st, uint64_t cap = kSnapStage) {
  st.cap = std::max<uint64_t>(cap, 1);
  for (int i = 0; i < 2; ++i) {
    cudaError_t e = cuda_alloc(st.buf[i], st.cap);
    if (e == cudaSuccess) e = cuda_create(st.ev[i]);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

int snap_stager(fi_epp* h, SnapStager& st) {
  if (snap_stager_alloc(st) != cudaSuccess) {
    cudaGetLastError();
    return fail(h, FI_ERR_NOMEM, "cannot allocate the pinned snapshot staging");
  }
  return FI_OK;
}

// device [src, src + bytes) -> host dst, on stream s (returns when dst is written)
cudaError_t snap_d2h(cudaStream_t s, SnapStager& st, uint8_t* dst, const void* src, uint64_t bytes) {
  int prev = -1;
  uint64_t prev_off = 0, prev_n = 0;
  cudaError_t e = cudaSuccess;
  for (uint64_t off = 0; off < bytes && e == cudaSuccess; off += st.cap) {
    const uint64_t n = std::min(st.cap, bytes - off);
    const int k = st.k;
    st.k ^= 1;
    // (buf[k] was drained by the previous iteration's host copy)
    e = cudaMemcpyAsync(st.buf[k].get(), static_cast<const uint8_t*>(src) + off, n, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaEventRecord(st.ev[k].get(), s);
    if (e == cudaSuccess && prev >= 0) e = cudaEventSynchronize(st.ev[prev].get());
    if (e == cudaSuccess && prev >= 0) std::memcpy(dst + prev_off, st.buf[prev].get(), prev_n);
    prev = k;
    prev_off = off;
    prev_n = n;
  }
  if (e == cudaSuccess && prev >= 0) e = cudaEventSynchronize(st.ev[prev].get());
  if (e == cudaSuccess && prev >= 0) std::memcpy(dst + prev_off, st.buf[prev].get(), prev_n);
  return e;
}

// host [src, src + bytes) -> device dst, queued on s_index (src may be reused when the call returns)
int snap_h2d(fi_epp* h, SnapStager& st, void* dst, const uint8_t* src, uint64_t bytes) {
  cudaStream_t si = h->s_index.get();
  for (uint64_t off = 0; off < bytes; off += st.cap) {
    const uint64_t n = std::min(st.cap, bytes - off);
    const int k = st.k;
    st.k ^= 1;
    FI_CUDA(cudaEventSynchronize(st.ev[k].get()));  // the copy out of buf[k] two pieces ago is done
    std::memcpy(st.buf[k].get(), src + off, n);
    FI_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(dst) + off, st.buf[k].get(), n, cudaMemcpyHostToDevice, si));
    FI_CUDA(cudaEventRecord(st.ev[k].get(), si));
  }
  h->stats.h2d_bytes += bytes;
  return FI_OK;
}

// nodes per chunk of the device staging of node keys and rows (at least one export tile)
uint64_t snap_chunk_nodes(uint32_t We) { return std::max<uint64_t>(1024, (64ull << 20) / (8 + 4ull * We)); }

unsigned snap_threads() { return std::min(usable_cores(), 16u); }

// save and load need a single-rank handle over the whole pool whose LRU, if it has one, is the device LRU
int snapshot_handle_ok(fi_epp* h, const char* what) {
  if (h->world > 1) return fail(h, FI_ERR_STATE, std::string("sharded pool: ") + what + " needs a single-rank handle");
  if (h->cfg.endpoint_begin != 0 || h->cfg.endpoint_count != h->cfg.num_endpoints)
    return fail(h, FI_ERR_STATE, std::string(what) + " needs a handle over the whole pool");
  if (h->cfg.lru_capacity) {
    int rc = choose_lru_mode(h);
    if (rc != FI_OK) return rc;
    if (h->lru_mode == 0) return fail(h, FI_ERR_STATE, std::string(what) + ": the host LRU serves the handle");
  }
  return FI_OK;
}

int sync_all_streams(fi_epp* h) {
  for (cudaStream_t s : {h->s_main.get(), h->s_index.get(), h->s_copy.get(), h->s_a.get()}) FI_CUDA(cudaStreamSynchronize(s));
  return FI_OK;
}

// The sizes of a snapshot of the state every call issued so far leaves (the save's and the capture's first step)
struct SnapSizes {
  uint64_t n = 0;                           // regular nodes the export walks: min(used, C)
  uint32_t tiles = 0;                       // index_snap_tiles(n)
  std::vector<uint64_t> tile_off, lru_off;  // [tiles + 1] live nodes before each tile, [E + 1] LRU entries before each endpoint
  std::vector<uint32_t> caps, lens;         // the payload's caps and lru_len sections
  SnapHeader hd{};                          // complete but for the checksum
  SnapLayout l{};
};

// The staged ops are flushed (settle_updates; drain: then every stream of h is synchronised, picks in flight included).
// Then, behind the updates already queued on s_index, the count pass, the index counters and the LRUs' entry counts
// are read back with one synchronisation of s_index.  The tile counts' buffer is stream-ordered: a cudaFree would wait
// for the picks in flight.
int snap_sizes(fi_epp* h, bool drain, SnapSizes& z) {
  int rc = settle_updates(h);
  if (rc == FI_OK && drain) rc = sync_all_streams(h);
  if (rc != FI_OK) return rc;
  cudaStream_t si = h->s_index.get();
  const uint32_t E = h->cfg.num_endpoints, C = h->cfg.lru_capacity;
  const uint32_t all = index_snap_tiles(h->ix.v.C);
  uint32_t* d_tile = nullptr;
  if (cudaMallocAsync(&d_tile, (size_t)all * sizeof(uint32_t), si) != cudaSuccess) {
    cudaGetLastError();
    return fail(h, FI_ERR_NOMEM, "cannot allocate the snapshot's tile counts");
  }
  std::vector<uint32_t> tile(all);
  IndexCounters ctr;
  z.caps.assign(E, 0);
  z.lens.assign(E, 0);
  if (C) z.caps = h->lru_caps;
  cudaError_t e;
  {
    LaunchScope ls(h, si, K_OTHER);
    e = launch_index_snap_count(h->ix.v, h->d_ctr.get(), d_tile, si);
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(tile.data(), d_tile, (size_t)all * sizeof(uint32_t), cudaMemcpyDeviceToHost, si);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&ctr, h->d_ctr.get(), sizeof(ctr), cudaMemcpyDeviceToHost, si);
  if (e == cudaSuccess && h->dlru) e = cudaMemcpyAsync(z.lens.data(), h->dlru->v.count, (size_t)E * sizeof(uint32_t), cudaMemcpyDeviceToHost, si);
  const cudaError_t ef = cudaFreeAsync(d_tile, si);
  if (e == cudaSuccess) e = ef;
  if (e == cudaSuccess) e = cudaStreamSynchronize(si);
  FI_CUDA(e);
  z.n = std::min<uint64_t>(ctr.used, h->ix.v.C);
  z.tiles = index_snap_tiles(z.n);
  z.tile_off.assign((size_t)z.tiles + 1, 0);
  z.lru_off.assign((size_t)E + 1, 0);
  for (uint32_t t = 0; t < z.tiles; ++t) z.tile_off[t + 1] = z.tile_off[t] + tile[t];
  for (uint32_t x = 0; x < E; ++x) z.lru_off[x + 1] = z.lru_off[x] + z.lens[x];
  const uint64_t n_nodes = z.tile_off[z.tiles], n_lru = z.lru_off[E];
  z.l = snap_layout(E, n_nodes, n_lru);
  SnapHeader& hd = z.hd;
  std::memcpy(hd.magic, kSnapMagic, 8);
  hd.version = kSnapVersion;
  hd.header_bytes = kSnapHeaderBytes;
  hd.block_bytes = h->cfg.block_bytes;
  hd.max_blocks = h->cfg.max_blocks;
  hd.lru_capacity = C;
  hd.num_endpoints = E;
  hd.n_nodes = n_nodes;
  hd.n_lru = n_lru;
  hd.payload_bytes = z.l.end;
  return FI_OK;
}

}  // namespace

// Save (S.2d).  Blocking; the handle is not changed.  Sizes first (snap_sizes), which gives the header.  Then the
// sections are written in payload order: the capacities and LRU lengths from the host, every LRU's keys from one dump
// of all endpoints, the nodes chunk by chunk through the device staging; last the checksum, over the caller's buffer on
// host threads.
int fi_epp_snapshot_save(fi_epp* h, void* buf, uint64_t cap, uint64_t* bytes) {
  if (!h || !bytes) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = snapshot_handle_ok(h, "fi_epp_snapshot_save");
  if (rc != FI_OK) return rc;
  SnapSizes z;
  rc = snap_sizes(h, /*drain=*/true, z);  // (picks in flight included: the state saved is the one every earlier call left)
  if (rc != FI_OK) return rc;
  cudaStream_t si = h->s_index.get();
  const uint32_t E = h->cfg.num_endpoints, We = snap_row_words(E);
  const SnapLayout& l = z.l;
  const uint64_t n_nodes = z.hd.n_nodes, n_lru = z.hd.n_lru;
  *bytes = kSnapHeaderBytes + l.end;
  if (!buf) return FI_OK;
  if (cap < *bytes) return fail(h, FI_ERR_CAPACITY, "snapshot buffer of " + std::to_string(cap) + " bytes, " + std::to_string(*bytes) + " needed");

  SnapStager st;
  rc = snap_stager(h, st);
  if (rc != FI_OK) return rc;
  auto d2h = [&](uint8_t* dst, const void* src, uint64_t n) {
    FI_CUDA(snap_d2h(si, st, dst, src, n));
    h->stats.d2h_bytes += n;
    return FI_OK;
  };
  uint8_t* out = static_cast<uint8_t*>(buf);
  uint8_t* pay = out + kSnapHeaderBytes;
  SnapHeader hd = z.hd;
  std::memcpy(pay + l.caps, z.caps.data(), 4ull * E);
  std::memcpy(pay + l.lru_len, z.lens.data(), 4ull * E);
  // every LRU, oldest first, in one launch
  if (n_lru) {
    DevPtr<uint64_t> d_keys, d_off;
    DevPtr<uint32_t> d_n;
    if (cuda_alloc(d_keys, n_lru) != cudaSuccess || cuda_alloc(d_off, E) != cudaSuccess || cuda_alloc(d_n, E) != cudaSuccess) {
      cudaGetLastError();
      return fail(h, FI_ERR_NOMEM, "cannot allocate the snapshot's LRU staging");
    }
    FI_CUDA(cudaMemcpyAsync(d_off.get(), z.lru_off.data(), (size_t)E * sizeof(uint64_t), cudaMemcpyHostToDevice, si));
    {
      LaunchScope ls(h, si, K_OTHER);
      FI_CUDA(launch_lru_dump_all(h->dlru->v, d_off.get(), d_keys.get(), d_n.get(), nullptr, si));
    }
    std::vector<uint32_t> got(E);
    FI_CUDA(cudaMemcpyAsync(got.data(), d_n.get(), (size_t)E * sizeof(uint32_t), cudaMemcpyDeviceToHost, si));
    rc = d2h(pay + l.lru_keys, d_keys.get(), 8 * n_lru);
    if (rc != FI_OK) return rc;
    if (got != z.lens) return fail(h, FI_ERR_STATE, "device LRU: live records differ from the entry counts (broken invariant)");
  }
  // the nodes, a range of tiles per chunk of the device staging
  if (n_nodes) {
    const uint64_t chunk = snap_chunk_nodes(We);
    const std::vector<uint64_t>& tile_off = z.tile_off;
    DevPtr<uint64_t> d_keys, d_tile_off;
    DevPtr<uint32_t> d_rows;
    if (cuda_alloc(d_keys, chunk) != cudaSuccess || cuda_alloc(d_rows, chunk * We) != cudaSuccess ||
        cuda_alloc(d_tile_off, (size_t)z.tiles + 1) != cudaSuccess) {
      cudaGetLastError();
      return fail(h, FI_ERR_NOMEM, "cannot allocate the snapshot's node staging");
    }
    FI_CUDA(cudaMemcpyAsync(d_tile_off.get(), tile_off.data(), ((size_t)z.tiles + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, si));
    for (uint32_t t0 = 0; t0 < z.tiles;) {
      uint32_t t1 = t0;
      while (t1 < z.tiles && tile_off[t1 + 1] - tile_off[t0] <= chunk) ++t1;
      const uint64_t base = tile_off[t0], m = tile_off[t1] - base;
      {
        LaunchScope ls(h, si, K_OTHER);
        FI_CUDA(launch_index_snap_export(h->ix.v, z.n, t0, t1, d_tile_off.get(), base, We, d_keys.get(), d_rows.get(), si));
      }
      rc = d2h(pay + l.node_keys + 8 * base, d_keys.get(), 8 * m);
      if (rc == FI_OK) rc = d2h(pay + l.node_rows + 4ull * We * base, d_rows.get(), 4ull * We * m);
      if (rc != FI_OK) return rc;
      t0 = t1;
    }
  }
  hd.checksum = snap_checksum(&hd, pay, l.end, snap_threads());
  std::memcpy(out, &hd, sizeof(hd));
  return FI_OK;
}

// A snapshot taken on the device (S.2d, captures).  The payload from the lru_keys section on lives in one device image,
// which the capture's kernels write on the handle's s_index; the header and the caps and lru_len sections are known
// on the host from the sizing step.  read and free use only what the object owns: its device, its stream, the image,
// the small buffer beside it and the event recorded after the export.  Both buffers are stream-ordered allocations on
// the capture's stream, so that freeing them stalls no stream of the handle (cudaFree synchronises the device).
struct fi_epp_capture {
  Stream s;                 // declared first so that it is destroyed last
  Event ev_ready, ev_done;  // the buffers are allocated (recorded on s); the export is done (recorded on h's s_index)
  int device = 0;
  SnapHeader hd{};          // checksum 0: read computes it
  SnapLayout l{};
  std::vector<uint32_t> caps_lens;  // the caps and lru_len sections, in payload order
  uint8_t* image = nullptr;         // payload bytes [l.lru_keys, l.end)
  uint8_t* aux = nullptr;           // tile_off[tiles + 1] u64 | lru_off[E] u64 | dumped[E] u32 | bad u32
  uint64_t aux_bad = 0;             // byte offset of `bad`: 1 if an LRU's live records differ from its entry count
  ~fi_epp_capture() {
    if (!s) return;
    cudaSetDevice(device);
    // behind the export (a wait for an event never recorded waits for nothing)
    if (ev_done) cudaStreamWaitEvent(s.get(), ev_done.get(), 0);
    if (image) cudaFreeAsync(image, s.get());
    if (aux) cudaFreeAsync(aux, s.get());
  }
};

namespace {

// the capture's device work on s_index, after the wait for its buffers: the dump of every LRU and one export of every
// tile, straight into the image at their sections' offsets
int capture_enqueue(fi_epp* h, fi_epp_capture& c, const SnapSizes& z) {
  cudaStream_t si = h->s_index.get();
  const uint32_t E = h->cfg.num_endpoints, We = snap_row_words(E);
  const SnapLayout& l = c.l;
  uint64_t* d_tile_off = reinterpret_cast<uint64_t*>(c.aux);
  uint64_t* d_lru_off = d_tile_off + z.tiles + 1;
  uint32_t* d_dumped = reinterpret_cast<uint32_t*>(d_lru_off + E);
  uint32_t* d_bad = d_dumped + E;
  FI_CUDA(cudaStreamWaitEvent(si, c.ev_ready.get(), 0));
  // (pageable sources: the copies have taken the data when cudaMemcpyAsync returns)
  FI_CUDA(cudaMemcpyAsync(d_tile_off, z.tile_off.data(), ((size_t)z.tiles + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, si));
  FI_CUDA(cudaMemcpyAsync(d_lru_off, z.lru_off.data(), (size_t)E * sizeof(uint64_t), cudaMemcpyHostToDevice, si));
  FI_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), si));
  if (z.hd.n_lru) {
    LaunchScope ls(h, si, K_OTHER);
    FI_CUDA(launch_lru_dump_all(h->dlru->v, d_lru_off, reinterpret_cast<uint64_t*>(c.image), d_dumped, d_bad, si));
  }
  if (z.hd.n_nodes) {
    LaunchScope ls(h, si, K_OTHER);
    FI_CUDA(launch_index_snap_export(h->ix.v, z.n, 0, z.tiles, d_tile_off, 0, We, reinterpret_cast<uint64_t*>(c.image + (l.node_keys - l.lru_keys)),
                                     reinterpret_cast<uint32_t*>(c.image + (l.node_rows - l.lru_keys)), si));
  }
  return FI_OK;
}

}  // namespace

// Capture (S.2d).  Holds h->mu for the sizing step (one synchronisation of s_index, no wait for picks), the allocation
// of the image and the queueing of its device work on s_index, behind every update issued before it and ahead of every
// later one.  Picks neither wait for it nor are waited for.
int fi_epp_snapshot_capture(fi_epp* h, fi_epp_capture** out, uint64_t* bytes) {
  if (!h || !out || !bytes) return FI_ERR_INVALID;
  *out = nullptr;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = snapshot_handle_ok(h, "fi_epp_snapshot_capture");
  if (rc != FI_OK) return rc;
  SnapSizes z;
  rc = snap_sizes(h, /*drain=*/false, z);
  if (rc != FI_OK) return rc;
  const uint32_t E = h->cfg.num_endpoints;
  auto c = std::make_unique<fi_epp_capture>();
  c->device = h->cfg.device;
  c->hd = z.hd;
  c->l = z.l;
  c->caps_lens = z.caps;
  c->caps_lens.insert(c->caps_lens.end(), z.lens.begin(), z.lens.end());
  const uint64_t img = z.l.end - z.l.lru_keys;
  c->aux_bad = 8ull * (z.tiles + 1) + 12ull * E;
  cudaError_t e = cuda_create(c->s);
  if (e == cudaSuccess) e = cuda_create(c->ev_ready);
  if (e == cudaSuccess) e = cuda_create(c->ev_done);
  cudaStream_t cs = c->s.get();
  if (e == cudaSuccess && img) e = cudaMallocAsync(reinterpret_cast<void**>(&c->image), img, cs);
  if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void**>(&c->aux), c->aux_bad + sizeof(uint32_t), cs);
  if (e == cudaSuccess) e = cudaEventRecord(c->ev_ready.get(), cs);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(h, e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA,
                "snapshot capture: a device image of " + std::to_string(img) + " bytes: " + cudaGetErrorString(e) +
                    " (fi_epp_snapshot_save needs only bounded staging)");
  }
  rc = capture_enqueue(h, *c, z);
  // (recorded on failure too: the buffers are freed behind whatever reached s_index)
  const cudaError_t ed = cudaEventRecord(c->ev_done.get(), h->s_index.get());
  if (rc != FI_OK) return rc;
  FI_CUDA(ed);
  FI_CUDA(cudaStreamWaitEvent(cs, c->ev_done.get(), 0));
  *bytes = kSnapHeaderBytes + z.l.end;
  *out = c.release();
  return FI_OK;
}

// Read (S.2d).  Never touches the handle: the capture's stream waits for the export, the image comes out through
// bounded pinned staging, and the checksum is computed on host threads.
int fi_epp_snapshot_read(fi_epp_capture* c, void* buf, uint64_t cap) {
  if (!c || !buf) return FI_ERR_INVALID;
  const SnapLayout& l = c->l;
  if (cap < kSnapHeaderBytes + l.end) return FI_ERR_CAPACITY;
  if (cudaSetDevice(c->device) != cudaSuccess) return FI_ERR_CUDA;
  cudaStream_t cs = c->s.get();
  uint32_t bad = 0;
  cudaError_t e = cudaMemcpyAsync(&bad, c->aux + c->aux_bad, sizeof(bad), cudaMemcpyDeviceToHost, cs);
  if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
  if (e != cudaSuccess) return FI_ERR_CUDA;
  if (bad) return FI_ERR_STATE;  // (as the save: an LRU's live records differ from its entry count)
  uint8_t* pay = static_cast<uint8_t*>(buf) + kSnapHeaderBytes;
  const uint64_t img = l.end - l.lru_keys;
  if (img) {
    SnapStager st;
    e = snap_stager_alloc(st, std::min(kSnapStage, img));
    if (e != cudaSuccess) {
      cudaGetLastError();
      return e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA;
    }
    if (snap_d2h(cs, st, pay + l.lru_keys, c->image, img) != cudaSuccess) return FI_ERR_CUDA;
  }
  std::memcpy(pay, c->caps_lens.data(), 4 * c->caps_lens.size());
  SnapHeader hd = c->hd;
  hd.checksum = snap_checksum(&hd, pay, l.end, snap_threads());
  std::memcpy(buf, &hd, sizeof(hd));
  return FI_OK;
}

void fi_epp_snapshot_free(fi_epp_capture* c) { delete c; }

// Load (S.2d).  The blob is checked on the host first (snap_check, marker keys, the configuration, room in the index);
// then, with every earlier call complete, new index tables and a new device LRU are built from it on s_index and
// checked for duplicate keys; only then are they swapped in.  Until the swap nothing of the handle changes.
int fi_epp_snapshot_load(fi_epp* h, const void* buf, uint64_t len) {
  if (!h || (!buf && len)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = snapshot_handle_ok(h, "fi_epp_snapshot_load");
  if (rc != FI_OK) return rc;
  SnapHeader hd;
  uint64_t pairs = 0;
  std::string why;
  if (!snap_check(buf, len, snap_threads(), &hd, &pairs, &why)) return fail(h, FI_ERR_INVALID, why);
  const uint32_t E = h->cfg.num_endpoints, C = h->cfg.lru_capacity, We = snap_row_words(E);
  if (hd.block_bytes != h->cfg.block_bytes || hd.max_blocks != h->cfg.max_blocks || hd.lru_capacity != C || hd.num_endpoints != E)
    return fail(h, FI_ERR_INVALID, "snapshot of another configuration (block_bytes, max_blocks, lru_capacity or num_endpoints)");
  const uint8_t* pay = static_cast<const uint8_t*>(buf) + kSnapHeaderBytes;
  const SnapLayout l = snap_layout(E, hd.n_nodes, hd.n_lru);
  uint64_t m0 = kSnapNone, m1 = kSnapNone;
  if (!snap_markers(pay + l.node_keys, hd.n_nodes, &m0, &m1)) return fail(h, FI_ERR_INVALID, "snapshot repeats a node key");
  const uint64_t regular = hd.n_nodes - (m0 != kSnapNone) - (m1 != kSnapNone);
  const uint64_t slots = pool_resized_slots(h->index_slots_given, E, C, regular);
  if (regular * 10 > slots * 6) return fail(h, FI_ERR_CAPACITY, "snapshot keys above 60% of index_slots: raise index_slots");
  std::vector<uint32_t> caps(E), lens(E);
  std::memcpy(caps.data(), pay + l.caps, 4ull * E);
  std::memcpy(lens.data(), pay + l.lru_len, 4ull * E);
  std::vector<uint64_t> lru_off(E + 1, 0);
  for (uint32_t e = 0; e < E; ++e) lru_off[e + 1] = lru_off[e] + lens[e];

  rc = update_begin(h);
  if (rc != FI_OK) return rc;
  rc = sync_all_streams(h);
  if (rc != FI_OK) return rc;
  cudaStream_t si = h->s_index.get();
  // ---- allocations: nothing of the handle changes before all of them are in place
  IndexTables nix;
  rc = alloc_index(h, slots, h->W, nix);
  if (rc != FI_OK) return rc;
  std::unique_ptr<DevLruStore> nlru;
  if (C) {
    uint32_t TS = 0, L = 0;
    if (h->dlru) {
      TS = h->dlru->v.TS;
      L = h->dlru->v.L;
    } else {
      rc = size_dev_lru(h, &TS, &L);
      if (rc != FI_OK) return rc;
    }
    nlru = std::make_unique<DevLruStore>();
    rc = alloc_dev_lru(h, *nlru, E, TS, L, caps.data());
    if (rc != FI_OK) {
      cudaGetLastError();
      return rc;
    }
  }
  const uint64_t chunk = snap_chunk_nodes(We);
  DevPtr<uint64_t> d_keys, d_lkeys, d_loff;
  DevPtr<uint32_t> d_rows, d_llen, d_dup;
  DevPtr<IndexCounters> d_sctr;
  cudaError_t e = cuda_alloc(d_dup, 2);
  if (e == cudaSuccess) e = cuda_alloc(d_sctr, 1);
  if (e == cudaSuccess && hd.n_nodes) e = cuda_alloc(d_keys, std::min(chunk, hd.n_nodes));
  if (e == cudaSuccess && hd.n_nodes) e = cuda_alloc(d_rows, std::min(chunk, hd.n_nodes) * We);
  if (e == cudaSuccess && hd.n_lru) e = cuda_alloc(d_lkeys, hd.n_lru);
  if (e == cudaSuccess && C) e = cuda_alloc(d_loff, E);
  if (e == cudaSuccess && C) e = cuda_alloc(d_llen, E);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(h, e == cudaErrorMemoryAllocation ? FI_ERR_NOMEM : FI_ERR_CUDA, std::string("snapshot staging: ") + cudaGetErrorString(e));
  }
  SnapStager st;
  rc = snap_stager(h, st);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaMemsetAsync(d_dup.get(), 0, 2 * sizeof(uint32_t), si));
  FI_CUDA(cudaMemsetAsync(d_sctr.get(), 0, sizeof(IndexCounters), si));

  // ---- build: the LRUs, then the nodes in blob order
  if (nlru) {
    rc = snap_h2d(h, st, d_lkeys.get(), pay + l.lru_keys, 8 * hd.n_lru);
    if (rc != FI_OK) return rc;
    // (pageable sources: the copies have taken the data when cudaMemcpyAsync returns)
    FI_CUDA(cudaMemcpyAsync(d_loff.get(), lru_off.data(), (size_t)E * sizeof(uint64_t), cudaMemcpyHostToDevice, si));
    FI_CUDA(cudaMemcpyAsync(d_llen.get(), lens.data(), (size_t)E * sizeof(uint32_t), cudaMemcpyHostToDevice, si));
    LaunchScope ls(h, si, K_INDEX);
    FI_CUDA(launch_lru_load(nlru->v, d_lkeys.get(), d_loff.get(), d_llen.get(), d_dup.get(), si));
  }
  for (uint64_t g0 = 0; g0 < hd.n_nodes; g0 += chunk) {
    const uint64_t m = std::min(chunk, hd.n_nodes - g0);
    // (the staging is rewritten only behind the previous chunk's import: all of it runs on s_index)
    rc = snap_h2d(h, st, d_keys.get(), pay + l.node_keys + 8 * g0, 8 * m);
    if (rc == FI_OK) rc = snap_h2d(h, st, d_rows.get(), pay + l.node_rows + 4ull * We * g0, 4ull * We * m);
    if (rc != FI_OK) return rc;
    LaunchScope ls(h, si, K_INDEX);
    FI_CUDA(launch_index_snap_import(nix.v, d_sctr.get(), d_keys.get(), d_rows.get(), m, g0, m0, m1, We, d_dup.get(), si));
  }
  // ---- check
  uint32_t dup = 0, lru_err = 0;
  IndexCounters sctr;
  FI_CUDA(cudaMemcpyAsync(&dup, d_dup.get(), sizeof(dup), cudaMemcpyDeviceToHost, si));
  FI_CUDA(cudaMemcpyAsync(&sctr, d_sctr.get(), sizeof(sctr), cudaMemcpyDeviceToHost, si));
  if (nlru) FI_CUDA(cudaMemcpyAsync(&lru_err, nlru->v.error, sizeof(lru_err), cudaMemcpyDeviceToHost, si));
  FI_CUDA(cudaStreamSynchronize(si));
  if (dup) return fail(h, FI_ERR_INVALID, "snapshot repeats a key in the index or in an LRU");
  if (sctr.overflow) return fail(h, FI_ERR_CAPACITY, "snapshot keys do not fit the index");
  if (lru_err) return fail(h, FI_ERR_STATE, "device LRU: invariant " + std::to_string(lru_err) + " broken while loading");

  // ---- swap in the loaded state (the old tables stay allocated until the end of the call)
  const IndexCounters fresh{regular, 0, 0, 0};
  FI_CUDA(cudaMemcpyAsync(h->d_ctr.get(), &fresh, sizeof(fresh), cudaMemcpyHostToDevice, si));
  if (nlru && h->dlru) {  // the statistics keep counting
    FI_CUDA(cudaMemcpyAsync(nlru->ctr.get(), h->dlru->ctr.get(), 8 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, si));
    *nlru->stat = *h->dlru->stat;
  }
  if (nlru) FI_CUDA(cudaEventRecord(nlru->ev.get(), si));
  std::swap(h->ix, nix);
  h->ix_spare.reset();  // a later rebuild allocates it in the new size
  h->cfg.index_slots = h->ix.v.C;
  h->ctr_used_known = regular;
  h->ctr_unchecked = 0;
  if (nlru) {
    std::swap(h->dlru, nlru);
    h->lru_caps = caps;
    for (uint32_t x = 0; x < E; ++x) h->lrus[x].shrink(caps[x], [](uint64_t) {});  // (empty: they only take the limit)
  }
  rc = update_end(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamSynchronize(si));
  return FI_OK;
}

int fi_epp_snapshot_info(const void* buf, uint64_t len, struct fi_epp_snapshot_info* out) {
  if ((!buf && len) || !out) return FI_ERR_INVALID;
  SnapHeader hd;
  uint64_t pairs = 0;
  std::string why;
  if (!snap_check(buf, len, snap_threads(), &hd, &pairs, &why)) return FI_ERR_INVALID;
  out->block_bytes = hd.block_bytes;
  out->max_blocks = hd.max_blocks;
  out->lru_capacity = hd.lru_capacity;
  out->num_endpoints = hd.num_endpoints;
  out->n_nodes = hd.n_nodes;
  out->n_lru = hd.n_lru;
  out->pairs = pairs;
  out->bytes = len;
  return FI_OK;
}

// Per-endpoint LRU capacities (SPEC S.2b; upstream's autoTune).  The listed endpoints' LRUs evict their least recently
// used keys down to the new capacities, each evicted pair CLEARed as an eviction inside an Add would be; later Adds
// evict against them.  The host LRU's limits are set whichever LRU serves the handle (before the first Add it is not
// chosen yet, and both are empty then); the device LRU reads h->lru_caps when it is allocated.
int fi_epp_set_lru_capacities(fi_epp* h, const uint32_t* endpoints, const uint32_t* capacities, uint32_t n,
                              uint64_t* entries_evicted) {
  if (!h || ((!endpoints || !capacities) && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (entries_evicted) *entries_evicted = 0;
  const uint32_t C = h->cfg.lru_capacity;
  if (!C) return fail(h, FI_ERR_STATE, "lru_capacity is 0: no LRU to size");
  for (uint32_t i = 0; i < n; ++i) {
    if (endpoints[i] >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint out of range");
    if (capacities[i] > C) return fail(h, FI_ERR_INVALID, "LRU capacity above lru_capacity");
    if (capacities[i] && capacities[i] < h->cfg.max_blocks) return fail(h, FI_ERR_INVALID, "LRU capacity below max_blocks");
  }
  if (h->world > 1) return fail(h, FI_ERR_STATE, "sharded pool: fi_epp_set_lru_capacities needs a single-rank handle");
  const uint32_t lo = h->cfg.endpoint_begin, EL = h->cfg.endpoint_count;
  std::vector<uint32_t> caps = h->lru_caps;
  std::vector<uint32_t> local;  // distinct local endpoints listed
  std::vector<uint8_t> listed(EL, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t e = endpoints[i] - lo;
    if (e >= EL) continue;  // another rank's shard
    caps[e] = capacities[i] ? capacities[i] : C;  // the last entry wins
    if (!listed[e]) {
      listed[e] = 1;
      local.push_back(e);
    }
  }
  if (local.empty()) return FI_OK;
  int rc = settle_updates(h);
  if (rc != FI_OK) return rc;
  uint64_t evicted = 0;
  if (h->lru_mode == 1 && h->dlru) {
    rc = lru_device_resize(h, local, caps, &evicted);
    if (rc != FI_OK) return rc;
  }
  // host LRU: the evictions are staged like the deltas of an Add; the sets of a device-LRU handle are empty and only
  // take the limit
  for (uint32_t e : local) {
    rc = FI_OK;
    h->lrus[e].shrink(caps[e], [&](uint64_t key) {
      if (rc == FI_OK) rc = submit_op(h, key, lo + e, FI_OP_CLEAR);
      ++evicted;
    });
    if (rc != FI_OK) return rc;
  }
  h->lru_caps.swap(caps);
  if (entries_evicted) {
    rc = flush_ops(h);
    if (rc != FI_OK) return rc;
    FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
    rc = check_counters(h);  // (a broken device-LRU invariant would show here)
    if (rc != FI_OK) return rc;
    *entries_evicted = evicted;
  }
  return FI_OK;
}

int fi_epp_index_add_chain(fi_epp* h, uint32_t endpoint, const uint64_t* hashes, uint32_t n) {
  if (!h || (!hashes && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (!h->cfg.lru_capacity) return fail(h, FI_ERR_STATE, "lru_capacity is 0: the host LRU is disabled");
  if (h->world > 1) return fail(h, FI_ERR_STATE, "sharded pool: use the collective fi_epp_index_add_chains");  // (device LRU too)
  if (endpoint >= h->cfg.num_endpoints) return fail(h, FI_ERR_INVALID, "endpoint out of range");
  const uint32_t e = endpoint - h->cfg.endpoint_begin;
  if (e >= h->cfg.endpoint_count) return FI_OK;  // another rank's shard
  int rc = choose_lru_mode(h);
  if (rc != FI_OK) return rc;
  if (h->lru_mode == 1) return lru_device_add(h, &endpoint, hashes, false, n, &n, 1, FI_OK);
  rc = check_counters(h);
  if (rc != FI_OK) return rc;
  LruSet& l = h->lrus[e];
  for (uint32_t i = 0; i < n; ++i) {
    uint64_t ev = 0;
    bool did = false;
    const bool inserted = l.touch(hashes[i], &ev, &did);
    if (did) {
      rc = submit_op(h, ev, endpoint, FI_OP_CLEAR);
      if (rc != FI_OK) return rc;
    }
    if (inserted) {
      rc = submit_op(h, hashes[i], endpoint, FI_OP_SET);
      if (rc != FI_OK) return rc;
    }
  }
  // the deltas stay staged: they are launched when the staging buffer fills and, at the latest,
  // by the next pick / sync (one launch group per batch of decisions instead of one per chain)
  return FI_OK;
}

// Upstream PreRequest for a whole batch of decisions: indexer.Add(chain_r, endpoints[r]) for r = 0..R-1, in
// request order per endpoint (the endpoints' LRUs are independent of each other, so they are walked in
// parallel on the host worker pool; the result equals R sequential fi_epp_index_add_chain calls).
int fi_epp_index_add_chains(fi_epp* h, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch_blocks,
                            const uint32_t* nblocks, uint32_t R) {
  if (!h || ((!endpoints || !chains || !nblocks) && R)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  // The LRU depends on configuration and options only, so every rank of a sharded pool runs the same one and takes
  // part in its collective, a rank whose arguments were rejected (err) too.
  const int mode_err = choose_lru_mode(h);
  int err = h->cfg.lru_capacity ? check_add_requests(h, endpoints, nblocks, R, pitch_blocks, "the chain pitch")
                                : fail(h, FI_ERR_STATE, "lru_capacity is 0: the host LRU is disabled");
  if (err == FI_OK) err = mode_err;
  if (h->lru_mode == 1) return lru_device_add(h, endpoints, chains, false, pitch_blocks, nblocks, R, err);
  if (err == FI_OK) err = check_counters(h);

  // bucket the requests by endpoint, walk the LRUs on the worker pool and plan the staging (lru_batch.h)
  std::vector<WorkerOps>& outs = h->lru_outs;  // persistent: capacity survives from batch to batch
  size_t nseg = 0;
  std::vector<StageGroup> groups;
  const auto t_start = std::chrono::steady_clock::now();
  if (!h->pool) {
    unsigned t = std::min(usable_cores(), 128u);
    if (const char* ev = std::getenv("FI_EPP_LRU_THREADS")) t = (unsigned)std::max(1L, std::strtol(ev, nullptr, 10));
    if (h->lru_threads) t = h->lru_threads;
    h->pool.reset(new WorkerPool(t));
  }
  if (err == FI_OK) nseg = lru_walk_batch(h->lrus, h->cfg.endpoint_begin, h->cfg.endpoint_count, endpoints, chains, pitch_blocks, nblocks, R, *h->pool, outs);
  const auto t_walked = std::chrono::steady_clock::now();
  if (err == FI_OK) groups = plan_staging(outs, nseg, h->n_sets, h->n_clears, kOpChunk);

  // Step i copies group i into the staging buffers and flushes it.  A single rank leaves the tail staged: it is
  // launched with the next flush, at the latest by the next pick / sync.  On a sharded pool every group is one gossip
  // round, the tail included.
  struct CopyJob {
    fi_index_op* dst;
    const fi_index_op* src;
    size_t n;
  };
  const int rc = run_rounds(h, groups.size(), err, [&](uint64_t i) -> int {
    const StageGroup& g = groups[i];
    std::vector<CopyJob> jobs;  // big copies into the pinned staging buffers go through the worker pool
    const size_t kPiece = 1u << 16;
    for (const StagePiece& p : g.pieces) {
      const fi_index_op* src = (p.clear ? outs[p.worker].clears : outs[p.worker].sets)[p.seg].data() + p.src;
      fi_index_op* dst = (p.clear ? h->h_clears : h->h_sets)[h->cur_buf].get() + p.dst;
      for (size_t o = 0; o < p.n; o += kPiece) jobs.push_back(CopyJob{dst + o, src + o, std::min(kPiece, p.n - o)});
    }
    h->pool->run((uint32_t)jobs.size(), [&](uint32_t t, unsigned) {
      std::memcpy(jobs[t].dst, jobs[t].src, jobs[t].n * sizeof(fi_index_op));
    });
    h->n_sets = g.n_sets;
    h->n_clears = g.n_clears;
    h->clears_untracked |= g.n_clears > 0;
    return i + 1 < groups.size() || h->world > 1 ? flush_ops(h) : FI_OK;
  });
  if (h->verbose && err == FI_OK) {
    const auto t_end = std::chrono::steady_clock::now();
    size_t nops = 0;
    for (auto& o : outs)
      for (size_t sg = 0; sg < o.nseg; ++sg) nops += o.sets[sg].size() + o.clears[sg].size();
    std::fprintf(stderr, "[fi_epp] add_chains: %u requests, %zu ops, %zu segment(s), %u workers: LRU walk %.2f ms, staging %.2f ms\n",
                 R, nops, nseg, h->pool->size(), std::chrono::duration<double, std::milli>(t_walked - t_start).count(),
                 std::chrono::duration<double, std::milli>(t_end - t_walked).count());
  }
  return rc;
}

// The same with the chains already in device memory (e.g. the chains_out of fi_epp_pick_batch_device): nothing
// but the two small host arrays crosses PCIe.  Device LRU only.
int fi_epp_index_add_chains_device(fi_epp* h, const uint32_t* endpoints, const void* d_chains, uint32_t pitch_blocks,
                                   const uint32_t* nblocks, uint32_t R, void* stream) {
  if (!h || ((!endpoints || !nblocks) && R)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  const int mode_err = choose_lru_mode(h);  // (as in fi_epp_index_add_chains)
  int err = FI_OK;
  if (!h->cfg.lru_capacity) {
    err = fail(h, FI_ERR_STATE, "lru_capacity is 0: no LRU");
  } else if (!d_chains && R > h->last_plain_R) {
    err = fail(h, FI_ERR_STATE, "no pick batch of that size to take the chains from");
  } else {
    if (!d_chains) {  // the chains of the handle's most recent stream-ordered pick, still in its own buffer
      d_chains = h->d_chain.get();
      pitch_blocks = h->MP;
    }
    err = check_add_requests(h, endpoints, nblocks, R, pitch_blocks, "the chain pitch");
  }
  if (err == FI_OK) err = mode_err;
  if (h->lru_mode != 1) return err != FI_OK ? err : fail(h, FI_ERR_STATE, "fi_epp_index_add_chains_device needs the device LRU");
  if (err == FI_OK) {  // the chains were produced on the caller's stream
    FI_CUDA(cudaEventRecord(h->ev_user.get(), (cudaStream_t)stream));
    FI_CUDA(cudaStreamWaitEvent(h->s_index.get(), h->ev_user.get(), 0));
  }
  return lru_device_add(h, endpoints, static_cast<const uint64_t*>(d_chains), true, pitch_blocks, nblocks, R, err);
}

// Diagnostics: the device LRU's content for one endpoint, least recently used first.
int fi_epp_lru_dump(fi_epp* h, uint32_t endpoint, uint64_t* out, uint32_t cap, uint32_t* n_out) {
  if (!h || !n_out || (!out && cap)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  *n_out = 0;
  const uint32_t e = endpoint - h->cfg.endpoint_begin;
  if (e >= h->cfg.endpoint_count) return fail(h, FI_ERR_INVALID, "endpoint outside this handle's shard");
  if (h->lru_mode != 1 || !h->dlru) return h->lru_mode == 0 ? fail(h, FI_ERR_STATE, "the handle runs the host LRU") : FI_OK;
  DevPtr<uint64_t> d_out;
  DevPtr<uint32_t> d_n;
  FI_CUDA(cuda_alloc(d_out, (size_t)h->dlru->v.capacity + 1));
  if (cuda_alloc(d_n, 1) != cudaSuccess) return fail(h, FI_ERR_NOMEM, "cudaMalloc failed");
  uint32_t n = 0;
  FI_CUDA(launch_lru_dump(h->dlru->v, e, d_out.get(), d_n.get(), h->s_index.get()));
  FI_CUDA(cudaMemcpyAsync(&n, d_n.get(), sizeof(n), cudaMemcpyDeviceToHost, h->s_index.get()));
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  if (n) FI_CUDA(cudaMemcpy(out, d_out.get(), (size_t)std::min(n, cap) * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  *n_out = n;
  return FI_OK;
}

// Diagnostics: totals of the device-resident LRU since create — out[0] SETs emitted, [1] CLEARs emitted,
// [2] doomed winners, [3] endpoint maintenance passes, [4] requests deferred to a conservative pass, [5] sub-batches.
int fi_epp_lru_counters(fi_epp* h, uint64_t out[6]) {
  if (!h || !out) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  for (int i = 0; i < 6; ++i) out[i] = 0;
  if (h->lru_mode != 1 || !h->dlru) return FI_OK;
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  out[0] = h->dlru->stat->n_sets;
  out[1] = h->dlru->stat->n_clears;
  out[2] = h->dlru->stat->n_doomed;
  out[3] = h->dlru->stat->n_maintained;
  out[4] = h->lru_deferred;
  out[5] = h->lru_sub_batches;
  return FI_OK;
}

int fi_epp_index_sync(fi_epp* h) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = flush_ops(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  return check_counters(h);
}

int fi_epp_index_stats(fi_epp* h, fi_index_stats* out) {
  if (!h || !out) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = flush_ops(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  IndexCounters c;
  FI_CUDA(cudaMemcpy(&c, h->d_ctr.get(), sizeof(c), cudaMemcpyDeviceToHost));
  out->slots = h->ix.v.C;
  out->used = c.used;
  out->tombstones = c.tombstones;
  out->rebuilds = h->rebuilds;
  out->ops_applied = h->ops_applied;
  uint64_t l = 0;
  if (h->lru_mode == 1 && h->dlru) {
    std::vector<uint32_t> cnt(h->dlru->v.EL);
    FI_CUDA(cudaMemcpy(cnt.data(), h->dlru->v.count, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (uint32_t c2 : cnt) l += c2;
    out->ops_applied += h->dlru->stat->n_sets + h->dlru->stat->n_clears;
  } else {
    for (auto& s : h->lrus) l += s.size();
  }
  out->lru_entries = l;
  return FI_OK;
}

// diagnostics for tests: out[i] = 1 iff (ops[i].endpoint, ops[i].hash) is in the GPU index
int fi_epp_index_contains(fi_epp* h, const fi_index_op* q, uint64_t n, uint8_t* out) {
  if (!h || (!q && n) || (!out && n)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  int rc = flush_ops(h);
  if (rc != FI_OK) return rc;
  if (n == 0) return FI_OK;
  DevPtr<fi_index_op> dq;
  DevPtr<uint8_t> dout;
  FI_CUDA(cuda_alloc(dq, n));
  if (cuda_alloc(dout, n) != cudaSuccess) return fail(h, FI_ERR_NOMEM, "cudaMalloc failed");
  FI_CUDA(cudaMemcpyAsync(dq.get(), q, n * sizeof(fi_index_op), cudaMemcpyHostToDevice, h->s_index.get()));
  {
    LaunchScope ls(h, h->s_index.get(), K_OTHER);
    FI_CUDA(launch_index_contains(h->ix.v, dq.get(), n, h->cfg.endpoint_begin, h->cfg.endpoint_count, dout.get(), h->s_index.get()));
  }
  FI_CUDA(cudaMemcpyAsync(out, dout.get(), n, cudaMemcpyDeviceToHost, h->s_index.get()));
  FI_CUDA(cudaStreamSynchronize(h->s_index.get()));
  return FI_OK;
}

static int check_batch(fi_epp* h, const uint64_t* offsets, uint32_t R, uint64_t* total) {
  if (R > h->cfg.max_batch) return fail(h, FI_ERR_CAPACITY, "batch larger than max_batch");
  if (offsets[0] != 0) return fail(h, FI_ERR_INVALID, "offsets[0] must be 0");
  for (uint32_t r = 0; r < R; ++r)
    if (offsets[r + 1] < offsets[r]) return fail(h, FI_ERR_INVALID, "offsets must be non-decreasing");
  *total = offsets[R];
  if (*total > h->cfg.max_prompt_bytes) return fail(h, FI_ERR_CAPACITY, "prompt bytes larger than max_prompt_bytes");
  return FI_OK;
}

static int stage_inputs(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                        uint64_t total, bool copy_prompts = true) {
  std::memcpy(h->h_offsets.get(), offsets, (size_t)(R + 1) * sizeof(uint64_t));
  std::memcpy(h->h_h0.get(), h0, (size_t)R * sizeof(uint64_t));
  FI_CUDA(cudaMemcpyAsync(h->d_offsets.get(), h->h_offsets.get(), (size_t)(R + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, h->s_main.get()));
  FI_CUDA(cudaMemcpyAsync(h->d_h0.get(), h->h_h0.get(), (size_t)R * sizeof(uint64_t), cudaMemcpyHostToDevice, h->s_main.get()));
  if (total && copy_prompts) {
    FI_CUDA(cudaMemcpyAsync(h->d_prompts.get(), prompts, total, cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += total;
  }
  h->stats.h2d_bytes += (size_t)(2 * R + 1) * sizeof(uint64_t);
  return FI_OK;
}

int fi_epp_hash_batch(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                      uint64_t* chains_out, uint32_t* nblocks_out) {
  if (!h || !offsets || (!h0 && R) || (!prompts && R && offsets[R])) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (R == 0) return FI_OK;
  uint64_t total = 0;
  int rc = check_batch(h, offsets, R, &total);
  if (rc != FI_OK) return rc;
  rc = stage_inputs(h, prompts, offsets, h0, R, total);
  if (rc != FI_OK) return rc;
  rc = claim_chain_slot0(h, h->s_main.get());
  if (rc != FI_OK) return rc;
  h->last_plain_R = 0;  // d_chain no longer holds a pick batch's chains
  rc = run_hash(h, h->d_prompts.get(), h->d_offsets.get(), h->d_h0.get(), 0, R, h->s_main.get(), nullptr);
  if (rc != FI_OK) return rc;
  rc = copy_chains_out(h, h->d_chain.get(), chains_out, R, cudaMemcpyDeviceToHost, h->s_main.get());
  if (rc != FI_OK) return rc;
  if (nblocks_out) {
    FI_CUDA(cudaMemcpyAsync(h->h_nblocks.get(), h->d_nblocks.get(), (size_t)R * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_main.get()));
    h->stats.d2h_bytes += (size_t)R * sizeof(uint32_t);
  }
  FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
  if (nblocks_out) std::memcpy(nblocks_out, h->h_nblocks.get(), (size_t)R * sizeof(uint32_t));
  return FI_OK;
}

// ---- picks: every entry point below is one PickCall through pick_host, pick_device or pick_submit ----------------
// the argument checks of every pick call, before the handle is touched (FI_ERR_INVALID); the ranked entry points, which
// take k >= 1, reject k == 0 themselves
static bool bad_pick_args(const PickCall& c, bool host) {
  return !c.offsets || (!c.h0 && c.R) || (!c.out && !c.counts && (c.R || c.k)) || c.k > FI_EPP_MAX_RANKED ||
         (c.k == 0 && c.subsets) || (host && !c.prompts && c.R && c.offsets[c.R]);
}

// The handle's checks of every pick call, under its lock and before an empty batch returns (a batch over max_batch is
// never empty).  Subset picks are ranked picks (k >= 1) with per-request candidate bitsets, which are pool-wide: a
// handle over part of the pool cannot apply them (FI_ERR_STATE, like a sharded pool).
static int check_pick_handle(fi_epp* h, const PickCall& c) {
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (c.k && h->world > 1) return fail(h, FI_ERR_STATE, "ranked picks need a single-rank pool");
  if (c.counts && h->world > 1) return fail(h, FI_ERR_STATE, "match counts need a single-rank pool");
  if (c.subsets && (h->cfg.endpoint_begin != 0 || h->cfg.endpoint_count != h->cfg.num_endpoints))
    return fail(h, FI_ERR_STATE, "subset picks need a single handle over the whole pool");
  if (c.R > h->cfg.max_batch) return fail(h, FI_ERR_CAPACITY, "batch larger than max_batch");
  return FI_OK;
}

// Host buffers: the inputs are staged through pinned memory (run_pick feeds the prompts), and the picks come back
// through d_picks / h_picks ([R][P]) or the ranked pair ([R][P][k]) before the call returns.
static int pick_host(fi_epp* h, const PickCall& c) {
  if (!h || bad_pick_args(c, true)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = check_pick_handle(h, c);
  if (rc != FI_OK || c.R == 0) return rc;
  const uint32_t R = c.R;
  uint64_t total = 0;
  rc = check_batch(h, c.offsets, R, &total);
  if (rc != FI_OK) return rc;
  PickCall d{h->d_prompts.get(), h->d_offsets.get(), h->d_h0.get(), nullptr, nullptr, R, c.k, h->d_picks.get(), nullptr};  // on device buffers
  fi_pick* h_out = h->h_picks.get();
  if (c.k) {
    // the k-wide result buffers exist only on handles that rank; sized for max_batch so that R does not regrow them
    const size_t need = (size_t)h->cfg.max_batch * h->P * c.k;
    if (need > h->ranked.cap) FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    rc = grow_staging(h, h->ranked, need, need, true);
    if (rc != FI_OK) return rc;
    d.out = h->ranked.d.get();
    h_out = h->ranked.h.get();
  }
  if (c.counts) {
    // the count rows exist only on handles that ask for counts; sized for max_batch rows of the pool as it is now
    const size_t need = (size_t)h->cfg.max_batch * h->cfg.endpoint_count;
    if (need > h->counts.cap) FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    rc = grow_staging(h, h->counts, need, need, true);
    if (rc != FI_OK) return rc;
    d.out = nullptr;
    d.counts = h->counts.d.get();
  }
  rc = stage_inputs(h, c.prompts, c.offsets, c.h0, R, total, /*copy_prompts=*/false);
  if (rc != FI_OK) return rc;
  if (c.adapters) {
    std::memcpy(h->h_adapters.get(), c.adapters, (size_t)R * sizeof(uint64_t));
    FI_CUDA(cudaMemcpyAsync(h->d_adapters.get(), h->h_adapters.get(), (size_t)R * sizeof(uint64_t), cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += (size_t)R * sizeof(uint64_t);
    d.adapters = h->d_adapters.get();
  }
  if (c.subsets) {
    // the bitset staging exists only on handles that restrict picks; sized for max_batch
    const size_t pitch = (h->cfg.num_endpoints + 31) / 32, rows = (size_t)h->cfg.max_batch * pitch;
    rc = grow_staging(h, h->subsets, rows, rows, true);
    if (rc != FI_OK) return rc;
    const size_t sb = (size_t)R * pitch * sizeof(uint32_t);
    std::memcpy(h->subsets.h.get(), c.subsets, sb);
    FI_CUDA(cudaMemcpyAsync(h->subsets.d.get(), h->subsets.h.get(), sb, cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += sb;
    d.subsets = h->subsets.d.get();
  }
  rc = run_pick(h, d, &c);
  if (rc != FI_OK) return rc;
  void* h_res = h_out;
  const void* d_res = d.out;
  size_t pb = (size_t)R * h->P * std::max(c.k, 1u) * sizeof(fi_pick);
  if (c.counts) {
    h_res = h->counts.h.get();
    d_res = d.counts;
    pb = (size_t)R * h->cfg.endpoint_count * sizeof(uint16_t);
  }
  FI_CUDA(cudaMemcpyAsync(h_res, d_res, pb, cudaMemcpyDeviceToHost, h->s_main.get()));
  h->stats.d2h_bytes += pb;
  rc = copy_chains_out(h, h->d_chain.get(), c.chains_out, R, cudaMemcpyDeviceToHost, h->s_main.get());
  if (rc != FI_OK) return rc;
  if (c.nblocks_out) {
    FI_CUDA(cudaMemcpyAsync(h->h_nblocks.get(), h->d_nblocks.get(), (size_t)R * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->s_main.get()));
    h->stats.d2h_bytes += (size_t)R * sizeof(uint32_t);
  }
  FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
  volatile uint32_t* xerr = h->shard ? h->shard->h_xerr.get() : nullptr;
  if (xerr && *xerr) {  // (sharded) reported once; the tags are monotonic, so later steps can succeed again
    *xerr = 0;
    return fail(h, FI_ERR_COMM, "peer exchange timed out waiting for another rank");
  }
  std::memcpy(c.counts ? (void*)c.counts : (void*)c.out, h_res, pb);
  if (c.nblocks_out) std::memcpy(c.nblocks_out, h->h_nblocks.get(), (size_t)R * sizeof(uint32_t));
  return FI_OK;
}

// Device buffers, in the caller's stream order.  The inputs stay where they are: no staging copy and no prompt-bytes
// limit, so the entry points' total_prompt_bytes is not needed.
static int pick_device(fi_epp* h, const PickCall& c, void* stream) {
  if (!h || bad_pick_args(c, false)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  int rc = check_pick_handle(h, c);
  if (rc != FI_OK || c.R == 0) return rc;
  cudaStream_t us = (cudaStream_t)stream;
  FI_CUDA(cudaEventRecord(h->ev_user.get(), us));
  FI_CUDA(cudaStreamWaitEvent(h->s_main.get(), h->ev_user.get(), 0));
  rc = run_pick(h, c, nullptr);
  if (rc != FI_OK) return rc;
  rc = copy_chains_out(h, h->d_chain.get(), c.chains_out, c.R, cudaMemcpyDeviceToDevice, h->s_main.get());
  if (rc != FI_OK) return rc;
  if (c.nblocks_out)
    FI_CUDA(cudaMemcpyAsync(c.nblocks_out, h->d_nblocks.get(), (size_t)c.R * sizeof(uint32_t), cudaMemcpyDeviceToDevice, h->s_main.get()));
  FI_CUDA(cudaEventRecord(h->ev_done.get(), h->s_main.get()));
  FI_CUDA(cudaStreamWaitEvent(us, h->ev_done.get(), 0));
  return FI_OK;
}

// Pipelined submit (docs/SPEC.md S.9): the arguments, checks and output of pick_device, staged through submit_pick.
// Handles that cannot pipeline (sharded pools, block sizes that are not a multiple of 32) run pick_device itself.  Either
// way the batch takes the next ticket.  lagged: the index counters may lag (check_counters_lagged); ticket_empty: an
// empty batch takes a ticket too.
static int pick_submit(fi_epp* h, const PickCall& c, void* stream, uint64_t* ticket, bool lagged, bool ticket_empty) {
  if (!h || bad_pick_args(c, false)) return FI_ERR_INVALID;
  bool plain;
  {
    std::lock_guard<std::mutex> lk(h->mu);
    plain = h->world > 1 || !h->fast_hash;
  }
  uint64_t t = 0;
  int rc;
  if (plain) {
    rc = pick_device(h, c, stream);
    if (rc != FI_OK || (c.R == 0 && !ticket_empty)) return rc;
    std::lock_guard<std::mutex> lk(h->mu);
    rc = issue_ticket(h, &t);  // the batch's number, as a pipelined submit would have given it
  } else {
    std::lock_guard<std::mutex> lk(h->mu);
    rc = check_pick_handle(h, c);
    if (rc != FI_OK || (c.R == 0 && !ticket_empty)) return rc;
    // an empty batch is complete once everything before it is
    rc = c.R ? submit_pick(h, c, (cudaStream_t)stream, &t, lagged) : issue_ticket(h, &t);
  }
  if (rc == FI_OK && ticket) *ticket = t;
  return rc;
}

int fi_epp_pick_batch(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                      fi_pick* out, uint64_t* chains_out) {
  return pick_host(h, PickCall{prompts, offsets, h0, nullptr, nullptr, R, 0, out, chains_out});
}

int fi_epp_pick_batch_lora(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                           const uint64_t* adapters, uint32_t R, fi_pick* out, uint64_t* chains_out) {
  return pick_host(h, PickCall{prompts, offsets, h0, adapters, nullptr, R, 0, out, chains_out});
}

int fi_epp_pick_batch_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                             uint64_t total_prompt_bytes, void* d_out, void* d_chains_out, void* stream) {
  return pick_device(h, device_call(d_prompts, d_offsets, d_h0, nullptr, nullptr, R, 0, d_out, d_chains_out), stream);
}

int fi_epp_pick_batch_device_lora(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                  const void* d_adapters, uint32_t R, uint64_t total_prompt_bytes, void* d_out,
                                  void* d_chains_out, void* stream) {
  return pick_device(h, device_call(d_prompts, d_offsets, d_h0, d_adapters, nullptr, R, 0, d_out, d_chains_out), stream);
}

int fi_epp_pick_batch_ranked(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                             const uint64_t* adapters, uint32_t R, uint32_t k, fi_pick* out, uint64_t* chains_out) {
  if (k == 0) return FI_ERR_INVALID;
  return pick_host(h, PickCall{prompts, offsets, h0, adapters, nullptr, R, k, out, chains_out});
}

int fi_epp_pick_batch_device_ranked(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                    const void* d_adapters, uint32_t R, uint64_t total_prompt_bytes, uint32_t k,
                                    void* d_out, void* d_chains_out, void* stream) {
  if (k == 0) return FI_ERR_INVALID;
  return pick_device(h, device_call(d_prompts, d_offsets, d_h0, d_adapters, nullptr, R, k, d_out, d_chains_out), stream);
}

int fi_epp_pick_batch_subset(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                             const uint64_t* adapters, const uint32_t* subsets, uint32_t R, uint32_t k, fi_pick* out,
                             uint64_t* chains_out) {
  if (k == 0) return FI_ERR_INVALID;
  return pick_host(h, PickCall{prompts, offsets, h0, adapters, subsets, R, k, out, chains_out});
}

int fi_epp_pick_batch_device_subset(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                    const void* d_adapters, const void* d_subsets, uint32_t R,
                                    uint64_t total_prompt_bytes, uint32_t k, void* d_out, void* d_chains_out,
                                    void* stream) {
  if (k == 0) return FI_ERR_INVALID;
  return pick_device(h, device_call(d_prompts, d_offsets, d_h0, d_adapters, d_subsets, R, k, d_out, d_chains_out), stream);
}

int fi_epp_match_counts(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                        uint16_t* counts, uint32_t* nblocks_out, uint64_t* chains_out) {
  if (!counts && R) return FI_ERR_INVALID;
  return pick_host(h, PickCall{prompts, offsets, h0, nullptr, nullptr, R, 0, nullptr, chains_out, counts, nblocks_out});
}

int fi_epp_match_counts_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                               uint64_t total_prompt_bytes, void* d_counts, void* d_nblocks_out, void* d_chains_out,
                               void* stream) {
  if (!d_counts && R) return FI_ERR_INVALID;
  PickCall c = device_call(d_prompts, d_offsets, d_h0, nullptr, nullptr, R, 0, nullptr, d_chains_out);
  c.counts = (uint16_t*)d_counts;
  c.nblocks_out = (uint32_t*)d_nblocks_out;
  return pick_device(h, c, stream);
}

int fi_epp_pick_submit(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                       uint64_t total_prompt_bytes, void* d_out, void* stream) {
  return pick_submit(h, device_call(d_prompts, d_offsets, d_h0, nullptr, nullptr, R, 0, d_out, nullptr), stream, nullptr,
                     /*lagged=*/false, /*ticket_empty=*/false);
}

int fi_epp_pick_submit_ex(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, const void* d_adapters,
                          const void* d_subsets, uint32_t R, uint64_t total_prompt_bytes, uint32_t k, void* d_out,
                          void* d_chains_out, void* stream, uint64_t* ticket) {
  return pick_submit(h, device_call(d_prompts, d_offsets, d_h0, d_adapters, d_subsets, R, k, d_out, d_chains_out), stream,
                     ticket, /*lagged=*/true, /*ticket_empty=*/true);
}

// The pipelined path always runs on the whole GPU: out = {0, 0, 0} (include/fi_epp.h).
int fi_epp_pipeline_info(fi_epp* h, int32_t out[3]) {
  if (!h || !out) return FI_ERR_INVALID;
  out[0] = out[1] = out[2] = 0;
  return FI_OK;
}

int fi_epp_pick_wait(fi_epp* h, void* stream) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  FI_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->ev_pick.get(), 0));  // s_main runs the batches in order
  if (!h->profiling && !h->pending_ev.empty() && h->ev_trace0) {
    h->tracing = true;
    dump_trace(h, 0);
  }
  return FI_OK;
}

int fi_epp_pick_wait_batch(fi_epp* h, uint64_t ticket, void* stream) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (ticket >= h->tickets) return fail(h, FI_ERR_INVALID, "ticket never issued");
  // s_main completes the batches in order: a ticket older than the ring is done by the oldest one it still tracks
  const uint64_t oldest = h->tickets - std::min<uint64_t>(h->tickets, fi_epp::kTicketRing);
  const uint64_t t = std::max(ticket, oldest);
  FI_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, h->ev_ticket[t % fi_epp::kTicketRing].get(), 0));
  if (!h->profiling && !h->pending_ev.empty() && h->ev_trace0) {
    h->tracing = true;
    dump_trace(h, 0);
  }
  return FI_OK;
}

// PreRequest for a submitted batch (docs/SPEC.md S.9): fi_epp_index_add_chains_device(.., NULL, ..) with the chains
// of batch `ticket`, read from its pipeline slot, through the non-stalling device-LRU path (lru_add_submitted).
int fi_epp_index_add_submitted(fi_epp* h, uint64_t ticket, const uint32_t* endpoints, const uint32_t* nblocks,
                               uint32_t R) {
  if (!h || ((!endpoints || !nblocks) && R)) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (ticket >= h->tickets) return fail(h, FI_ERR_INVALID, "ticket never issued");
  if (!h->cfg.lru_capacity) return fail(h, FI_ERR_STATE, "lru_capacity is 0: no LRU");
  if (h->world > 1) return fail(h, FI_ERR_STATE, "sharded pool: use the collective fi_epp_index_add_chains");
  int slot = -1;
  for (int s = 0; s < 2; ++s)
    if (h->slot_ticket[s] == ticket) slot = s;
  if (slot < 0)
    return fail(h, FI_ERR_STATE, "the chains of that batch are gone (two later submits, a stream-ordered pick or hash "
                                 "since, or a batch that was not pipelined)");
  if (R > h->slot_R[slot]) return fail(h, FI_ERR_STATE, "R larger than the submitted batch");
  int rc = check_add_requests(h, endpoints, nblocks, R, h->cfg.max_blocks, "max_blocks");
  if (rc != FI_OK) return rc;
  rc = choose_lru_mode(h);
  if (rc != FI_OK) return rc;
  if (h->lru_mode != 1) return fail(h, FI_ERR_STATE, "fi_epp_index_add_submitted needs the device LRU");
  return lru_add_submitted(h, (uint32_t)slot, endpoints, nblocks, R);
}

int fi_epp_comm_unique_id(uint8_t out[FI_EPP_UNIQUE_ID_BYTES]) {
  if (!out) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  std::string e;
  if (!g_nccl.load(&e)) {
    std::fprintf(stderr, "fi_epp_comm_unique_id: %s\n", e.c_str());
    return FI_ERR_COMM;
  }
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != ncclSuccess) return FI_ERR_COMM;
  static_assert(sizeof(ncclUniqueId) == FI_EPP_UNIQUE_ID_BYTES, "unique id size");
  std::memcpy(out, &id, sizeof(id));
  return FI_OK;
}

int fi_epp_comm_init(fi_epp* h, const uint8_t id_bytes[FI_EPP_UNIQUE_ID_BYTES], uint32_t rank, uint32_t world) {
  if (!h || !id_bytes || world == 0 || rank >= world) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (h->shard) return fail(h, FI_ERR_STATE, "communicator already initialised");
  // the sharded pick is tested only with chains that fit one match window (DESIGN.md §4.9)
  if (h->cfg.max_blocks > 1023) return fail(h, FI_ERR_STATE, "sharded pools need max_blocks <= 1023");
  if (world > 32) return fail(h, FI_ERR_INVALID, "more than 32 ranks: the directory keeps one presence bit per rank");
  if (h->ops_applied || h->n_sets || h->n_clears)
    return fail(h, FI_ERR_STATE, "fi_epp_comm_init must precede the first index update (the directory is built by gossip)");
  if (world == 1) {
    h->rank = 0;
    h->world = 1;
    return FI_OK;
  }
  {
    std::lock_guard<std::mutex> lk2(g_nccl_mu);
    std::string e;
    if (!g_nccl.load(&e)) return fail(h, FI_ERR_COMM, e);
  }
  // the shard state is built whole before the handle takes it: a failed call leaves a single-rank handle
  auto sh = std::make_unique<ShardState>();
  ncclUniqueId id;
  std::memcpy(&id, id_bytes, sizeof(id));
  int rc = g_nccl.CommInitRank(&sh->comm, (int)world, id, (int)rank);
  if (rc != ncclSuccess) {
    sh->comm = nullptr;
    return fail(h, FI_ERR_COMM, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"));
  }
  const uint64_t R = h->cfg.max_batch;
  FI_CUDA(cuda_alloc(sh->d_local, R * h->P));
  FI_CUDA(cuda_alloc(sh->d_gather, (size_t)world * R * h->P));
  FI_CUDA(cuda_alloc(sh->d_glog_n, 2));
  FI_CUDA(cudaMemset(sh->d_glog_n.get(), 0, 2 * sizeof(unsigned long long)));
  FI_CUDA(cuda_alloc(sh->d_glog_a, kOpChunk));
  FI_CUDA(cuda_alloc(sh->d_glog_v, kOpChunk));
  FI_CUDA(cuda_alloc(sh->d_ghdr, (size_t)(world + 1) * 2));
  FI_CUDA(cuda_alloc(sh->h_ghdr, (size_t)(world + 1) * 2));
  FI_CUDA(cuda_alloc(sh->d_ggather, (size_t)world * kOpChunk));
  PeerXchg px{};
  rc = setup_peer_exchange(h, *sh, rank, world, &px);
  if (rc != FI_OK) return rc;
  h->shard = std::move(sh);
  h->px = px;
  h->rank = rank;
  h->world = world;
  return FI_OK;
}

int fi_epp_comm_exchange(fi_epp* h) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (h->world <= 1) return FI_EXCHANGE_NONE;
  return h->px.enabled ? FI_EXCHANGE_PEER : FI_EXCHANGE_NCCL;
}

int fi_epp_set_option(fi_epp* h, const char* name, int64_t value) {
  if (!h || !name) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  const std::string n(name);
  if (n == "exchange") {
    if (h->world <= 1) return fail(h, FI_ERR_STATE, "exchange: not a sharded pool");
    if (value == FI_EXCHANGE_NCCL) {
      h->px.enabled = 0;
    } else if (value == FI_EXCHANGE_PEER) {
      if (!h->px.base[h->rank == 0 ? 1 : 0]) return fail(h, FI_ERR_STATE, "exchange: the peers' buffers were never mapped");
      h->px.enabled = 1;
    } else {
      return fail(h, FI_ERR_INVALID, "exchange: FI_EXCHANGE_PEER or FI_EXCHANGE_NCCL");
    }
    return FI_OK;
  }
  if (n == "shard_hash") {
    h->split_hash = value != 0;
    return FI_OK;
  }
  if (n == "feed_slices") {
    if (value < 1 || value > fi_epp::kMaxFeedSlices) return fail(h, FI_ERR_INVALID, "feed_slices: 1..16");
    h->feed_slices = (uint32_t)value;
    return FI_OK;
  }
  if (n == "device_lru") {
    if (value != 0 && value != 1) return fail(h, FI_ERR_INVALID, "device_lru: 0 or 1");
    if (h->lru_mode >= 0 && h->lru_mode != (int)value) return fail(h, FI_ERR_STATE, "device_lru: the handle's LRU is already in use");
    h->lru_want = (int)value;
    return FI_OK;
  }
  if (n == "lru_table_slots") {
    if (value < 0 || value > (1ll << 30)) return fail(h, FI_ERR_INVALID, "lru_table_slots: 0 .. 2^30");
    if (h->dlru) return fail(h, FI_ERR_STATE, "lru_table_slots: the device LRU is already allocated");
    h->lru_table_slots = (uint32_t)value;
    return FI_OK;
  }
  if (n == "lru_threads") {
    if (value < 1 || value > 1024) return fail(h, FI_ERR_INVALID, "lru_threads: 1..1024");
    h->lru_threads = (unsigned)value;
    h->pool.reset();
    return FI_OK;
  }
  return fail(h, FI_ERR_INVALID, "unknown option: " + n);
}

int fi_epp_set_profiling(fi_epp* h, int on) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  cudaSetDevice(h->cfg.device);
  drain_profile(h);
  h->profiling = on != 0;
  return FI_OK;
}

int fi_epp_get_stats(fi_epp* h, fi_epp_stats* out) {
  if (!h || !out) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  drain_profile(h);
  if (h->profiling) {
    FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    unsigned long long pb[8] = {0};
    FI_CUDA(cudaMemcpy(pb, h->d_probed.get(), sizeof(pb), cudaMemcpyDeviceToHost));
    h->stats.probed_blocks = pb[0];
    h->stats.hashed_blocks = pb[6];
    if (pb[5] && h->verbose)  // FI_MATCH_TIMING build: where a request's time goes inside match_pick
      std::fprintf(stderr, "[fi_epp] match_pick phases, cycles per request over %llu requests: stage %.0f, first lookup %.0f, "
                   "chunks %.0f, score+pick %.0f\n", pb[5], (double)pb[1] / pb[5], (double)pb[2] / pb[5], (double)pb[3] / pb[5],
                   (double)pb[4] / pb[5]);
  }
  *out = h->stats;
  return FI_OK;
}

int fi_epp_reset_stats(fi_epp* h) {
  if (!h) return FI_ERR_INVALID;
  std::lock_guard<std::mutex> lk(h->mu);
  cudaSetDevice(h->cfg.device);
  drain_profile(h);
  cudaStreamSynchronize(h->s_main.get());
  cudaMemset(h->d_probed.get(), 0, 8 * sizeof(unsigned long long));
  h->stats = fi_epp_stats{};
  return FI_OK;
}

}  // extern "C"
