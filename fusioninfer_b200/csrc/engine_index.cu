// engine_index.cu — the ordering rule of index updates (engine.h), the staging of index ops, the directory gossip of
// sharded pools, and the index entry points of the C ABI.
#include "engine.h"

namespace {

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

}  // namespace

namespace fi::engine {

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
  if (e != cudaSuccess) return fail(h, alloc_status(e), std::string("index allocation: ") + cudaGetErrorString(e));
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

// queue the copy of the index counters that the next check_counters reads
int read_counters(fi_epp* h) {
  FI_CUDA(cudaMemcpyAsync(h->h_ctr.get(), h->d_ctr.get(), sizeof(IndexCounters), cudaMemcpyDeviceToHost, h->s_index.get()));
  FI_CUDA(cudaEventRecord(h->ev_ctr.get(), h->s_index.get()));
  h->ctr_pending = true;
  return FI_OK;
}

int settle_updates(fi_epp* h, bool lagged, uint64_t extra) {
  int rc = flush_ops(h);
  if (rc != FI_OK) return rc;
  return lagged ? check_counters_lagged(h, extra) : check_counters(h);
}

int update_begin(fi_epp* h, Settle settle, uint64_t extra) {
  int rc = FI_OK;
  if (settle == Settle::kAll || settle == Settle::kLagged) rc = settle_updates(h, settle == Settle::kLagged, extra);
  if (settle == Settle::kCheck) rc = check_counters(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamWaitEvent(h->s_index.get(), h->ev_pick.get(), 0));
  return FI_OK;
}

// done (optional) is recorded behind the update's work and copies, before ev_index
int update_end(fi_epp* h, Readback rb, cudaEvent_t done) {
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

}  // namespace fi::engine

extern "C" {

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

}  // extern "C"
