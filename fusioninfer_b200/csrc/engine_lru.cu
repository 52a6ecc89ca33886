// engine_lru.cu — the two LRUs behind indexer.Add: the host LRU (lru.h, lru_batch.h) and the device-resident LRU
// (lru_kernels.cu), their capacities, and the Add entry points of the C ABI.
#include <chrono>

#include "engine.h"

namespace {

uint32_t pow2_ceil32(uint32_t v) {
  uint32_t p = 1;
  while (p < v) p <<= 1;
  return p;
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

}  // namespace

namespace fi::engine {

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

}  // namespace fi::engine

extern "C" {

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

}  // extern "C"
