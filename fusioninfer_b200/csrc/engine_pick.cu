// engine_pick.cu — the pick paths: block hashing, the match enqueue, the stream-ordered and pipelined picks, match
// counts and match lists, and their entry points in the C ABI.
#include "engine.h"

namespace {

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

// One pick call of any variant: the single pick (k == 0), the ranked pick (k > 0, docs/SPEC.md S.6a) and the subset
// pick (subsets, S.5a), each with or without LoRA adapters.  Host or device pointers, by entry point.
struct PickCall {
  const uint8_t* prompts = nullptr;
  const uint64_t* offsets = nullptr;   // [R + 1]
  const uint64_t* h0 = nullptr;        // [R]
  const uint64_t* adapters = nullptr;  // [R] adapter ids, or null
  const uint32_t* subsets = nullptr;   // [R][ceil(E/32)] candidate bitsets, or null
  uint32_t R = 0;
  uint32_t k = 0;                      // 0: out is [R][P]; else [R][P][k]
  fi_pick* out = nullptr;
  uint64_t* chains_out = nullptr;      // [R][max_blocks], or null
  // match counts (S.3a) instead of picks: out is null, counts [R][endpoint_count]; nblocks_out [R] or null
  uint16_t* counts = nullptr;
  uint32_t* nblocks_out = nullptr;
  // match lists (S.3b) instead of picks: out and counts are null; list_offsets [R + 1], entries [cap].  The match writes
  // the handle's list scratch, and run_pick's pack step fills these (the host call's copy-out has entries null).
  uint64_t* list_offsets = nullptr;
  fi_match_entry* entries = nullptr;
  uint64_t cap = 0;
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
    FI_CUDA(cudaMemcpyAsync(h->ept.eps.get(), h->eps.data(), h->eps.size() * sizeof(EndpointDev), cudaMemcpyHostToDevice, h->s_main.get()));
    h->stats.h2d_bytes += h->eps.size() * sizeof(EndpointDev);
    LaunchScope ls(h, h->s_main.get(), K_OTHER);
    FI_CUDA(launch_prepare_endpoints(h->ept.eps.get(), h->cfg.num_endpoints, h->cfg.endpoint_begin, h->cfg.endpoint_count, h->st,
                                     h->ept.sc.get(), h->ept.elig.get(), h->d_zero.get(), h->ept.ztie.get(), h->s_main.get()));
    h->eps_dirty = false;  // (eps is pageable host memory: the copy has been staged by the time it returns)
  }
  if (h->lora_dirty) {
    FI_CUDA(cudaMemcpyAsync(h->ept.lora.get(), h->lora.data(), h->lora.size() * sizeof(LoraDev), cudaMemcpyHostToDevice, h->s_main.get()));
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
  if (c.list_offsets) {
    mp.lists = h->lists.slots.get();
    mp.nnz = h->lists.nnz.get();
  }
  if (c.subsets) {
    mp.subsets = c.subsets;
    mp.sub_pitch = (h->cfg.num_endpoints + 31) / 32;
    mp.eps = h->ept.eps.get();
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
      ms.lists = mp.lists ? mp.lists + (size_t)r0 * h->cfg.endpoint_count : nullptr;  // the slices' own slots
      ms.nnz = mp.nnz ? mp.nnz + r0 : nullptr;
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

// The pack step of match lists (S.3b), behind the match launches on s_main: the offsets, then the entries below c.cap
int pack_lists(fi_epp* h, const PickCall& c) {
  {
    LaunchScope ls(h, h->s_main.get(), K_OTHER);
    FI_CUDA(launch_list_scan(h->lists.nnz.get(), c.R, c.list_offsets, h->s_main.get()));
  }
  if (c.cap && c.entries) {
    LaunchScope ls(h, h->s_main.get(), K_OTHER);
    FI_CUDA(launch_list_copy(h->lists.slots.get(), h->cfg.endpoint_count, c.list_offsets, c.R, h->cfg.endpoint_begin, 0,
                             c.cap, c.entries, h->s_main.get()));
  }
  return FI_OK;
}

int run_pick(fi_epp* h, const PickCall& c, const PickCall* feed) {
  int rc = run_pick_impl(h, c, feed);
  if (rc == FI_OK && c.list_offsets) rc = pack_lists(h, c);
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

}  // namespace

extern "C" {

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
  return !c.offsets || (!c.h0 && c.R) || (!c.out && !c.counts && !c.list_offsets && (c.R || c.k)) || c.k > FI_EPP_MAX_RANKED ||
         (c.cap && !c.entries) ||
         (c.k == 0 && c.subsets) || (host && !c.prompts && c.R && c.offsets[c.R]);
}

// The handle's checks of every pick call, under its lock and before an empty batch returns (a batch over max_batch is
// never empty).  Subset picks are ranked picks (k >= 1) with per-request candidate bitsets, which are pool-wide: a
// handle over part of the pool cannot apply them (FI_ERR_STATE, like a sharded pool).
static int check_pick_handle(fi_epp* h, const PickCall& c) {
  if (cudaSetDevice(h->cfg.device) != cudaSuccess) return fail(h, FI_ERR_CUDA, "cudaSetDevice failed");
  if (c.k && h->world > 1) return fail(h, FI_ERR_STATE, "ranked picks need a single-rank pool");
  if (c.counts && h->world > 1) return fail(h, FI_ERR_STATE, "match counts need a single-rank pool");
  if (c.list_offsets && h->world > 1) return fail(h, FI_ERR_STATE, "match lists need a single-rank pool");
  if (c.subsets) {
    const int rc = check_whole_pool(h, "a subset pick");
    if (rc != FI_OK) return rc;
  }
  if (c.R > h->cfg.max_batch) return fail(h, FI_ERR_CAPACITY, "batch larger than max_batch");
  return FI_OK;
}

// The list scratch for max_batch requests of the pool as it is, its slots and counts together or neither (the first
// lists call, and the first after a resize); a scratch in use by queued work is replaced only after s_main drains.
static int alloc_list_scratch(fi_epp* h) {
  const size_t need = (size_t)h->cfg.max_batch * h->cfg.endpoint_count;
  if (h->lists.slots && need <= h->lists.cap) return FI_OK;
  FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
  h->lists = fi_epp::ListScratch{};
  fi_epp::ListScratch t;
  cudaError_t e = cuda_alloc(t.slots, need);
  if (e == cudaSuccess) e = cuda_alloc(t.nnz, h->cfg.max_batch);
  if (e != cudaSuccess) {
    alloc_status(e);
    return fail(h, FI_ERR_NOMEM, "cannot allocate the match-list scratch of " + std::to_string(need * 4) + " bytes");
  }
  t.cap = need;
  h->lists = std::move(t);
  return FI_OK;
}

// The host lists call after its offsets have arrived: the first min(total, cap) entries, at most kListChunk per copy
// through list_chunk; FI_ERR_CAPACITY when the total exceeds cap.
static int copy_out_lists(fi_epp* h, const PickCall& c) {
  const uint64_t total = c.list_offsets[c.R], n = std::min(total, c.cap);
  for (uint64_t lo = 0; lo < n; lo += kListChunk) {
    const uint64_t hi = std::min(n, lo + kListChunk);
    int rc = grow_staging(h, h->list_chunk, hi - lo, std::min(n, kListChunk), true);
    if (rc != FI_OK) return rc;
    {
      LaunchScope ls(h, h->s_main.get(), K_OTHER);
      FI_CUDA(launch_list_copy(h->lists.slots.get(), h->cfg.endpoint_count, h->list_offsets.d.get(), c.R,
                               h->cfg.endpoint_begin, lo, hi, h->list_chunk.d.get(), h->s_main.get()));
    }
    const size_t bytes = (size_t)(hi - lo) * sizeof(fi_match_entry);
    FI_CUDA(cudaMemcpyAsync(h->list_chunk.h.get(), h->list_chunk.d.get(), bytes, cudaMemcpyDeviceToHost, h->s_main.get()));
    h->stats.d2h_bytes += bytes;
    FI_CUDA(cudaStreamSynchronize(h->s_main.get()));
    std::memcpy(c.entries + lo, h->list_chunk.h.get(), bytes);
  }
  if (total > c.cap) return fail(h, FI_ERR_CAPACITY, "match lists: " + std::to_string(total) + " entries, cap " + std::to_string(c.cap));
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
  if (c.list_offsets) {  // the offsets come back here; the entries after them, once their total is known
    rc = alloc_list_scratch(h);
    if (rc == FI_OK) rc = grow_staging(h, h->list_offsets, (size_t)h->cfg.max_batch + 1, (size_t)h->cfg.max_batch + 1, true);
    if (rc != FI_OK) return rc;
    d.out = nullptr;
    d.list_offsets = h->list_offsets.d.get();
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
  if (c.list_offsets) {
    h_res = h->list_offsets.h.get();
    d_res = d.list_offsets;
    pb = (size_t)(R + 1) * sizeof(uint64_t);
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
  std::memcpy(c.list_offsets ? (void*)c.list_offsets : c.counts ? (void*)c.counts : (void*)c.out, h_res, pb);
  if (c.nblocks_out) std::memcpy(c.nblocks_out, h->h_nblocks.get(), (size_t)R * sizeof(uint32_t));
  if (c.list_offsets) return copy_out_lists(h, c);
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
  if (c.list_offsets) {
    rc = alloc_list_scratch(h);
    if (rc != FI_OK) return rc;
  }
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

int fi_epp_match_lists(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                       uint64_t* list_offsets, fi_match_entry* entries, uint64_t cap, uint32_t* nblocks_out,
                       uint64_t* chains_out) {
  if (!list_offsets && R) return FI_ERR_INVALID;
  PickCall c{prompts, offsets, h0, nullptr, nullptr, R, 0, nullptr, chains_out, nullptr, nblocks_out};
  c.list_offsets = list_offsets;
  c.entries = entries;
  c.cap = cap;
  const int rc = pick_host(h, c);
  if (rc == FI_OK && R == 0 && list_offsets) list_offsets[0] = 0;
  return rc;
}

int fi_epp_match_lists_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                              uint64_t total_prompt_bytes, void* d_list_offsets, void* d_entries, uint64_t cap,
                              void* d_nblocks_out, void* d_chains_out, void* stream) {
  if (!d_list_offsets && R) return FI_ERR_INVALID;
  PickCall c = device_call(d_prompts, d_offsets, d_h0, nullptr, nullptr, R, 0, nullptr, d_chains_out);
  c.nblocks_out = (uint32_t*)d_nblocks_out;
  c.list_offsets = (uint64_t*)d_list_offsets;
  c.entries = (fi_match_entry*)d_entries;
  c.cap = cap;
  const int rc = pick_device(h, c, stream);
  if (rc == FI_OK && R == 0 && d_list_offsets && cudaMemsetAsync(d_list_offsets, 0, sizeof(uint64_t), (cudaStream_t)stream) != cudaSuccess)
    return fail(h, FI_ERR_CUDA, std::string("cudaMemsetAsync: ") + cudaGetErrorString(cudaGetLastError()));
  return rc;
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

}  // extern "C"
