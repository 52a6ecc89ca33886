// engine.cu — host side of libfi_epp: the C ABI of include/fi_epp.h.  This file holds the handle's lifetime and
// options, its endpoint and score tables, its statistics and the pool resize; engine.h lists the files that hold the
// rest.
//
// A handle owns the device buffers, four CUDA streams (compute, index maintenance, prompt copies, pipelined hashing),
// the pinned op ring that keeps the GPU index live (async H2D on the side stream, ordered before the next pick), the
// host LRU, the per-batch score tables, and the optional NCCL communicator for endpoint-range sharded pools.  No CPU
// fallback: creation fails without a CUDA device.
#include <cmath>

#include "engine.h"
#include "xxh64.cuh"

namespace {

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

// The endpoint and score tables of a pool of E endpoints and rows of W words into `out`, all or nothing: `out` is left
// as it was on failure.  All but eps, which is uploaded before its first read (eps_dirty), start zeroed (on s_index).
int alloc_endpoint_tables(fi_epp* h, uint32_t E, uint32_t W, EndpointTables& out) {
  const size_t Epad = (size_t)W * 32, n_sc = FI_EPP_MAX_PROFILES * FI_EPP_MAX_SCORERS * Epad, n_bits = (size_t)FI_EPP_MAX_PROFILES * W;
  EndpointTables t;
  cudaError_t e = cuda_alloc(t.eps, E);
  if (e == cudaSuccess) e = cuda_alloc(t.sc, n_sc);
  if (e == cudaSuccess) e = cuda_alloc(t.elig, n_bits);
  if (e == cudaSuccess) e = cuda_alloc(t.ztie, n_bits);
  if (e == cudaSuccess) e = cuda_alloc(t.lora, Epad);
  if (e != cudaSuccess) return fail(h, alloc_status(e), std::string("endpoint tables: ") + cudaGetErrorString(e));
  cudaStream_t si = h->s_index.get();
  FI_CUDA(cudaMemsetAsync(t.sc.get(), 0, n_sc * sizeof(double), si));
  FI_CUDA(cudaMemsetAsync(t.elig.get(), 0, n_bits * sizeof(uint32_t), si));
  FI_CUDA(cudaMemsetAsync(t.ztie.get(), 0, n_bits * sizeof(uint32_t), si));
  FI_CUDA(cudaMemsetAsync(t.lora.get(), 0, Epad * sizeof(LoraDev), si));
  out = std::move(t);
  return FI_OK;
}

// point the handle's ScoreTables at h->ept, for rows of h->W words
void use_endpoint_tables(fi_epp* h) {
  h->st.Epad = h->W * 32;
  h->st.sc = h->ept.sc.get();
  h->st.elig = h->ept.elig.get();
  h->st.ztie = h->ept.ztie.get();
  h->st.lora = h->ept.lora.get();
}

// The host LRU sets of the local endpoints, empty, endpoint x's limited to caps[x] (which becomes h->lru_caps).  One
// virtual reservation backs them all: an endpoint's tables become resident when it is first touched.
void reset_host_lrus(fi_epp* h, std::vector<uint32_t> caps) {
  const uint32_t C = h->cfg.lru_capacity;
  h->lrus.clear();  // (first: the reservation releases the arena the old sets took their tables from)
  LruArena* arena = h->lru_arena.reserve(caps.size() * LruSet::bytes_needed(C)) ? &h->lru_arena : nullptr;
  h->lrus = std::vector<LruSet>(caps.size(), LruSet(C, arena));
  for (size_t x = 0; x < caps.size(); ++x)
    if (caps[x] != C) h->lrus[x].shrink(caps[x], [](uint64_t) {});
  h->lru_caps = std::move(caps);
}

}  // namespace

namespace fi::engine {

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

// Wait for all four streams of h; the first error, if any, fails the call once every stream has been waited for.
int sync_all_streams(fi_epp* h) {
  cudaError_t first = cudaSuccess;
  for (cudaStream_t s : {h->s_main.get(), h->s_index.get(), h->s_copy.get(), h->s_a.get()}) {
    const cudaError_t e = cudaStreamSynchronize(s);
    if (first == cudaSuccess) first = e;
  }
  if (first != cudaSuccess) return fail(h, FI_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(first));
  return FI_OK;
}

// The rule of the calls that work on the pool as a whole (resize, snapshots, subset picks): a single-rank handle over
// every endpoint.  `what` names the call in the message.
int check_whole_pool(fi_epp* h, const char* what) {
  if (h->world > 1) return fail(h, FI_ERR_STATE, std::string("sharded pool: ") + what + " needs a single-rank handle");
  if (h->cfg.endpoint_begin != 0 || h->cfg.endpoint_count != h->cfg.num_endpoints)
    return fail(h, FI_ERR_STATE, std::string(what) + " needs a handle over the whole pool");
  return FI_OK;
}

// A replacement of the index and the device LRU (fi_epp_resize_pool, fi_epp_snapshot_load) is one update in three
// steps.  replace_begin: every call before it completes first, picks in flight included.  Then the caller allocates
// the new tables, before anything of the handle changes, and fills them on s_index.  replace_commit swaps them in.
int replace_begin(fi_epp* h) {
  int rc = update_begin(h);
  if (rc != FI_OK) return rc;
  return sync_all_streams(h);
}

// The new index `nix` (null: the index stays) and device LRU `nlru` (null: none, or it stays) take the place of the
// handle's, the device LRU's statistics carry over, and with an LRU the host LRU sets take the capacities `caps`.  The
// old tables go back to the caller's owners, which free them after the update is done: the call returns when s_index
// has drained.
int replace_commit(fi_epp* h, IndexTables* nix, std::unique_ptr<DevLruStore>& nlru, std::vector<uint32_t>& caps) {
  cudaStream_t si = h->s_index.get();
  if (nlru && h->dlru) {  // the statistics keep counting
    FI_CUDA(cudaMemcpyAsync(nlru->ctr.get(), h->dlru->ctr.get(), 8 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, si));
    *nlru->stat = *h->dlru->stat;
  }
  if (nlru) FI_CUDA(cudaEventRecord(nlru->ev.get(), si));
  if (nix) {
    std::swap(h->ix, *nix);
    h->ix_spare.reset();  // a later rebuild allocates it in the new shape
  }
  h->cfg.index_slots = h->ix.v.C;
  if (nlru) std::swap(h->dlru, nlru);
  if (h->cfg.lru_capacity) reset_host_lrus(h, std::move(caps));
  int rc = update_end(h);
  if (rc != FI_OK) return rc;
  FI_CUDA(cudaStreamSynchronize(si));
  return FI_OK;
}

}  // namespace fi::engine

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
  sync_all_streams(h);  // (an error changes nothing: the handle goes)
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
      return die(alloc_status(e__));                                    \
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
  if (cfg->lru_capacity) reset_host_lrus(h, std::vector<uint32_t>(cfg->endpoint_count, cfg->lru_capacity));

  // endpoints + score tables
  h->eps.assign(cfg->num_endpoints, EndpointDev{0.0, 0, 0, 0, 0});
  {
    int rc = alloc_endpoint_tables(h, cfg->num_endpoints, h->W, h->ept);
    if (rc != FI_OK) return die(rc);
  }
  use_endpoint_tables(h);
  FI_TRY(cuda_alloc(h->d_zero, FI_EPP_MAX_PROFILES));
  h->st.n_profiles = h->P;
  h->st.zero = h->d_zero.get();
  h->lora.assign(h->st.Epad, LoraDev{});
  FI_TRY(cuda_alloc(h->d_adapters, R));
  FI_TRY(cuda_alloc(h->h_adapters, R));
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
  int rc = check_whole_pool(h, "fi_epp_resize_pool");
  if (rc != FI_OK) return rc;
  if (h->lru_mode == 0) return fail(h, FI_ERR_STATE, "fi_epp_resize_pool: the host LRU serves the handle");
  if (En == E) return FI_OK;
  rc = replace_begin(h);
  if (rc != FI_OK) return rc;
  // The slot floor counts the live keys before a shrink's removal: an upper bound of those after it, known before
  // anything changes.
  IndexCounters ctr;
  FI_CUDA(cudaMemcpy(&ctr, h->d_ctr.get(), sizeof(ctr), cudaMemcpyDeviceToHost));
  const uint32_t Wn = pool_row_words(En), keep = std::min(E, En);
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
  EndpointTables ept;
  rc = alloc_endpoint_tables(h, En, Wn, ept);
  if (rc != FI_OK) return rc;
  cudaStream_t si = h->s_index.get();

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
  // the new ones start empty (alloc_dev_lru), and the totals carry over (replace_commit)
  if (nlru) {
    const DevLru& o = h->dlru->v;
    const DevLru& n = nlru->v;
    FI_CUDA(cudaMemcpyAsync(n.slots, o.slots, (size_t)keep * (o.TS + 2) * sizeof(LruSlot), cudaMemcpyDeviceToDevice, si));
    FI_CUDA(cudaMemcpyAsync(n.log, o.log, (size_t)keep * o.L * sizeof(uint64_t), cudaMemcpyDeviceToDevice, si));
    const std::pair<uint32_t*, const uint32_t*> arrays[] = {{n.head, o.head}, {n.tail, o.tail},   {n.count, o.count}, {n.used, o.used},
                                                            {n.hold, o.hold}, {n.dcount, o.dcount}, {n.ovf, o.ovf}};
    for (const auto& a : arrays) FI_CUDA(cudaMemcpyAsync(a.first, a.second, (size_t)keep * sizeof(uint32_t), cudaMemcpyDeviceToDevice, si));
    FI_CUDA(cudaMemcpyAsync(n.any_ovf, o.any_ovf, 2 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, si));  // any_ovf, error
  }

  // ---- swap in the new pool (the old buffers stay allocated until the work above is done)
  h->W = Wn;
  h->eps.resize(keep);
  h->eps.resize(En, EndpointDev{0.0, 0, 0, 0, 0});
  h->lora.resize(keep);
  h->lora.resize(Wn * 32, LoraDev{});
  std::swap(h->ept, ept);
  use_endpoint_tables(h);
  h->eps_dirty = h->lora_dirty = true;
  // lazily created buffers sized by the pool: their next use allocates them anew
  h->d_rm.reset();
  h->subsets = Staging<uint32_t>{};
  h->lists = fi_epp::ListScratch{};
  h->lru_plan_buf = Staging<uint32_t>{};
  h->lru_resize = Staging<uint32_t>{};
  for (fi_epp::PipeAdd& pa : h->padd) pa.plan = Staging<uint32_t>{};
  h->cfg.num_endpoints = h->cfg.endpoint_count = En;
  // (no Add has run through the host LRUs, lru_mode != 0: they are empty and only carry the capacities)
  return replace_commit(h, rebuild ? &nix : nullptr, nlru, caps);
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
