/*
 * fi_epp.h — C ABI of the H100-native prefix-cache-aware Endpoint Picker.
 *
 * This is the drop-in boundary for the ONE hot path this repo implements
 * (BASELINE.json north_star; SURVEY.md §8): per request, hash the prompt into
 * chained fixed-size block keys, look the chain up against every candidate
 * endpoint's cached-prefix set, combine the match length with KV-cache /
 * queue load into a weighted fp64 score, and argmax to choose a pod.
 *
 * What it replaces.  FusionInfer (the reference, /root/reference) does not
 * contain this loop: its router role only *configures and deploys* the
 * Gateway-API-Inference-Extension EPP image
 *   pkg/router/epp.go:46        DefaultEPPImage  …/epp:v1.2.1
 *   pkg/router/epp.go:125-129   args --pool-name --pool-namespace --config-file
 *   pkg/router/strategy.go:51-68,115-165  the EndpointPickerConfig YAML
 * and the loop itself runs inside that image (upstream Go packages
 * pkg/epp/scheduling/framework/plugins/{multi/prefix,scorer,picker}).  There
 * is no cgo/FFI in the reference (Dockerfile:24 builds CGO_ENABLED=0), so the
 * entry points below are shaped after the upstream plugin seams a Go EPP
 * would bind through cgo:
 *
 *   upstream seam (Go, module sigs.k8s.io/gateway-api-inference-extension v1.2.1,
 *   go.mod:16)                                      → entry point here
 *   ------------------------------------------------------------------------
 *   config loader for the YAML of strategy.go:52-67 → fi_epp_config_from_yaml
 *   prefix.Plugin hashPrompt (xxhash chain)         → fi_epp_hash_batch
 *   prefix indexer.Add / LRU eviction (PreRequest)  → fi_epp_index_add_chains (a batch
 *                                                     of decisions), fi_epp_index_add_chain,
 *                                                     fi_epp_index_apply
 *   prefix autoTune (LRU sized per pod from its     → fi_epp_set_lru_capacities
 *   KV-cache block count)
 *   datastore pod metrics refresh (kv, queue, role) → fi_epp_endpoints_update
 *   SchedulerProfile.Run: filter → scorers → picker → fi_epp_pick_batch
 *   prefix.Plugin.Score alone (matchLen / total per  → fi_epp_match_counts (the host runs
 *   pod; the other plugins run in the framework)       the rest of any config)
 *   pd-profile-handler (decode then prefill)        → fi_epp_pick_batch with
 *                                                     cfg.pd_enabled
 *
 * Conventions (cgo-safe): every function returns 0 (FI_OK) or a negative
 * fi_status; nothing throws across the ABI; the caller owns every buffer and
 * no pointer is retained after a call returns; one fi_epp handle is internally
 * serialised by a mutex (concurrency comes from batching); calls on different
 * handles may run concurrently, also on handles of one device; library threads
 * never call back into the host language.  fi_epp_last_error is the message of
 * the handle's latest failing call, and is not meaningful while other threads
 * use the handle (read the status instead).  There is NO CPU fallback: without
 * a CUDA device fi_epp_create fails with FI_ERR_CUDA.
 *
 * Ties.  Upstream's MaxScorePicker shuffles the candidates before its stable sort, i.e. equal totals are
 * resolved at random (SURVEY.md Appendix A.5).  Here the order among endpoints with equal totals is a rotation
 * of the pool that starts at a position derived from the request, so that picks are reproducible (and
 * bit-comparable with the CPU oracle) yet spread over the tied pods the way upstream's shuffle does:
 *     seed  = n_blocks > 0 ? h_1 (the first chained block hash) : h0[r] ^ (r + 1) * 0x9E3779B97F4A7C15
 *     x     = seed;  x ^= x >> 30;  x *= 0xBF58476D1CE4E5B9;  x ^= x >> 27;  x *= 0x94D049BB133111EB;  x ^= x >> 31
 *     start = ((x >> 32) * num_endpoints) >> 32
 *     among equal totals the endpoint with the smallest (endpoint - start) mod num_endpoints wins
 * (r = index of the request within the call).
 */
#ifndef FI_EPP_H_
#define FI_EPP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FI_EPP_ABI_VERSION 2u
#define FI_EPP_MAX_PROFILES 4u
#define FI_EPP_MAX_SCORERS 4u
#define FI_EPP_MAX_FILTERS 4u /* by-label filters per profile */
#define FI_EPP_MAX_LABELS 24u /* (label, value) pairs a configuration can filter on */
#define FI_EPP_MAX_BLOCKS 4095u /* counts are kept in 12 bit-planes on the GPU.  A handle with max_blocks > 1023
                                 * serves every single-rank call; fi_epp_comm_init refuses it (FI_ERR_STATE). */
#define FI_NO_ENDPOINT 0xFFFFFFFFu
#define FI_EPP_UNIQUE_ID_BYTES 128u

typedef enum fi_status {
  FI_OK = 0,
  FI_ERR_INVALID = -1,  /* bad argument / config */
  FI_ERR_CUDA = -2,     /* CUDA runtime error, or no device (there is no CPU fallback) */
  FI_ERR_NOMEM = -3,
  FI_ERR_CAPACITY = -4, /* batch, prompt bytes or index larger than configured */
  FI_ERR_STATE = -5,
  FI_ERR_COMM = -6,     /* NCCL / peer-memory error */
  FI_ERR_CONFIG = -7    /* EndpointPickerConfig YAML rejected */
} fi_status;

/* SURVEY.md Appendix A.3.  UPSTREAM: stop at the first block no endpoint holds,
 * count per endpoint the blocks it holds before that.  LPM: per-endpoint longest
 * contiguous prefix.  Identical whenever every endpoint's set is prefix-closed. */
typedef enum fi_match_mode { FI_MATCH_UPSTREAM = 0, FI_MATCH_LPM = 1 } fi_match_mode;

/* plugin `type:` names of pkg/router/strategy.go:55,74,89,104 */
typedef enum fi_scorer_kind {
  FI_SCORER_PREFIX = 1,  /* prefix-cache-scorer          */
  FI_SCORER_KV_UTIL = 2, /* kv-cache-utilization-scorer  */
  FI_SCORER_QUEUE = 3,   /* queue-scorer                 */
  FI_SCORER_LORA = 4     /* lora-affinity-scorer         */
} fi_scorer_kind;

/* Label bits of an endpoint (fi_endpoint_state.role_mask) — what the by-label filters of strategy.go:135-144
 * test.  The three `fusioninfer.io/component-type` values (api/core/v1alpha1/inferenceservice_types.go:26-33)
 * have fixed bits; any other (label, value) pair a configuration filters on is given one of the bits from
 * FI_ROLE_FIRST_FREE up by fi_epp_config_from_yaml, which records the assignment in fi_epp_config.labels —
 * the host sets that bit on every pod carrying the label value when it calls fi_epp_endpoints_update. */
#define FI_ROLE_WORKER 1u
#define FI_ROLE_PREFILLER 2u
#define FI_ROLE_DECODER 4u
#define FI_ROLE_FIRST_FREE 8u

#define FI_ENDPOINT_ALIVE 1u

typedef struct fi_scorer {
  uint32_t kind;  /* fi_scorer_kind */
  int32_t weight; /* `weight:` of the pluginRef (strategy.go:66,157,163); >= 0 */
} fi_scorer;

typedef struct fi_profile {
  char name[32];      /* schedulingProfiles[].name */
  uint32_t role_mask; /* first by-label filter (0: none): the endpoint must carry one of these label bits */
  uint32_t n_scorers;
  fi_scorer scorers[FI_EPP_MAX_SCORERS]; /* in profile order: fp64 accumulation order */
  /* further by-label filters of the profile.  Filters chain like upstream's filter plugins: an endpoint is
   * eligible iff it is alive and passes EVERY filter f, i.e. (ep.role_mask & f) != 0. */
  uint32_t n_more_filters;
  uint32_t more_filters[FI_EPP_MAX_FILTERS - 1];
} fi_profile;

/* One (label, value) pair of a by-label filter and the endpoint bit that stands for it. */
typedef struct fi_label_bit {
  char label[64]; /* e.g. "fusioninfer.io/component-type" */
  char value[56]; /* one of the filter's validValues */
  uint32_t bit;   /* single bit of fi_endpoint_state.role_mask */
  uint32_t reserved;
} fi_label_bit;

typedef struct fi_epp_config {
  uint32_t struct_size; /* sizeof(fi_epp_config), checked */
  uint32_t abi_version; /* FI_EPP_ABI_VERSION */
  int32_t device;       /* CUDA ordinal */
  uint32_t block_bytes; /* blockSize | hashBlockSize (strategy.go:57,147); 64 = 16 u32 tokens */
  uint32_t max_blocks;  /* maxPrefixBlocksToMatch (strategy.go:58,148) */
  uint32_t lru_capacity; /* lruCapacityPerServer (strategy.go:59,149); 0: no LRU (fi_epp_index_add_chain* fail) */
  uint32_t num_endpoints;  /* global pool size E */
  uint32_t endpoint_begin; /* this handle's shard [begin, begin+count) of the pool.  Without fi_epp_comm_init such a
                            * handle indexes, learns and picks only its own endpoints, with the queue scorer's min /
                            * max and the tie rotation of the whole pool (docs/SPEC.md S.2e) */
  uint32_t endpoint_count;
  uint32_t match_mode; /* fi_match_mode */
  uint32_t max_batch;  /* largest R accepted by one pick/hash call */
  uint32_t reserved0;
  uint64_t max_prompt_bytes; /* largest total prompt bytes per call (device staging) */
  uint64_t index_slots;      /* key slots of the GPU index, power of two; 0 = 2x num_endpoints*lru_capacity (load <= 0.5: a shard
                              * is a directory of the whole pool's keys, with membership rows for its own endpoints) */
  uint32_t n_profiles;
  uint32_t pd_enabled;        /* pd-profile-handler present (strategy.go:129-133) */
  uint32_t pd_decode_profile; /* profile index run first */
  uint32_t pd_prefill_profile;
  double pd_threshold;        /* `threshold:` — prefill runs iff (1-hit)*len(prompt) >= threshold */
  fi_profile profiles[FI_EPP_MAX_PROFILES];
  /* written by fi_epp_config_from_yaml, read by the host: which role_mask bit each filtered (label, value) has */
  uint32_t n_labels;
  uint32_t reserved1;
  fi_label_bit labels[FI_EPP_MAX_LABELS];
} fi_epp_config;

/* One row of the pod datastore the scorers read (upstream metrics refresh). */
typedef struct fi_endpoint_state {
  uint32_t endpoint;   /* global index in [0, num_endpoints) */
  uint32_t role_mask;  /* FI_ROLE_* */
  double kv_util;      /* KVCacheUsagePercent in [0,1] */
  int32_t queue_depth; /* WaitingQueueSize */
  uint32_t flags;      /* FI_ENDPOINT_ALIVE */
} fi_endpoint_state;

/* LoRA adapters resident / queued on one endpoint (upstream pod metrics ActiveModels,
 * WaitingModels, MaxActiveModels) — read by the lora-affinity-scorer
 * (pkg/router/strategy.go:100-113).  Adapter ids are any 64-bit ids the host uses
 * consistently, e.g. fi_epp_model_seed(adapter name). */
#define FI_EPP_MAX_LORA 8u
typedef struct fi_endpoint_lora {
  uint32_t endpoint;   /* global index */
  uint32_t max_active; /* MaxActiveModels */
  uint32_t n_active;   /* <= FI_EPP_MAX_LORA */
  uint32_t n_waiting;  /* <= FI_EPP_MAX_LORA */
  uint64_t active[FI_EPP_MAX_LORA];
  uint64_t waiting[FI_EPP_MAX_LORA];
} fi_endpoint_lora;

typedef enum fi_index_opcode { FI_OP_SET = 1, FI_OP_CLEAR = 2 } fi_index_opcode;

/* One membership change of the logical index {(endpoint, block hash)}. */
typedef struct fi_index_op {
  uint64_t hash;
  uint32_t endpoint; /* global index */
  uint32_t op;       /* fi_index_opcode */
} fi_index_op;

/* One routing decision (16 bytes). */
typedef struct fi_pick {
  uint32_t endpoint;     /* global index, or FI_NO_ENDPOINT */
  uint16_t match_blocks; /* prefix blocks matched at the picked endpoint */
  uint16_t n_blocks;     /* blocks hashed for this request */
  double score;          /* weighted fp64 total of the picked endpoint */
} fi_pick;

/* One matched endpoint of a request's match list (fi_epp_match_lists, 8 bytes). */
typedef struct fi_match_entry {
  uint32_t endpoint;     /* global index */
  uint16_t match_blocks; /* > 0 */
  uint16_t reserved;     /* written as 0 */
} fi_match_entry;

typedef struct fi_index_stats {
  uint64_t slots;      /* key slots */
  uint64_t used;       /* slots holding a key or a tombstone */
  uint64_t tombstones; /* keys whose row became empty */
  uint64_t rebuilds;
  uint64_t ops_applied;
  uint64_t lru_entries; /* entries of the per-endpoint LRUs (device-resident or host), summed */
} fi_index_stats;

typedef struct fi_epp_stats {
  uint64_t kernel_launches; /* kernels of this library launched since create/reset */
  uint64_t pick_calls;
  uint64_t requests;
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  /* per-kernel device time, accumulated only while profiling is on.  Block hashing and the chain walk (one
   * kernel) are reported entirely under *_hash_blocks; the *_chain_probe fields stay 0. */
  double ms_hash_blocks, ms_chain_probe, ms_match_pick, ms_index_apply, ms_other;
  uint64_t n_hash_blocks, n_chain_probe, n_match_pick, n_index_apply, n_other;
  uint64_t probed_blocks; /* sum over requests of N_probe (SURVEY.md §8d), profiling only */
  uint64_t hashed_blocks; /* blocks whose prompt bytes were read, summed over requests; profiling only, counted when
                           * block_bytes % 32 == 0.  A pick without chains_out on a single-rank handle with
                           * lru_capacity == 0 stops hashing each request after its first block the index does not
                           * hold, so it reads fewer blocks than its requests' n_blocks */
} fi_epp_stats;

typedef struct fi_epp fi_epp;

uint32_t fi_epp_abi_version(void);
const char* fi_epp_status_string(int status);

/* Fill cfg with the defaults of generatePrefixCacheConfig (strategy.go:51-68)
 * except block_bytes = 64 (16 uint32 tokens, SURVEY.md §8d). */
int fi_epp_config_default(fi_epp_config* cfg);

/* Parse an EndpointPickerConfig YAML document (exactly the schema
 * strategy.go:52-67,126-164 emits, plus custom passthrough strategy.go:29-31)
 * into cfg's plugin-derived fields (block_bytes, max_blocks, lru_capacity,
 * profiles, pd_*).  Deployment fields (device, endpoints, sizes) are untouched.
 * On FI_ERR_CONFIG a message is written to err (NUL-terminated, truncated). */
int fi_epp_config_from_yaml(const char* yaml, size_t len, fi_epp_config* cfg, char* err, size_t err_len);

/* Widest ranked pick (fi_epp_pick_batch_ranked): a max-score-picker may ask for this many endpoints per profile. */
#define FI_EPP_MAX_RANKED 16u
/* maxNumOfEndpoints of the max-score-picker each profile references, in the profile order
 * fi_epp_config_from_yaml produces (1 when absent); entries past the document's profiles are 0.  FI_ERR_CONFIG for
 * a value that is not an integer in [1, FI_EPP_MAX_RANKED], and for everything fi_epp_config_from_yaml rejects
 * (which itself does not look at maxNumOfEndpoints). */
int fi_epp_config_picker_endpoints(const char* yaml, size_t len, uint32_t out[FI_EPP_MAX_PROFILES], char* err,
                                   size_t err_len);

int fi_epp_create(const fi_epp_config* cfg, fi_epp** out);
void fi_epp_destroy(fi_epp* h);
const char* fi_epp_last_error(const fi_epp* h);

/* h0 = XXH64(seed 0, model ‖ salt): the chain seed of SURVEY.md Appendix A.1. */
int fi_epp_model_seed(const void* model, size_t model_len, const void* salt, size_t salt_len, uint64_t* h0);

/* Replace the state of the listed endpoints (every rank receives the whole
 * pool: queue min/max are global).  Unlisted endpoints keep their state;
 * endpoints never listed are not alive. */
int fi_epp_endpoints_update(fi_epp* h, const fi_endpoint_state* states, uint32_t n);

/* Adapter residency of the listed endpoints (lora-affinity-scorer).  Endpoints never listed
 * hold no adapter and have max_active 0. */
int fi_epp_endpoints_lora_update(fi_epp* h, const fi_endpoint_lora* states, uint32_t n);

/* Asynchronous, ordered: every op submitted before a pick call is visible to
 * that pick.  Ops for endpoints outside this handle's shard are ignored.
 *
 * Sharded pools (after fi_epp_comm_init with world > 1): every rank's index is a directory of the WHOLE pool's
 * block hashes — membership rows only for its own endpoints — so that "the first block no pod holds" (where
 * upstream's matchLongestPrefix stops) is a local lookup.  The owner of an endpoint applies its ops and the
 * resulting key appear/vanish transitions are exchanged between the ranks inside this call: index updates of
 * a sharded pool are COLLECTIVE — every rank calls fi_epp_index_apply / fi_epp_index_add_chains the same
 * number of times in the same order, each with its own ops (possibly none). */
int fi_epp_index_apply(fi_epp* h, const fi_index_op* ops, uint64_t n);

/* upstream indexer.RemovePod: forget everything the index and the LRU hold for the listed endpoints (pod deleted,
 * restarted with an empty KV cache, or its index about to be reused for a new pod).  Every (endpoint, hash) pair
 * leaves the index, whether an Add or a direct SET put it there; keys no endpoint holds any more leave with it; the
 * endpoints' LRUs become empty (a later Add inserts anew).  Endpoint state (fi_epp_endpoints_update) is untouched.
 * Duplicates and endpoints that hold nothing are no-ops.  Asynchronous and ordered like fi_epp_index_apply: ops
 * submitted before the call are applied first, picks called before it (in-flight fi_epp_pick_submit batches
 * included) do not see the removal, every later pick does.  pairs_removed != NULL: block until applied and write
 * how many (endpoint, hash) pairs left the index.  FI_ERR_INVALID if an endpoint is >= num_endpoints (nothing is
 * applied); FI_ERR_STATE on a sharded pool. */
int fi_epp_index_remove_endpoints(fi_epp* h, const uint32_t* endpoints, uint32_t n, uint64_t* pairs_removed);

/* Resize the pool of a single-rank handle over the whole pool to num_endpoints endpoints (docs/SPEC.md S.2c), keeping
 * what the kept endpoints [0, min(E, num_endpoints)) have cached.  Afterwards the handle behaves exactly like one
 * created with num_endpoints = endpoint_count = num_endpoints and everything else the same, fed the same calls, except
 * that everything ever addressed to an endpoint a shrink dropped is left out of that history, and that index_slots
 * stays as given at create (0: the default, now computed for the new pool, but never below what the live keys need).
 *   Shrink: endpoints [num_endpoints, E) leave the pool; their pairs leave the index as fi_epp_index_remove_endpoints
 *   removes them, and their state, adapters, LRUs and LRU capacities are forgotten.  pairs_removed != NULL receives
 *   how many (endpoint, hash) pairs left.
 *   Grow: endpoints [E, num_endpoints) are new: not alive, no adapters, max_active 0, an empty LRU of capacity
 *   lru_capacity.  An endpoint a shrink dropped comes back this way.
 *   The kept endpoints keep their index pairs, LRU contents and recency order, capacities, states and adapters.  The
 *   tie rotation, the subset row width (ceil(num_endpoints / 32) words), every endpoint range check and the queue
 *   scorer's min / max follow the new pool from the next call on.  num_endpoints == E is a no-op.
 * Blocking: every call issued before it completes on the device against the old pool (fi_epp_pick_submit batches in
 * flight and staged index ops included), every later call sees the new pool.  Tickets stay valid; the chains a ticket
 * holds are not released, and fi_epp_index_add_submitted checks the ticket's endpoints against the new pool.  Errors
 * change nothing: FI_ERR_INVALID if num_endpoints is 0 or above 4096; FI_ERR_STATE on a sharded pool, on a handle over
 * part of the pool, or on a handle the host LRU already serves (before the first Add both LRUs stay ready for the
 * new pool); FI_ERR_NOMEM if the new tables do not fit (everything is allocated before anything changes, so the old
 * and the new tables are both held while the call runs). */
int fi_epp_resize_pool(fi_epp* h, uint32_t num_endpoints, uint64_t* pairs_removed);

/* Index snapshots (docs/SPEC.md S.2d): what a handle has learned — every (endpoint, hash) pair of the index, whatever
 * put it there, every endpoint's LRU in recency order, and every endpoint's LRU capacity — as a device-independent byte
 * blob in host memory, so that a restarted picker (or a new replica) starts warm.  Endpoint states and adapters are
 * not part of it: the caller re-sends them after a load, as after create.  The blob format (version 1, little-endian)
 * is part of the ABI: fusioninfer_b200/csrc/snapshot_format.h and S.2d lay it out.  A blob of another format version
 * is refused, never guessed at.  (The header's struct has no typedef: its tag names it, and the plain name is the
 * function fi_epp_snapshot_info.) */
struct fi_epp_snapshot_info {
  uint32_t block_bytes, max_blocks, lru_capacity, num_endpoints;
  uint64_t n_nodes; /* keys in the index */
  uint64_t n_lru;   /* LRU entries, summed over the endpoints */
  uint64_t pairs;   /* (endpoint, hash) pairs: the total popcount of the rows */
  uint64_t bytes;   /* 64 + payload bytes */
};

/* Write h's learned state to buf.  buf == NULL: *bytes = the size the snapshot needs, FI_OK.  cap < that size:
 * FI_ERR_CAPACITY, *bytes = the size, nothing written.  Blocking: every call issued before it (staged ops, Adds,
 * removals, capacity changes, fi_epp_pick_submit batches in flight) is applied first; the handle is not changed.  The
 * index's live nodes are written in node order (insertion order), so a load numbers a cached prefix's nodes
 * consecutively again.  buf is ordinary pageable memory of any size; it is filled through bounded pinned staging.
 * FI_ERR_STATE on a sharded pool, on a handle over part of the pool, or on a handle the host LRU serves. */
int fi_epp_snapshot_save(fi_epp* h, void* buf, uint64_t cap, uint64_t* bytes);

/* Snapshot captures (docs/SPEC.md S.2d): a snapshot taken on the device at a point in h's call order, copied out
 * later without h, so that periodic saves do not stall the serving loop.  Owned by the library. */
typedef struct fi_epp_capture fi_epp_capture;

/* Take a snapshot of h on the device.  *bytes = the size of its blob, *out = the capture.  Point in time: every call
 * issued on h before it is in the blob (staged ops, stream-ordered and fi_epp_index_add_submitted Adds, removals,
 * capacity changes, resizes, loads); no later call is.  It does not wait for pick batches in flight, and later picks
 * do not wait for it; later index updates run after its device work, in s_index order.  It holds h only to flush the
 * staged ops, for one synchronisation of the index stream (the sizes), to allocate the device image (one buffer of
 * the payload size, held until fi_epp_snapshot_free) and to queue the export.  Errors leave *out NULL, allocate
 * nothing and leave h unchanged: FI_ERR_INVALID for NULL arguments; FI_ERR_STATE as for fi_epp_snapshot_save;
 * FI_ERR_NOMEM if the image does not fit on the device (fi_epp_snapshot_save, which needs only bounded staging, is
 * the fallback). */
int fi_epp_snapshot_capture(fi_epp* h, fi_epp_capture** out, uint64_t* bytes);

/* Write the capture's blob to buf: exactly the bytes fi_epp_snapshot_save would have written had it been called in
 * place of fi_epp_snapshot_capture.  Never takes or touches the handle, so it may run on any thread while others use
 * h, and after fi_epp_resize_pool, fi_epp_snapshot_load or fi_epp_destroy(h).  Blocks until the device image is
 * complete; buf is ordinary pageable memory, filled through bounded pinned staging; the checksum is computed on host
 * threads.  Repeatable: every read gives the same bytes.  cap < the blob's size: FI_ERR_CAPACITY, nothing written.
 * FI_ERR_STATE (nothing written) if the device LRU's invariant was found broken, as the save reports it.  Calls on one
 * capture must not overlap. */
int fi_epp_snapshot_read(fi_epp_capture* c, void* buf, uint64_t cap);

/* Release a capture (NULL: no-op).  Allowed while its device work still runs, with or without a read, and after h is
 * destroyed; it does not stall h's streams. */
void fi_epp_snapshot_free(fi_epp_capture* c);

/* Replace h's index, LRUs and LRU capacities with the snapshot's.  h must have the block_bytes, max_blocks,
 * lru_capacity and num_endpoints of the handle that saved it; its index_slots, LRU table size and device may differ.
 * Afterwards h behaves exactly like the saved handle at the moment of the save, for every later call sequence, except
 * that h keeps its own endpoint states and adapters, and its statistics (ops_applied, rebuilds, fi_epp_lru_counters,
 * fi_epp_get_stats) keep counting; fi_epp_index_stats' used and lru_entries describe the loaded state, without
 * tombstones.  Before the first Add, the call allocates the device LRU as the first Add would.
 * Blocking, ordered like fi_epp_resize_pool: every call issued before it completes against the old state (staged ops and
 * fi_epp_pick_submit batches in flight included), every later call sees the loaded state.  Tickets stay valid:
 * fi_epp_index_add_submitted of an earlier ticket adds its chains to the loaded state.
 * Errors change nothing (new tables are built and checked, then swapped in): FI_ERR_INVALID for a blob that is not
 * well-formed (S.2d; duplicate keys are found on the device while building) or whose block_bytes, max_blocks,
 * lru_capacity or num_endpoints differ from h's; FI_ERR_CAPACITY if the keys exceed 60 % of an index_slots given at
 * create (with index_slots 0 the index grows as fi_epp_resize_pool grows it); FI_ERR_STATE as for
 * fi_epp_snapshot_save; FI_ERR_NOMEM if the old and new tables do not fit together. */
int fi_epp_snapshot_load(fi_epp* h, const void* buf, uint64_t len);

/* No handle, no device: check a blob's structure (everything S.2d asks except that keys are distinct) and read its
 * header into *out.  FI_ERR_INVALID if it is not well-formed. */
int fi_epp_snapshot_info(const void* buf, uint64_t len, struct fi_epp_snapshot_info* out);

/* Per-endpoint LRU capacities (docs/SPEC.md S.2b; upstream's autoTune sizes a pod's LRU from the KV-cache blocks the
 * pod reports).  Every endpoint's LRU capacity starts at lru_capacity; this sets it to capacities[i] for endpoints[i]
 * (0 = lru_capacity; the last entry of an endpoint listed twice wins).  An LRU that holds more keys than its new
 * capacity evicts its least recently used ones down to it, and each evicted (endpoint, hash) pair leaves the index,
 * as an eviction inside an Add does; raising a capacity evicts nothing.  Every later Add (fi_epp_index_add_submitted
 * of an earlier ticket included) evicts against the new capacity.  fi_epp_index_remove_endpoints empties an LRU but
 * keeps its capacity.  Ordered like fi_epp_index_apply: ops and removals submitted before the call are applied first,
 * picks called before it (in-flight fi_epp_pick_submit batches included) do not see its evictions, every later pick
 * does.  Asynchronous, except that a call which LOWERS a capacity on a handle served by the device LRU blocks: it
 * reads back the LRUs' entry counts to plan its evictions, and so waits for the index updates queued before it (and
 * for the picks those wait for).  Endpoints of other shards are ignored; n = 0 is a no-op.  entries_evicted != NULL:
 * block until applied and write how many LRU entries were evicted.  Errors apply nothing: FI_ERR_INVALID if an
 * endpoint is >= num_endpoints, a capacity is above lru_capacity, or a non-zero capacity is below max_blocks;
 * FI_ERR_STATE if lru_capacity is 0 or the pool is sharded.  Capacities set before the first Add apply to whichever
 * LRU (device or host) serves the handle. */
int fi_epp_set_lru_capacities(fi_epp* h, const uint32_t* endpoints, const uint32_t* capacities, uint32_t n,
                              uint64_t* entries_evicted);

/* Upstream indexer.Add(hashes, pod): touch each hash in `endpoint`'s LRU
 * (capacity lru_capacity, or the endpoint's own from fi_epp_set_lru_capacities), emit SET for new entries and CLEAR
 * for evicted ones.  Requires lru_capacity > 0.  Single-rank handles only (FI_ERR_STATE on a sharded pool). */
int fi_epp_index_add_chain(fi_epp* h, uint32_t endpoint, const uint64_t* hashes, uint32_t n);

/* The same for a whole batch of routing decisions — upstream's PreRequest step after a pick batch:
 * indexer.Add(chains[r*pitch_blocks .. +nblocks[r]), endpoints[r]) for r = 0..R-1 (FI_NO_ENDPOINT and
 * endpoints of other shards are skipped).  Equal to R fi_epp_index_add_chain calls in request order.  With the
 * device-resident LRU (the default, see below) the chains are copied to the GPU and the whole batch is applied
 * by a handful of kernels; with the host LRU the endpoints' LRUs are walked in parallel on host worker threads
 * (FI_EPP_LRU_THREADS, default = usable cores, at most 128).  `chains` / `nblocks` are what fi_epp_pick_batch
 * returned (chains_out, picks' n_blocks).  Collective on a sharded pool. */
int fi_epp_index_add_chains(fi_epp* h, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch_blocks,
                            const uint32_t* nblocks, uint32_t R);

/* The same with the chains already in device memory — the chains_out of fi_epp_pick_batch_device, written on
 * `stream` — so that only the two small host arrays cross PCIe.  Served by the device-resident LRU
 * (fusioninfer_b200/csrc/lru_kernels.cu), which is also what fi_epp_index_add_chain(s) use on a handle with
 * lru_capacity >= max_blocks (sharded pools included) unless fi_epp_set_option(h, "device_lru", 0) / FI_EPP_DEVICE_LRU=0
 * selected the host LRU before the first Add; FI_ERR_STATE when the handle runs the host LRU.
 * d_chains == NULL: the chains of this handle's most recent fi_epp_pick_batch / fi_epp_pick_batch_device call,
 * read from the handle's own buffer (pitch_blocks ignored; R <= that call's R) — the PreRequest step right after
 * a pick, with nothing but the decisions crossing PCIe. */
int fi_epp_index_add_chains_device(fi_epp* h, const uint32_t* endpoints, const void* d_chains, uint32_t pitch_blocks,
                                   const uint32_t* nblocks, uint32_t R, void* stream);

/* Diagnostics: the keys of `endpoint` in the device-resident LRU, least recently used first (at most `cap`
 * written, *n_out = how many it holds).  FI_ERR_STATE when the handle runs the host LRU. */
int fi_epp_lru_dump(fi_epp* h, uint32_t endpoint, uint64_t* out, uint32_t cap, uint32_t* n_out);

/* Diagnostics: totals of the device-resident LRU since create — out[0] SETs emitted, [1] CLEARs emitted, [2] keys
 * touched but gone again by the end of their batch, [3] per-endpoint maintenance passes (log compaction + table
 * rebuild), [4] requests deferred to a conservative pass (their endpoint's table could not take the batch's new
 * keys), [5] sub-batches run. */
int fi_epp_lru_counters(fi_epp* h, uint64_t out[6]);

int fi_epp_index_sync(fi_epp* h); /* block until submitted ops are applied */

/* Diagnostics: out[i] = 1 iff (q[i].endpoint, q[i].hash) is in this handle's GPU index. */
int fi_epp_index_contains(fi_epp* h, const fi_index_op* q, uint64_t n, uint8_t* out);
int fi_epp_index_stats(fi_epp* h, fi_index_stats* out);

/* Hash only.  prompts: concatenated prompt bytes; offsets: R+1 byte offsets;
 * h0: R chain seeds.  chains_out: R*max_blocks hashes (row r holds
 * nblocks_out[r] valid entries); either output may be NULL. */
int fi_epp_hash_batch(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                      uint32_t R, uint64_t* chains_out, uint32_t* nblocks_out);

/* The hot path, host buffers (pinned memory from fi_epp_pinned_alloc avoids a
 * staging copy).  out: R*n_profiles picks, out[r*n_profiles + p] for profile p.
 * With pd_enabled the prefill profile's pick is FI_NO_ENDPOINT when the
 * threshold test skips it.  chains_out optional (R*max_blocks). */
int fi_epp_pick_batch(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                      uint32_t R, fi_pick* out, uint64_t* chains_out);

/* Same, every buffer already in device memory of cfg.device; work is ordered
 * after `stream` (a cudaStream_t, may be NULL) and `stream` waits for it. */
int fi_epp_pick_batch_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                             uint32_t R, uint64_t total_prompt_bytes, void* d_out, void* d_chains_out,
                             void* stream);

/* The same two calls with one target adapter id per request (lora-affinity-scorer: 1.0 if the
 * adapter is active on the endpoint, 0.8 if the endpoint has room for another adapter, 0.6 if it
 * is queued there, else 0).  adapters == NULL means "no adapter" (id 0) for every request. */
int fi_epp_pick_batch_lora(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                           const uint64_t* adapters, uint32_t R, fi_pick* out, uint64_t* chains_out);
int fi_epp_pick_batch_device_lora(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                  const void* d_adapters, uint32_t R, uint64_t total_prompt_bytes, void* d_out,
                                  void* d_chains_out, void* stream);

/* Ranked picks: upstream max-score-picker with maxNumOfEndpoints = k.  For each request and profile the profile's
 * eligible endpoints ordered by total descending, then by the request's tie rotation ("Ties" above) — the order
 * whose first entry is the pick of fi_epp_pick_batch, bit for bit.  Each entry carries the endpoint's own
 * match_blocks and fp64 total; fewer than k eligible endpoints: the tail is FI_NO_ENDPOINT, match 0, score 0.  With
 * pd_enabled the threshold test uses the decode profile's entry 0, and a skipped prefill profile's whole list is
 * FI_NO_ENDPOINT.  A profile's top k_p is the first k_p entries of its top k, so one call with k = max_p k_p (see
 * fi_epp_config_picker_endpoints) serves profiles with different limits.
 * out: R*n_profiles*k picks, out[(r*n_profiles + p)*k + j] = rank j of profile p.  1 <= k <= FI_EPP_MAX_RANKED
 * (else FI_ERR_INVALID); adapters may be NULL (as fi_epp_pick_batch_lora); FI_ERR_STATE on a sharded pool.
 * Otherwise they behave like fi_epp_pick_batch_lora / fi_epp_pick_batch_device_lora: the same staging, chains_out,
 * ordering against index updates, removals and pipelined submits, and fi_epp_index_add_chains_device(.., NULL, ..)
 * afterwards adds this call's chains. */
int fi_epp_pick_batch_ranked(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                             const uint64_t* adapters, uint32_t R, uint32_t k, fi_pick* out, uint64_t* chains_out);
int fi_epp_pick_batch_device_ranked(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                    const void* d_adapters, uint32_t R, uint64_t total_prompt_bytes, uint32_t k,
                                    void* d_out, void* d_chains_out, void* stream);

/* Subset picks: the ranked pick with a per-request candidate subset (the data plane's destination-endpoint subset
 * hint, docs/SPEC.md S.5a).  subsets: R rows of ceil(num_endpoints / 32) uint32 words; bit e%32 of word e/32 of
 * row r set means endpoint e is a candidate for request r.  A request without a hint has every bit set; an empty
 * hint is an all-zero row; bits at or above num_endpoints are ignored.  Only eligible candidates are ranked, and
 * the queue scorer's min / max are taken over each request's eligible candidates.  The prefix walk stays pool-wide
 * (it stops at the first block no endpoint of the pool holds), and so does the tie rotation.  A request and
 * profile without an eligible candidate gets FI_NO_ENDPOINT (match 0, score 0) in every entry.
 * subsets == NULL: every request is unrestricted, and the result is byte-identical to fi_epp_pick_batch_ranked.
 * k and out as fi_epp_pick_batch_ranked (k = 1 is the single pick over the subset, [R][P] layout).  Everything else
 * as the ranked calls: arguments, errors, staging, chains_out, ordering against index updates, removals and
 * pipelined submits, fi_epp_index_add_chains_device(.., NULL, ..) afterwards.  Non-NULL subsets on a handle that
 * covers only part of the pool (endpoint_begin / endpoint_count) or on a sharded pool: FI_ERR_STATE.  The host call
 * stages the bitsets in a buffer allocated by its first call with subsets (max_batch rows). */
int fi_epp_pick_batch_subset(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                             const uint64_t* adapters, const uint32_t* subsets, uint32_t R, uint32_t k,
                             fi_pick* out, uint64_t* chains_out);
int fi_epp_pick_batch_device_subset(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                                    const void* d_adapters, const void* d_subsets, uint32_t R,
                                    uint64_t total_prompt_bytes, uint32_t k, void* d_out, void* d_chains_out,
                                    void* stream);

/* Match counts: the prefix-cache-scorer on its own (docs/SPEC.md S.3a), for a configuration whose other plugins run on
 * the host (a picker, filter or scorer this library does not implement).  counts[r*endpoint_count + j] = the number
 * of prefix blocks of request r that local endpoint endpoint_begin + j holds, in the handle's match mode: S.3's
 * match[e], the match_blocks every pick of any variant would report for that endpoint on the same index.  It ignores
 * endpoint state, adapters, profiles, filters and PD: the host filters after the call and scores counts / n_blocks.
 * counts is dense [R][endpoint_count] uint16 with no row padding (any 2-byte aligned pointer); nblocks_out [R]
 * (optional) = the requests' n_blocks; chains_out (optional) as fi_epp_pick_batch's.  A handle over part of the pool
 * returns its own columns with the shard-local walk of S.2e.  Ordered and counted like the stream-ordered picks:
 * every index update issued before the call is seen, it is a pick call in fi_epp_stats and for the chain retention of
 * fi_epp_index_add_submitted, and fi_epp_index_add_chains_device(.., NULL, ..) afterwards adds this call's chains (the
 * PreRequest step after the host's own pick).  Errors write nothing: FI_ERR_INVALID for a NULL handle, offsets, h0 or
 * counts with R > 0; FI_ERR_CAPACITY for R > max_batch or (host call) prompt bytes above max_prompt_bytes;
 * FI_ERR_STATE on a sharded pool.  The host call stages the rows through buffers of max_batch * endpoint_count counts
 * allocated by its first call. */
int fi_epp_match_counts(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                        uint16_t* counts, uint32_t* nblocks_out, uint64_t* chains_out);
/* The same on device buffers, in `stream` order like fi_epp_pick_batch_device. */
int fi_epp_match_counts_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                               uint64_t total_prompt_bytes, void* d_counts, void* d_nblocks_out, void* d_chains_out,
                               void* stream);

/* Match lists (docs/SPEC.md S.3b): fi_epp_match_counts as one sparse list per request, for the same host-side plugins.
 * Request r's list holds (endpoint_begin + j, counts[r][j]) for every j with counts[r][j] > 0, in ascending endpoint
 * order, where counts is the matrix fi_epp_match_counts would return at the same point of the call order: upstream's
 * map of the pods that matched.  list_offsets [R + 1]: list_offsets[0] = 0 and request r's entries are
 * entries[list_offsets[r] .. list_offsets[r + 1]).  list_offsets is always written in full; only entries at positions
 * below cap are written, and cap = R * endpoint_count never falls short.  nblocks_out and chains_out (optional),
 * ordering, statistics, chains, partial-pool handles and the errors are fi_epp_match_counts': FI_ERR_INVALID also for
 * NULL list_offsets with R > 0 or NULL entries with cap > 0.  The host call returns FI_ERR_CAPACITY when
 * list_offsets[R] > cap, having written everything else; it waits once more for the total, and copies the entries
 * through bounded staging.  The lists run through a device scratch of max_batch * endpoint_count 4-byte slots and
 * max_batch counts, allocated by the first lists call.  R = 0: FI_OK, and list_offsets[0] = 0 when list_offsets is
 * not NULL.  Two calls on the same index state give identical bytes. */
int fi_epp_match_lists(fi_epp* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                       uint64_t* list_offsets, fi_match_entry* entries, uint64_t cap, uint32_t* nblocks_out,
                       uint64_t* chains_out);
/* The same on device buffers, in `stream` order like fi_epp_pick_batch_device: d_list_offsets [R + 1] u64, d_entries
 * cap entries (4-byte aligned).  A cap that falls short still returns FI_OK, with entries at cap and beyond untouched:
 * the caller compares list_offsets[R] with cap after the stream, and the call never blocks the host. */
int fi_epp_match_lists_device(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                              uint64_t total_prompt_bytes, void* d_list_offsets, void* d_entries, uint64_t cap,
                              void* d_nblocks_out, void* d_chains_out, void* stream);

/* Pipelined device path.  fi_epp_pick_submit enqueues one batch exactly like fi_epp_pick_batch_device (inputs
 * ready in `stream` order at the call) but does NOT order `stream` behind the result: batch k+1's block
 * hashing and chain walk run while batch k is still being matched (two batches in flight, internal
 * streams).  The inputs and `d_out` of a submitted batch must stay untouched until a fi_epp_pick_wait
 * issued after it: that call makes `stream` wait (on the device; the host does not block) for every batch
 * submitted so far.  Batches complete in submission order and see the index as of their submit call.
 * Sharded handles and block sizes that are not a multiple of 32 take the stream-ordered path inside. */
int fi_epp_pick_submit(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0, uint32_t R,
                       uint64_t total_prompt_bytes, void* d_out, void* stream);
int fi_epp_pick_wait(fi_epp* h, void* stream);

/* Pipelined calls for a serving loop (docs/SPEC.md S.9): submit(k+1) -> wait_batch(k) -> read picks ->
 * add_submitted(k).
 * fi_epp_pick_submit_ex: pipelined submit of any pick variant, byte-identical to its stream-ordered counterpart on the
 * index as of the call.  k == 0: [R][n_profiles] picks like fi_epp_pick_batch_device_lora (d_adapters may be NULL;
 * d_subsets must be NULL, else FI_ERR_INVALID).  1 <= k <= FI_EPP_MAX_RANKED: [R][n_profiles][k] like
 * fi_epp_pick_batch_device_subset (d_subsets NULL = the ranked call).  Argument checks and errors are the
 * counterpart's.  d_chains_out (optional): R * max_blocks hashes, as the counterparts' chains_out.  *ticket (may be
 * NULL): the batch's sequence number, monotonic per handle and shared with fi_epp_pick_submit (one per batch of
 * R > 0 there).  Handles that fi_epp_pick_submit serves stream-ordered (sharded, block_bytes % 32 != 0) run the
 * counterpart, which returns FI_ERR_STATE for ranked and subset picks on a sharded pool. */
int fi_epp_pick_submit_ex(fi_epp* h, const void* d_prompts, const void* d_offsets, const void* d_h0,
                          const void* d_adapters, const void* d_subsets, uint32_t R, uint64_t total_prompt_bytes,
                          uint32_t k, void* d_out, void* d_chains_out, void* stream, uint64_t* ticket);
/* `stream` waits (on the device; the host does not block) for batch `ticket` and the batches before it, not for
 * later ones (a ticket more than 8 submits old waits for the oldest of the last 8).  FI_ERR_INVALID for a ticket
 * never issued. */
int fi_epp_pick_wait_batch(fi_epp* h, uint64_t ticket, void* stream);
/* PreRequest for a submitted batch: indexer.Add(chain_r, endpoints[r]) for r < R (<= the batch's R), the chains read
 * from the handle's own buffer for that batch; equal to fi_epp_index_add_chains with those chains.  Ordered like every
 * index update: picks submitted before the call do not see it, every pick submitted after it does.  It skips the host
 * waits of fi_epp_index_add_chains_device (overflow readback, previous staging) and waits for the previous update's
 * index counters only when the last counters read leave too little room below the rebuild threshold for the keys the
 * pending updates may add; at index loads near that threshold it therefore waits like the stream-ordered Add
 * (DESIGN.md §4.0).  A batch's chains stay available until the
 * next-but-one submit or any stream-ordered pick or hash call; after that, for batches that were not pipelined
 * (sharded handles, block_bytes % 32 != 0), with the host LRU or with lru_capacity == 0: FI_ERR_STATE.  FI_ERR_INVALID
 * for a ticket never issued, an endpoint >= num_endpoints or nblocks[r] > max_blocks. */
int fi_epp_index_add_submitted(fi_epp* h, uint64_t ticket, const uint32_t* endpoints, const uint32_t* nblocks,
                               uint32_t R);
/* How the pipelined path runs: out[0] = 1 if the GPU is partitioned between its stages, out[1] / out[2] = SMs of the
 * partitions.  The pipelined path always runs on the whole GPU with two batches in flight, so out is {0, 0, 0}. */
int fi_epp_pipeline_info(fi_epp* h, int32_t out[3]);

void* fi_epp_pinned_alloc(size_t bytes);
void fi_epp_pinned_free(void* p);

/* Multi-GPU (one handle per GPU, endpoint-range shards).  Rank 0 makes an id,
 * the host distributes it out of band, every rank calls comm_init.  A handle with max_blocks > 1023 cannot be
 * sharded: comm_init returns FI_ERR_STATE. */
int fi_epp_comm_unique_id(uint8_t out[FI_EPP_UNIQUE_ID_BYTES]);
int fi_epp_comm_init(fi_epp* h, const uint8_t id[FI_EPP_UNIQUE_ID_BYTES], uint32_t rank, uint32_t world);
/* Must precede the first index update of the handle.  How the sharded pick reduces the ranks' local
 * (score, endpoint) picks: FI_EXCHANGE_NONE (one rank), FI_EXCHANGE_PEER (default: the match kernel stores its
 * pick into every rank's buffer over NVLink peer memory / CUDA IPC and the merge kernel polls tagged words —
 * no collective call for the reduction) or FI_EXCHANGE_NCCL (one ncclAllGather: env FI_EPP_EXCHANGE=nccl,
 * more than 16 ranks, or a rank that cannot map a peer's buffer).  Every rank hashes every prompt (env
 * FI_EPP_SHARD_HASH=split: hashing split over the ranks and the chains all-gathered instead — measured slower on
 * NVLink-connected GPUs: hashing 16 KiB from local HBM costs less than receiving 2 KiB over the link). */
#define FI_EXCHANGE_NONE 0
#define FI_EXCHANGE_PEER 1
#define FI_EXCHANGE_NCCL 2
int fi_epp_comm_exchange(fi_epp* h);

/* Runtime knobs (measurement and tuning; every one has a working default).  Names:
 *   "exchange"     sharded pick reduction: FI_EXCHANGE_PEER | FI_EXCHANGE_NCCL (PEER only if the peers were mapped)
 *   "shard_hash"   sharded hashing: 0 = every rank hashes every prompt (default), 1 = split over the ranks + all-gather of the chains
 *   "device_lru"   1 = per-endpoint LRUs resident in HBM (default when lru_capacity >= max_blocks), 0 = host LRU; before the first Add
 *   "lru_table_slots"  slots per endpoint table of the device LRU (0 = sized by free HBM, 4..32 x lru_capacity)
 *   "feed_slices"  slices of a host-buffer pick's prompt copy, 1..16 (default 8)
 *   "lru_threads"  host worker threads of fi_epp_index_add_chains (takes effect at the next call)
 * FI_ERR_INVALID for an unknown name or a value out of range. */
int fi_epp_set_option(fi_epp* h, const char* name, int64_t value);

int fi_epp_set_profiling(fi_epp* h, int on);
int fi_epp_get_stats(fi_epp* h, fi_epp_stats* out);
int fi_epp_reset_stats(fi_epp* h);

#ifdef __cplusplus
}
#endif
#endif /* FI_EPP_H_ */
