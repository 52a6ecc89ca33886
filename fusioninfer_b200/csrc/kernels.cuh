// kernels.cuh — device-side data layout and launcher declarations of libfi_epp.
//
// HBM layout (DESIGN.md "Data layout"):
//   prompts   concatenated prompt bytes, request r = [offsets[r], offsets[r+1])
//   chain     [R][MP] u64   chained block hashes h_1..h_n (SURVEY.md Appendix A.1)
//   index     keys    [C]     u64 table, buckets of 4 keys = one 32 B sector; 0 = empty, ~0 = tombstone
//             node_of [C]     u32 node of the key in that slot
//             klog    [C+3]   u64 key of node n (0: free / retired); nodes are numbered in insertion order,
//                             nodes C, C+1 belong to the hashes 0 and ~0, node C+2 is a never-written row
//             rows    [C+3][W] u32, row n = membership bitset of node n over the local endpoints
//                             (bit e%32 of word e/32)
//             cnt     [C+3]   u32 popcount of the row (this rank's endpoints holding the block)
//             rmask   [C+3]   u32 bit g set ⇔ rank g's row of this key is non-empty; key present ⇔ rmask != 0.
//                             One rank: rmask = (cnt > 0).  Endpoint-range shards: every rank's table is a
//                             DIRECTORY of the whole pool's keys (rows only for its own endpoints), kept exact by
//                             gossiping the owners' APPEAR / VANISH transitions (index_kernels.cu), so the first
//                             block NO endpoint holds — upstream's stopping point — is found locally.
//   picks     [R][P]        fi_pick
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fi_epp.h"

namespace fi {

constexpr uint32_t SLOT_MISS = 0xFFFFFFFFu;
constexpr uint64_t KEY_EMPTY = 0ull;
constexpr uint64_t KEY_TOMB = ~0ull;
constexpr int BUCKET_KEYS = 4;  // one 32-byte sector (64-byte buckets of 8 were measured slower: DESIGN.md)

struct IndexView {
  uint64_t* keys;
  uint32_t* node_of;
  uint64_t* klog;
  uint32_t* rows;
  uint32_t* cnt;
  uint32_t* rmask;  // per node: ranks whose local row is non-empty (bit = rank); key present ⇔ rmask != 0
  uint64_t bmask;   // buckets - 1
  uint64_t C;      // regular slots = buckets * BUCKET_KEYS
  uint32_t W;      // words per row (power of two)
  uint32_t logW;
};

// device-side counters of the index (one cache line)
struct IndexCounters {
  unsigned long long used;        // slots claimed = nodes allocated (keys + tombstones)
  unsigned long long tombstones;  // keys retired because no rank holds them any more
  unsigned long long overflow;    // != 0: an insert found no free slot
  unsigned long long pad;
};

// Transition log of one gossip round (sharded pools): the hashes whose LOCAL row went empty -> non-empty
// (appear) or non-empty -> empty (vanish) while this rank applied its own SET / CLEAR ops.  The other ranks
// replay them into their directories (rmask bit of this rank).
struct GossipLog {
  unsigned long long* n_appear;  // device counters (null: single rank, nothing is logged)
  unsigned long long* n_vanish;
  uint64_t* appear;              // [cap]
  uint64_t* vanish;              // [cap]
  uint64_t cap;
};

// Removal set of fi_epp_index_remove_endpoints, passed as a kernel parameter: the row words that hold a removed
// local endpoint (word[k], its bits[k], k < m) and the same as a whole-row mask (row[w], w < W).
constexpr uint32_t MAX_ROW_WORDS = 128;  // 4096 local endpoints (validate_config)
struct RemoveSet {
  uint32_t m;
  uint32_t word[MAX_ROW_WORDS];
  uint32_t bits[MAX_ROW_WORDS];
  uint32_t row[MAX_ROW_WORDS];
};

struct ProfileDev {
  uint32_t n_scorers;
  uint32_t n_filters;                    // by-label filters, ANDed (fi_profile: role_mask first, then more_filters)
  uint32_t filter[FI_EPP_MAX_FILTERS];
  uint32_t kind[FI_EPP_MAX_SCORERS];
  double weight[FI_EPP_MAX_SCORERS];
};

// alive and carrying, for every filter of the profile, at least one of its label bits
__host__ __device__ inline bool profile_admits(const ProfileDev& pr, uint32_t ep_flags, uint32_t ep_role_mask) {
  if (!(ep_flags & FI_ENDPOINT_ALIVE)) return false;
  for (uint32_t f = 0; f < pr.n_filters; ++f)
    if (!(ep_role_mask & pr.filter[f])) return false;
  return true;
}

// best total of a profile when no prefix block matches (per batch constant); the endpoints that attain it
// are the bit words ScoreTables::ztie — which of them wins depends on the request's tie rotation
struct ZeroBest {
  double score;
  uint32_t any;  // 0: no eligible local endpoint
  uint32_t pad;
};

struct EndpointDev {  // raw state of one endpoint of the GLOBAL pool
  double kv_util;
  int32_t queue_depth;
  uint32_t role_mask;
  uint32_t flags;
  uint32_t pad;
};

struct LoraDev {  // adapter residency of one LOCAL endpoint (lora-affinity-scorer)
  uint64_t active[FI_EPP_MAX_LORA];
  uint64_t waiting[FI_EPP_MAX_LORA];
  uint32_t n_active, n_waiting, max_active, pad;
};

struct ScoreTables {
  ProfileDev prof[FI_EPP_MAX_PROFILES];
  uint32_t n_profiles;
  uint32_t Epad;        // W * 32
  const double* sc;     // [P][S][Epad] clamp01'd per-endpoint scores of the non-prefix scorers
  const uint32_t* elig; // [P][W] eligibility bit words
  const ZeroBest* zero; // [P]
  const uint32_t* ztie; // [P][W] eligible local endpoints whose zero-match total equals zero[p].score
  const LoraDev* lora;  // [Epad] or null
  uint32_t has_lora;    // some profile has a lora-affinity-scorer: scores depend on the request's adapter,
  uint32_t pad;         // so every eligible endpoint is scored per request (no zero-match shortcut)
};

// Peer-memory exchange of the endpoint-range sharded mode (one buffer per rank, every rank's buffer
// mapped into every process over NVLink / CUDA IPC).  Low-latency protocol: every 32-bit datum travels
// in one aligned 64-bit store together with a 32-bit tag = the step number of the pick call, so a word is
// valid exactly when its tag matches — no fences, no flags, no barrier between the ranks.  The producer
// (match_pick_kernel: this rank's local pick) stores each word into slot [parity][own rank] of EVERY rank's
// buffer as soon as it exists; the consumer (merge_picks_kernel) polls only the words of the request it is
// about to reduce, so the transfer of later requests overlaps the work on earlier ones.  Parity double-buffers consecutive steps (a rank can
// be at most one step ahead of a peer, because its merge needs that peer's picks of the previous step).
constexpr int FI_MAX_RANKS = 16;
struct PeerXchg {
  uint32_t world, rank;
  uint32_t step;                // tag of this pick call (monotonic, starts at 1; buffers start zeroed)
  uint32_t enabled;             // 0: the NCCL all-gather path is used instead
  uint8_t* base[FI_MAX_RANKS];  // base[k] = rank k's exchange buffer as mapped here (base[rank] is local)
  uint64_t off_pick[2];         // u64 {tag:word}       [world][R][P][4]  endpoint, match_blocks, score lo, hi
  uint32_t* err;                // local: set to 1 if a poll timed out
};

struct MatchParams {
  const uint64_t* chain;
  const uint32_t* nblocks;
  const uint64_t* offsets;  // [R+1], prompt byte offsets (PD threshold); may be null if !apply_pd
  const uint64_t* adapters; // [R] target adapter id per request, or null (= id 0)
  uint32_t R;
  uint32_t MP;  // pitch of chain rows (multiple of 4)
  IndexView ix;
  ScoreTables st;
  uint32_t ep_begin;
  uint32_t ep_count;
  uint32_t E_global;  // pool size: ties rotate over the whole pool (tie_start)
  uint32_t r_base;    // index of this launch's request 0 within the caller's batch (sliced host feed)
  const uint64_t* h0; // [R] chain seeds (tie rotation of prompts shorter than one block)
  uint32_t lpm;  // fi_match_mode
  // pd-profile-handler
  uint32_t apply_pd, pd_decode, pd_prefill;
  double pd_threshold;
  fi_pick* out;                       // [R][P], or [R][P][k] when k > 0 (null for match counts)
  unsigned long long* probed_blocks;  // optional Σ N_probe
  uint32_t* work_counter;             // dynamic request queue of the launch (the launcher zeroes it first)
  uint32_t lane_zero;                 // always 0: makes the ticket address formally lane-dependent (match_kernels.cu take_ticket)
  uint32_t k;                         // 0: one pick per profile, out [R][P]; else the ranked pick, out [R][P][k] (S.6a)
  PeerXchg px;                        // sharded mode, peer-memory exchange (px.enabled)
  // subset picks (docs/SPEC.md S.5a), ranked launches only; appended so that the other fields keep their offsets
  const uint32_t* subsets;  // [R][sub_pitch] candidate bitset of each request over the pool, or null (unrestricted)
  uint32_t sub_pitch;       // words per subset row: ceil(E_global / 32); words past it read as 0
  const EndpointDev* eps;   // [E_global] raw endpoint state: the per-request queue min / max of a subset pick
  // match counts (docs/SPEC.md S.3a), appended like the subset fields: non-null selects the COUNTS variant, which
  // writes every local endpoint's match count instead of picks (out, k, PD and the score tables are not read)
  uint16_t* counts;  // [R][ep_count], dense, 2-byte aligned
  // the handle's max_blocks (appended like the fields above): above 1023 a count needs more than the 10 bit-planes of
  // one match window, and launch_match_pick runs the windowed variant (DESIGN.md §4.9)
  uint32_t max_blocks;
  // match lists (docs/SPEC.md S.3b), appended like the fields above: non-null selects the LISTS variant, which writes
  // request r's matched local endpoints as (column << 12) | count into lists[r * ep_count ..] and their number into
  // nnz[r] (counts is not read)
  uint32_t* lists;  // [R][ep_count]
  uint32_t* nnz;    // [R]
};

struct MergeParams {
  const fi_pick* gathered;  // [ranks][R][P]
  uint32_t ranks, R, P;
  const uint32_t* nblocks;
  const uint64_t* offsets;
  const uint64_t* chain;  // [R][MP]  (tie rotation: first block hash)
  const uint64_t* h0;     // [R]
  uint32_t MP, E_global;
  uint32_t apply_pd, pd_decode, pd_prefill;
  double pd_threshold;
  fi_pick* out;  // [R][P]
  PeerXchg px;   // px.enabled: poll every rank's tagged pick words in-kernel instead of after an all-gather
};

// ---- launchers (each returns the cudaGetLastError() of its launch) -----------
// block hashing and chain walk in one kernel, for block_bytes % 32 == 0 (cudaErrorInvalidValue otherwise).
// sm_count sets the tile: 32 or 64 requests per whole-SM CTA, the smallest whose grid fits one CTA per SM, and
// half-SM CTAs of 64 requests for larger batches
// early (optional): the index the batch's match reads; hash_chain may then leave a request's chain after its
// first block that index does not hold unhashed (zeros; hash_kernels.cu "early exit").  hashed (optional): += the
// blocks whose prompt bytes were read (profiling).
cudaError_t launch_hash_chain(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                              uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain, uint32_t* nblocks,
                              int sm_count, cudaStream_t s, const IndexView* early = nullptr,
                              unsigned long long* hashed = nullptr);
// the same with the tile shape given: walk = 1 or 2 with warps = 32 (whole SM), walk = 2 with warps = 16 (half SM)
cudaError_t launch_hash_chain_shape(uint32_t walk, uint32_t warps, const uint8_t* prompts, const uint64_t* offsets,
                                    const uint64_t* h0, uint32_t R, uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain,
                                    uint32_t* nblocks, cudaStream_t s, const IndexView* early = nullptr,
                                    unsigned long long* hashed = nullptr);
cudaError_t launch_hash_generic(const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                                uint32_t R, uint32_t B, uint32_t M, uint32_t MP, uint64_t* chain,
                                uint32_t* nblocks, cudaStream_t s);

cudaError_t launch_index_set(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t n,
                             uint32_t ep_begin, uint32_t ep_count, uint32_t rank, GossipLog log, cudaStream_t s);
cudaError_t launch_index_clear(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t n,
                               uint32_t ep_begin, uint32_t ep_count, uint32_t rank, GossipLog log, cudaStream_t s);
// the same with the op count read from device memory (ops produced by a kernel; cap = buffer capacity)
cudaError_t launch_index_clear_counted(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t cap,
                                       const unsigned long long* n_dev, uint32_t ep_begin, uint32_t ep_count, uint32_t rank,
                                       GossipLog log, cudaStream_t s);
// replay another rank's transitions into this rank's directory (n hashes; bit = that rank)
cudaError_t launch_index_remote_appear(IndexView ix, IndexCounters* ctr, const uint64_t* hashes, uint64_t n,
                                       uint32_t rank, cudaStream_t s);
cudaError_t launch_index_remote_vanish(IndexView ix, IndexCounters* ctr, const uint64_t* hashes, uint64_t n,
                                       uint32_t rank, cudaStream_t s);
cudaError_t launch_index_rebuild(IndexView from, IndexView to, IndexCounters* ctr, cudaStream_t s);
// clear the removal set's bits from every live row (and the two special nodes), retire the keys nobody holds any
// more, add the number of cleared bits to *removed.  whole_rows: 16-byte whole-row loads instead of one load per
// listed word (remove_whole_rows decides)
cudaError_t launch_index_remove_sweep(IndexView ix, IndexCounters* ctr, const RemoveSet& rs, bool whole_rows, uint32_t rank,
                                      unsigned long long* removed, int sm_count, cudaStream_t s);
// Every 32-byte sector of a row holds a listed word: then both sweep shapes move the same bytes and the whole-row
// one issues a quarter of the loads.  Rows narrower than 16 bytes always take the per-word shape.
inline bool remove_whole_rows(const RemoveSet& rs, uint32_t W) {
  if (W < 4) return false;
  const uint32_t sector_words = 8;
  const uint32_t sectors = (W + sector_words - 1) / sector_words;
  uint32_t hit = 0;
  bool seen[MAX_ROW_WORDS / 8 + 1] = {};
  for (uint32_t k = 0; k < rs.m; ++k) {
    const uint32_t s = rs.word[k] / sector_words;
    if (!seen[s]) {
      seen[s] = true;
      ++hit;
    }
  }
  return hit == sectors;
}
cudaError_t launch_index_contains(IndexView ix, const fi_index_op* q, uint64_t n, uint32_t ep_begin,
                                  uint32_t ep_count, uint8_t* out, cudaStream_t s);
// Snapshots (index_kernels.cu).  Export walks the regular nodes [0, n) (n = min(used, C)) and the markers C, C+1 in
// index_snap_tiles(n) tiles: the count pass reads n from ctr and writes the live nodes of each of the
// index_snap_tiles(C) tiles (0 past the walk); the export of tiles [t0, t1) writes their keys and their rows narrowed
// to We words at tile_off[t] - base (64-bit offsets: one export may cover every tile).  Import inserts n blob nodes
// starting at blob position g0 into fresh tables (m0, m1: the blob positions of the keys 0 and ~0, or ~0); *dup != 0:
// a key repeats.
uint32_t index_snap_tiles(uint64_t n);
cudaError_t launch_index_snap_count(IndexView ix, const IndexCounters* ctr, uint32_t* tile_live, cudaStream_t s);
cudaError_t launch_index_snap_export(IndexView ix, uint64_t n, uint32_t t0, uint32_t t1, const uint64_t* tile_off, uint64_t base,
                                     uint32_t We, uint64_t* keys, uint32_t* rows, cudaStream_t s);
cudaError_t launch_index_snap_import(IndexView ix, IndexCounters* ctr, const uint64_t* keys, const uint32_t* rows, uint64_t n,
                                     uint64_t g0, uint64_t m0, uint64_t m1, uint32_t We, uint32_t* dup, cudaStream_t s);

cudaError_t launch_prepare_endpoints(const EndpointDev* eps, uint32_t E_global, uint32_t ep_begin,
                                     uint32_t ep_count, ScoreTables st, double* sc, uint32_t* elig,
                                     ZeroBest* zero, uint32_t* ztie, cudaStream_t s);

cudaError_t launch_match_pick(const MatchParams& p, int sm_count, cudaStream_t s);
cudaError_t launch_merge_picks(const MergeParams& p, cudaStream_t s);
// the pack step of match lists (S.3b): offsets[R + 1] = the exclusive scan of nnz[R] (one CTA); then the entries of
// list positions [lo, hi) to out[position - lo], read from the slots lists[r * pitch ..] (one warp per request)
cudaError_t launch_list_scan(const uint32_t* nnz, uint32_t R, uint64_t* offsets, cudaStream_t s);
cudaError_t launch_list_copy(const uint32_t* lists, uint32_t pitch, const uint64_t* offsets, uint32_t R, uint32_t ep_begin,
                             uint64_t lo, uint64_t hi, fi_match_entry* out, cudaStream_t s);

}  // namespace fi
