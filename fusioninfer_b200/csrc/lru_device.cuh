// lru_device.cuh — data layout and launchers of the GPU-resident per-endpoint LRU (lru_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fi_epp.h"

namespace fi {

struct LruSlot {    // 16 bytes
  uint64_t key;     // 0 = empty, ~0 = tombstone (the hashes 0 / ~0 themselves live in two dedicated slots)
  uint32_t posp1;   // log position of the key's live record + 1; 0 = none yet (inserted by the running sub-batch)
  uint32_t ord;     // order (+1) of the key's last touch in the running sub-batch; 0 outside of one
};

struct DevLru {
  LruSlot* slots;   // [EL][TS + 2]
  uint64_t* log;    // [EL][L]
  uint32_t* head;   // [EL] next free log position
  uint32_t* tail;   // [EL] oldest position that may still be live
  uint32_t* count;  // [EL] live entries
  uint32_t* used;   // [EL] regular table slots consumed (entries + tombstones); reserved BEFORE an insert
  uint32_t* hold;   // [EL] scratch: head before the running sub-batch's appends
  uint32_t* dcount; // [EL] scratch: winners (distinct keys touched) of the running sub-batch
  uint32_t* ovf;    // [EL] the running sub-batch would overfill this endpoint's table: its requests are deferred
  uint32_t* any_ovf; // some ovf[e] was set by the running touch kernel
  uint32_t* error;  // != 0: an invariant broke (reported by the next host call)
  uint32_t* cap;    // [EL] the endpoint's LRU capacity (fi_epp_set_lru_capacities), in [max_blocks, capacity]: what
                    // the LRU holds.  Table and log room are sized and bounded by the uniform `capacity`.
  unsigned long long* n_sets;        // totals (fi_epp_index_stats, fi_epp_lru_counters): SETs emitted,
  unsigned long long* n_clears;      // CLEARs emitted,
  unsigned long long* n_doomed;      // winners that were gone again by the end of their sub-batch,
  unsigned long long* n_maintained;  // log compactions + table rebuilds
  uint32_t EL, TS, L, capacity;
  uint32_t insert_limit;  // a table never holds more than this many keys + tombstones (0.85 TS)
};

// one sub-batch of indexer.Add calls (lru_plan.h); K requests, `touches` blocks in total
struct LruBatch {
  const uint32_t* req_id;   // [K] row of `chains`
  const uint32_t* req_ep;   // [K] local endpoint
  const uint32_t* req_n;    // [K] blocks
  const uint32_t* req_off;  // [K] first touch's position in the sub-batch
  const uint32_t* ep_list;  // [K] requests grouped by endpoint, ascending
  const uint32_t* ep_start; // [EL + 1]
  const uint64_t* chains;   // device, [rows][pitch]
  uint32_t pitch;
  uint32_t K;
  uint32_t* slot_of;        // [touches] scratch: table slot of every touch
  uint32_t* wcount;         // [K] scratch: winners per request
  uint32_t* base;           // [K] scratch: rank of the request's first winner among its endpoint's winners
  fi_index_op* sets;        // [touches] out: SET for touches that added a key, op 0 elsewhere (chain order kept)
};

cudaError_t launch_lru_maintain(const DevLru& lru, const uint32_t* inc, bool force, cudaStream_t s);
cudaError_t launch_lru_touch(const DevLru& lru, const LruBatch& b, cudaStream_t s);
cudaError_t launch_lru_untouch(const DevLru& lru, const LruBatch& b, cudaStream_t s);
cudaError_t launch_lru_count(const DevLru& lru, const LruBatch& b, cudaStream_t s);
cudaError_t launch_lru_scan(const DevLru& lru, const LruBatch& b, cudaStream_t s);
cudaError_t launch_lru_append(const DevLru& lru, const LruBatch& b, fi_index_op* clears, unsigned long long* n_clears,
                              uint64_t clears_cap, uint32_t ep_begin, cudaStream_t s);
cudaError_t launch_lru_evict(const DevLru& lru, fi_index_op* clears, unsigned long long* n_clears, uint64_t clears_cap,
                             uint32_t ep_begin, cudaStream_t s);
// one round of a resize (fi_epp_set_lru_capacities): evict the quota[i] least recently used entries of local endpoint
// eps[i] for i < n (device arrays; the host plans the quotas so that a round's CLEARs fit clears_cap)
cudaError_t launch_lru_shrink(const DevLru& lru, const uint32_t* eps, const uint32_t* quota, uint32_t n, fi_index_op* clears,
                              unsigned long long* n_clears, uint64_t clears_cap, uint32_t ep_begin, cudaStream_t s);
// empty the LRUs of the n local endpoints eps[0..n) (device array; n <= 65535)
cudaError_t launch_lru_reset(const DevLru& lru, const uint32_t* eps, uint32_t n, cudaStream_t s);
// diagnostics: the live keys of local endpoint e, least recently used first
cudaError_t launch_lru_dump(const DevLru& lru, uint32_t e, uint64_t* out, uint32_t* n_out, cudaStream_t s);
// snapshots: every endpoint's live keys, oldest first, endpoint e's at out + off[e] (n_out[e]: how many; bad != null:
// *bad = 1 where that differs from count[e], a broken invariant); and the load of every endpoint's LRU into a fresh
// store from len[e] keys at keys + off[e] (*dup != 0: a key repeats in an LRU)
cudaError_t launch_lru_dump_all(const DevLru& lru, const uint64_t* off, uint64_t* out, uint32_t* n_out, uint32_t* bad,
                                cudaStream_t s);
cudaError_t launch_lru_load(const DevLru& lru, const uint64_t* keys, const uint64_t* off, const uint32_t* len, uint32_t* dup,
                            cudaStream_t s);

}  // namespace fi
