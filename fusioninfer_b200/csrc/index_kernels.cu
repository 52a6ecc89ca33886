// index_kernels.cu — GPU-resident open-addressed hash index of (endpoint, block-hash)
// membership, sm_90a.
//
// Logical content = upstream's prefix indexer (SURVEY.md Appendix A.2: hashToPods),
// physically a table keyed by block hash whose value is a bitset row over the local
// endpoints: one 128 B row read answers "which of 1024 endpoints hold this block".
// Keys live in buckets of 4 (one 32 B sector); linear probing over buckets.
// Inserts claim an EMPTY key with atomicCAS and give it the next NODE: nodes are
// numbered in insertion order and own the key's row (index_device.cuh), so a chain
// inserted in order occupies consecutive rows.  Membership bits flip with
// atomicOr/atomicAnd, cnt tracks the row popcount.
//
// Key presence is rmask[node] != 0: bit g says "rank g's row of this key is non-empty".
// With one rank that is just cnt > 0.  With an endpoint-range sharded pool every rank's
// table is a directory of the WHOLE pool's keys (rows only for its own endpoints): the
// owner of an endpoint applies the SET / CLEAR exactly (the row bit makes it idempotent)
// and logs the transitions of its row, empty -> non-empty (APPEAR) and back (VANISH); the
// other ranks replay those into their rmask (index_remote_*).  A key nobody holds any more
// becomes a tombstone and its node is retired (neither is reused until a rebuild compacts
// the live nodes in order), which keeps lookups exact without reading the row — and lets
// every rank find upstream's stopping point, the first block NO pod holds, on its own.
#include "index_device.cuh"
#include "kernels.cuh"

namespace fi {

namespace {

// find the table slot of h or claim an EMPTY one (*claimed = true: the caller allocates its node).
// SLOT_MISS on a full table.
__device__ uint32_t table_find_or_claim(const IndexView& ix, IndexCounters* ctr, uint64_t h, bool* claimed) {
  *claimed = false;
  uint64_t b = h & ix.bmask;
  for (uint64_t it = 0; it <= ix.bmask; ++it) {
    unsigned long long* kb = reinterpret_cast<unsigned long long*>(ix.keys + b * BUCKET_KEYS);
#pragma unroll 1
    for (int j = 0; j < BUCKET_KEYS; ++j) {
      unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(kb + j);
      if (k == h) return (uint32_t)(b * BUCKET_KEYS + j);
      if (k == KEY_EMPTY) {
        unsigned long long old = atomicCAS(kb + j, (unsigned long long)KEY_EMPTY, (unsigned long long)h);
        if (old == KEY_EMPTY) {
          *claimed = true;
          return (uint32_t)(b * BUCKET_KEYS + j);
        }
        if (old == h) return (uint32_t)(b * BUCKET_KEYS + j);
        // someone else claimed it for another key: keep scanning
      }
    }
    b = (b + 1) & ix.bmask;
  }
  atomicExch(&ctr->overflow, 1ull);
  return SLOT_MISS;
}

// Ordered reservation of one CTA pass: the flagged threads get CONSECUTIVE positions of *counter in
// thread (= op) order — one atomicAdd per CTA.  Used for the node numbers of new keys (the keys of a chain
// that arrives as consecutive ops end up next to each other in klog / rows) and for the APPEAR log (so that
// the ranks replaying it allocate consecutive nodes too).  Every thread of the CTA must call it.
__device__ unsigned long long cta_reserve(bool flag, unsigned long long* counter) {
  __shared__ uint32_t s_warp[8];
  __shared__ unsigned long long s_base;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xFFFFFFFFu, flag);
  const uint32_t rank_in_warp = __popc(m & ((1u << lane) - 1u));
  if (lane == 0) s_warp[warp] = __popc(m);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t tot = 0;
    for (int w = 0; w < 8; ++w) {
      const uint32_t c = s_warp[w];
      s_warp[w] = tot;
      tot += c;
    }
    s_base = tot ? atomicAdd(counter, (unsigned long long)tot) : 0ull;
  }
  __syncthreads();
  const unsigned long long pos = flag ? s_base + s_warp[warp] + rank_in_warp : ~0ull;
  __syncthreads();  // s_warp / s_base are reused by the next reservation
  return pos;
}

// node of a slot some other thread claimed: wait until that thread has published it
__device__ __forceinline__ uint32_t wait_node(const IndexView& ix, uint32_t slot) {
  const volatile uint32_t* p = ix.node_of + slot;
  uint32_t n;
  while ((n = *p) == NODE_INVALID) __nanosleep(20);
  return n;
}

// REMOTE = false: this rank's own SET ops (row bit, popcount, APPEAR log).
// REMOTE = true:  replay of rank `rank`'s APPEAR log: directory entry only (rmask bit of that rank).
template <bool REMOTE>
__global__ void __launch_bounds__(256) index_set_kernel(IndexView ix, IndexCounters* ctr, const fi_index_op* __restrict__ ops,
                                                        const uint64_t* __restrict__ hashes, uint64_t n, uint32_t ep_begin,
                                                        uint32_t ep_count, uint32_t rank, GossipLog log) {
  const uint32_t rbit = 1u << rank;
  const uint32_t zero_node = (uint32_t)(ix.C + 2);
  // every thread of a CTA runs the same number of passes (block-wide barriers inside)
  for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = base + threadIdx.x;
    uint64_t hsh = 0;
    bool active = false;
    uint32_t e = 0;
    if (i < n) {
      if (REMOTE) {
        hsh = hashes[i];
        active = true;
      } else {
        const fi_index_op op = ops[i];
        hsh = op.hash;
        e = op.endpoint - ep_begin;
        active = op.op == FI_OP_SET && e < ep_count;
      }
    }
    // 1. table slot (claim an empty one for a new key)
    bool claimed = false;
    uint32_t slot = SLOT_MISS, node = NODE_INVALID;
    if (active) {
      if (key_is_special(hsh)) node = (uint32_t)(ix.C + (hsh == KEY_TOMB ? 1 : 0));
      else slot = table_find_or_claim(ix, ctr, hsh, &claimed);
    }
    // 2. new keys get consecutive nodes in op order and publish them
    const unsigned long long mine = cta_reserve(claimed, &ctr->used);
    if (claimed) {
      if (mine < ix.C) {
        node = (uint32_t)mine;
        ix.klog[node] = hsh;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(ix.node_of + slot) = node;
      } else {
        // out of nodes (reported through ctr->overflow): retire the slot again so that "key in the table ⇔
        // some rank holds it" keeps holding, and release the threads waiting for its node
        atomicExch(&ctr->overflow, 1ull);
        ix.keys[slot] = KEY_TOMB;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(ix.node_of + slot) = zero_node;
      }
    }
    // 3. keys that were already there (possibly claimed by another CTA a moment ago): their node.  No
    // thread waits before it has published its own nodes, so the waits cannot form a cycle.
    if (active && !claimed && slot != SLOT_MISS) node = wait_node(ix, slot);
    bool appear = false;
    if (active && node != NODE_INVALID && node != zero_node) {
      if (REMOTE) {
        atomicOr(ix.rmask + node, rbit);
      } else {
        const uint32_t bit = 1u << (e & 31);
        const uint32_t old = atomicOr(ix.rows + ((uint64_t)node << ix.logW) + (e >> 5), bit);
        if (!(old & bit) && atomicAdd(ix.cnt + node, 1u) == 0u) {  // this rank's row: empty -> non-empty
          atomicOr(ix.rmask + node, rbit);
          appear = true;
        }
      }
    }
    if (!REMOTE && log.n_appear) {  // warp-uniform: sharded pools only
      const unsigned long long pos = cta_reserve(appear, log.n_appear);
      if (appear && pos < log.cap) log.appear[pos] = hsh;
    }
  }
}

// table slot of a regular key (not its node): the clear path retires the slot
__device__ uint32_t table_find_slot(const IndexView& ix, uint64_t h) {
  uint64_t b = h & ix.bmask;
  for (uint64_t it = 0; it <= ix.bmask; ++it) {
    const BucketRegs r = bucket_load(ix, b);
    const int j = bucket_scan(r, h);
    if (j < BUCKET_KEYS) return (uint32_t)(b * BUCKET_KEYS + j);
    if (j == BUCKET_KEYS) return SLOT_MISS;
    b = (b + 1) & ix.bmask;
  }
  return SLOT_MISS;
}

// rank `rbit`'s row of the key at (slot, node) has emptied: drop its directory bit; if no rank holds the key
// any more retire the key and its node (true: the caller counts the tombstone)
__device__ __forceinline__ bool rank_vanished_retires(const IndexView& ix, uint32_t slot, uint32_t node, uint32_t rbit) {
  const uint32_t oldm = atomicAnd(ix.rmask + node, ~rbit);
  if ((oldm & rbit) && (oldm & ~rbit) == 0u && slot != SLOT_MISS) {
    ix.keys[slot] = KEY_TOMB;
    ix.klog[node] = 0;
    return true;
  }
  return false;
}

__device__ __forceinline__ void rank_vanished(const IndexView& ix, IndexCounters* ctr, uint32_t slot, uint32_t node,
                                              uint32_t rbit) {
  if (rank_vanished_retires(ix, slot, node, rbit)) atomicAdd(&ctr->tombstones, 1ull);
}

template <bool REMOTE>
__global__ void __launch_bounds__(256) index_clear_kernel(IndexView ix, IndexCounters* ctr, const fi_index_op* __restrict__ ops,
                                                          const uint64_t* __restrict__ hashes, uint64_t n, uint32_t ep_begin,
                                                          uint32_t ep_count, uint32_t rank, GossipLog log,
                                                          const unsigned long long* __restrict__ n_dev) {
  const uint32_t rbit = 1u << rank;
  if (n_dev) {  // op count produced on the device (lru_evict_kernel): n is only the buffer's capacity
    const unsigned long long nd = *n_dev;
    n = nd < n ? nd : n;
  }
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t hsh;
    uint32_t e = 0;
    if (REMOTE) {
      hsh = hashes[i];
    } else {
      const fi_index_op op = ops[i];
      e = op.endpoint - ep_begin;
      if (op.op != FI_OP_CLEAR || e >= ep_count) continue;
      hsh = op.hash;
    }
    uint32_t slot = SLOT_MISS, node;
    if (key_is_special(hsh)) {
      node = (uint32_t)(ix.C + (hsh == KEY_TOMB ? 1 : 0));
    } else {
      slot = table_find_slot(ix, hsh);
      if (slot == SLOT_MISS) continue;
      node = ix.node_of[slot];
      if (node >= ix.C) continue;  // a slot parked by a node overflow
    }
    if (REMOTE) {
      rank_vanished(ix, ctr, slot, node, rbit);
      continue;
    }
    const uint32_t bit = 1u << (e & 31);
    const uint32_t old = atomicAnd(ix.rows + ((uint64_t)node << ix.logW) + (e >> 5), ~bit);
    if ((old & bit) && atomicSub(ix.cnt + node, 1u) == 1u) {  // this rank's row emptied
      rank_vanished(ix, ctr, slot, node, rbit);
      if (log.n_vanish) {
        const unsigned long long pos = atomicAdd(log.n_vanish, 1ull);
        if (pos < log.cap) log.vanish[pos] = hsh;
      }
    }
  }
}

// Re-insert every live node of `from` into the (fresh) index `to`, in node order, so that runs of
// consecutive nodes stay consecutive (each CTA pass compacts 256 consecutive old nodes into one range).  The two
// tables may differ in slots and row width (fi_epp_resize_pool): a row copies min(from.W, to.W) words — a wider
// target's extra words are zero from alloc_index, and a narrower one drops only words the removal sweep of the
// dropped endpoints has already cleared.
__global__ void __launch_bounds__(256) index_rebuild_kernel(IndexView from, IndexView to, IndexCounters* ctr) {
  const uint32_t W = from.W < to.W ? from.W : to.W;
  for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < from.C; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t s = base + threadIdx.x;
    uint64_t h = 0;
    if (s < from.C) h = from.klog[s];
    bool claimed = false;
    uint32_t slot = SLOT_MISS;
    if (h != 0) slot = table_find_or_claim(to, ctr, h, &claimed);  // keys are unique: always a fresh claim
    const unsigned long long d = cta_reserve(claimed, &ctr->used);
    if (claimed && d < to.C) {
      to.klog[d] = h;
      to.node_of[slot] = (uint32_t)d;
      to.cnt[d] = from.cnt[s];
      to.rmask[d] = from.rmask[s];
      const uint32_t* src = from.rows + (s << from.logW);
      uint32_t* dst = to.rows + (d << to.logW);
      for (uint32_t w = 0; w < W; ++w) dst[w] = src[w];
    }
  }
  // the two special nodes keep their place: the first two past the regular slots
  if (blockIdx.x == 0 && threadIdx.x < 2) {
    const uint64_t s = from.C + threadIdx.x, d = to.C + threadIdx.x;
    if (from.rmask[s]) {
      to.cnt[d] = from.cnt[s];
      to.rmask[d] = from.rmask[s];
      for (uint32_t w = 0; w < W; ++w) to.rows[(d << to.logW) + w] = from.rows[(s << from.logW) + w];
    }
  }
}

// ---- removal of whole endpoints (fi_epp_index_remove_endpoints) ------------------------------------------------
// One pass over the live nodes [0, min(used, C)) and the two special nodes C, C+1 — the table is not walked.  Index
// kernels run one at a time on the index stream and picks only read, so the thread that owns a row word stores it
// plainly; cnt takes an atomicSub because the words of a node may belong to different threads, and the thread that
// takes it to 0 retires the key exactly like a CLEAR does.

// sweep item t -> node: t < n the regular nodes, then C and C+1
__device__ __forceinline__ uint32_t sweep_node(const IndexView& ix, uint64_t t, uint64_t n) {
  return (uint32_t)(t < n ? t : ix.C + (t - n));
}

// true: the key was retired (removing every endpoint retires every key: the tombstones are counted per CTA, not
// with one atomic on the same counter each)
__device__ __forceinline__ bool remove_from_node(const IndexView& ix, uint32_t node, uint32_t gone, uint32_t rbit) {
  if (atomicSub(ix.cnt + node, gone) != gone) return false;
  const uint32_t slot = node < ix.C ? table_find_slot(ix, ix.klog[node]) : SLOT_MISS;
  return rank_vanished_retires(ix, slot, node, rbit);
}

__device__ __forceinline__ void sweep_total(uint32_t pairs, uint32_t tombs, unsigned long long* removed, IndexCounters* ctr) {
  __shared__ unsigned long long s_pairs;
  __shared__ uint32_t s_tombs;
  if (threadIdx.x == 0) s_pairs = s_tombs = 0;
  __syncthreads();
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    pairs += __shfl_xor_sync(0xFFFFFFFFu, pairs, d);
    tombs += __shfl_xor_sync(0xFFFFFFFFu, tombs, d);
  }
  if ((threadIdx.x & 31) == 0) {
    if (pairs) atomicAdd(&s_pairs, (unsigned long long)pairs);
    if (tombs) atomicAdd(&s_tombs, tombs);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_pairs) atomicAdd(removed, s_pairs);
    if (s_tombs) atomicAdd(&ctr->tombstones, (unsigned long long)s_tombs);
  }
}

// Per-word shape: a thread owns kSweepNodes nodes per pass and reads only the m listed words of each — removing one
// endpoint costs one 32-byte sector per node, not the whole row.  The loads of all its nodes are issued before any
// result is used.
constexpr int kSweepNodes = 4;
__global__ void __launch_bounds__(256) index_remove_words_kernel(IndexView ix, IndexCounters* ctr, const __grid_constant__ RemoveSet rs,
                                                                 uint32_t rbit, unsigned long long* removed) {
  const uint64_t used = *reinterpret_cast<volatile unsigned long long*>(&ctr->used);
  const uint64_t n = used < ix.C ? used : ix.C;
  const uint64_t nodes = n + 2, stride = (uint64_t)gridDim.x * blockDim.x;
  uint32_t mine = 0, tombs = 0;
  for (uint64_t t0 = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t0 < nodes; t0 += stride * kSweepNodes) {
    uint32_t node[kSweepNodes], gone[kSweepNodes];
#pragma unroll
    for (int u = 0; u < kSweepNodes; ++u) {
      const uint64_t t = t0 + u * stride;
      node[u] = t < nodes ? sweep_node(ix, t, n) : NODE_INVALID;
      gone[u] = 0;
    }
    for (uint32_t k = 0; k < rs.m; ++k) {
      const uint32_t w = rs.word[k], mk = rs.bits[k];
      uint32_t old[kSweepNodes];
#pragma unroll
      for (int u = 0; u < kSweepNodes; ++u) old[u] = node[u] != NODE_INVALID ? ix.rows[((uint64_t)node[u] << ix.logW) + w] : 0u;
#pragma unroll
      for (int u = 0; u < kSweepNodes; ++u) {
        const uint32_t hit = old[u] & mk;
        if (hit) {
          ix.rows[((uint64_t)node[u] << ix.logW) + w] = old[u] & ~mk;
          gone[u] += __popc(hit);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kSweepNodes; ++u) {
      if (gone[u]) {
        mine += gone[u];
        tombs += remove_from_node(ix, node[u], gone[u], rbit);
      }
    }
  }
  sweep_total(mine, tombs, removed, ctr);
}

// Whole-row shape: a thread owns one 16-byte chunk of a row, the W/4 chunks of a node are consecutive lanes of one
// warp (coalesced), and their counts are summed with shuffles so that one lane per node updates cnt.
__global__ void __launch_bounds__(256) index_remove_rows_kernel(IndexView ix, IndexCounters* ctr, const __grid_constant__ RemoveSet rs,
                                                                uint32_t rbit, unsigned long long* removed) {
  const uint64_t used = *reinterpret_cast<volatile unsigned long long*>(&ctr->used);
  const uint64_t n = used < ix.C ? used : ix.C;
  const uint32_t lchunks = ix.logW - 2, chunks = 1u << lchunks;  // W >= 4 (remove_whole_rows)
  const uint64_t items = (n + 2) << lchunks, stride = (uint64_t)gridDim.x * blockDim.x;
  uint32_t mine = 0, tombs = 0;
  // every lane of a warp runs the same number of passes (shuffles inside)
  for (uint64_t i0 = blockIdx.x * (uint64_t)blockDim.x; i0 < items; i0 += stride) {
    const uint64_t i = i0 + threadIdx.x;
    const uint32_t c = (uint32_t)(i & (chunks - 1));
    uint32_t node = NODE_INVALID, gone = 0;
    if (i < items) {
      node = sweep_node(ix, i >> lchunks, n);
      uint4* p = reinterpret_cast<uint4*>(ix.rows + ((uint64_t)node << ix.logW)) + c;
      const uint4 old = *p;
      const uint4 mk = make_uint4(rs.row[4 * c], rs.row[4 * c + 1], rs.row[4 * c + 2], rs.row[4 * c + 3]);
      gone = __popc(old.x & mk.x) + __popc(old.y & mk.y) + __popc(old.z & mk.z) + __popc(old.w & mk.w);
      if (gone) *p = make_uint4(old.x & ~mk.x, old.y & ~mk.y, old.z & ~mk.z, old.w & ~mk.w);
    }
    mine += gone;
    uint32_t node_gone = gone;
    for (uint32_t d = 1; d < chunks; d <<= 1) node_gone += __shfl_xor_sync(0xFFFFFFFFu, node_gone, d);
    if (c == 0 && node_gone) tombs += remove_from_node(ix, node, node_gone, rbit);
  }
  sweep_total(mine, tombs, removed, ctr);
}
static_assert(MAX_ROW_WORDS / 4 <= 32, "the 16-byte chunks of a row must fit in one warp");

// membership query (tests / diagnostics): out[i] = 1 iff (endpoint, hash) is present
__global__ void __launch_bounds__(256) index_contains_kernel(IndexView ix, const fi_index_op* __restrict__ q, uint64_t n,
                                                             uint32_t ep_begin, uint32_t ep_count,
                                                             uint8_t* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t e = q[i].endpoint - ep_begin;
    uint8_t r = 0;
    if (e < ep_count) {
      const uint32_t node = index_find(ix, q[i].hash);
      if (node != SLOT_MISS) r = (ix.rows[((uint64_t)node << ix.logW) + (e >> 5)] >> (e & 31)) & 1u;
    }
    out[i] = r;
  }
}

// ---- snapshots (fi_epp_snapshot_save / fi_epp_snapshot_load, docs/SPEC.md S.2d) -----------------------------------
// Export: an order-preserving compaction of the sweep items (the regular nodes [0, n) in order, then the marker nodes
// C, C+1: sweep_node) that hold a key — klog != 0 for a regular node, rmask != 0 for a marker.  Items come in tiles of
// kSnapTile, one CTA per tile: a count pass, a prefix sum on the host, then the export of a range of tiles into the
// staging buffers, each tile's live nodes at its offset.
constexpr uint32_t kSnapTile = 1024;

__device__ __forceinline__ bool snap_live(const IndexView& ix, uint32_t node) {
  return node < ix.C ? ix.klog[node] != 0 : ix.rmask[node] != 0;
}

// this thread's rank among the flagged threads of the CTA (kSnapTile threads)
__device__ __forceinline__ uint32_t snap_rank(bool flag) {
  __shared__ uint32_t s_w[kSnapTile / 32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xFFFFFFFFu, flag);
  if (lane == 0) s_w[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    const uint32_t c = s_w[lane];
    uint32_t inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, d);
      if ((int)lane >= d) inc += t;
    }
    s_w[lane] = inc - c;
  }
  __syncthreads();
  return s_w[warp] + __popc(m & ((1u << lane) - 1u));
}

// (n = min(ctr->used, C) is read here, so that the host learns it in the same readback as the tile counts; the grid
// covers the tiles of C + 2 items, and the tiles past n + 2 count 0)
__global__ void __launch_bounds__(kSnapTile) index_snap_count_kernel(IndexView ix, const IndexCounters* ctr, uint32_t* tile_live) {
  const uint64_t used = ctr->used, n = used < ix.C ? used : ix.C;
  const uint64_t t = (uint64_t)blockIdx.x * kSnapTile + threadIdx.x;
  const bool live = t < n + 2 && snap_live(ix, sweep_node(ix, t, n));
  const int c = __syncthreads_count(live);
  if (threadIdx.x == 0) tile_live[blockIdx.x] = (uint32_t)c;
}

// tiles [t0, t0 + gridDim.x): the live nodes' keys and their rows narrowed to We words, at tile_off[t] - base
__global__ void __launch_bounds__(kSnapTile) index_snap_export_kernel(IndexView ix, uint64_t n, uint32_t t0,
                                                                      const uint64_t* __restrict__ tile_off, uint64_t base,
                                                                      uint32_t We, uint64_t* keys, uint32_t* rows) {
  const uint32_t tile = t0 + blockIdx.x;
  const uint64_t t = (uint64_t)tile * kSnapTile + threadIdx.x;
  const uint32_t node = t < n + 2 ? sweep_node(ix, t, n) : 0u;
  const bool live = t < n + 2 && snap_live(ix, node);
  const uint32_t r = snap_rank(live);
  if (!live) return;
  const uint64_t d = tile_off[tile] - base + r;
  keys[d] = node < ix.C ? ix.klog[node] : node == ix.C ? KEY_EMPTY : KEY_TOMB;
  const uint32_t* src = ix.rows + ((uint64_t)node << ix.logW);
  for (uint32_t w = 0; w < We; ++w) rows[d * We + w] = src[w];
}

// Import: nodes [g0, g0 + n) of a snapshot (keys and rows of We words, in staging) into fresh tables, like a rebuild
// fed from the blob: a regular key gets node g minus the markers before it (m0, m1: the blob positions of the keys 0
// and ~0, or ~0), so the regular nodes are numbered consecutively in blob order; the markers take their fixed nodes.
// A key that is already there (a duplicate in the blob) sets *dup.
__global__ void __launch_bounds__(256) index_snap_import_kernel(IndexView ix, IndexCounters* ctr, const uint64_t* __restrict__ keys,
                                                                const uint32_t* __restrict__ rows, uint64_t n, uint64_t g0,
                                                                uint64_t m0, uint64_t m1, uint32_t We, uint32_t* dup) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t key = keys[i], g = g0 + i;
    uint32_t node;
    if (key_is_special(key)) {
      node = (uint32_t)(ix.C + (key == KEY_TOMB ? 1 : 0));
      if (atomicExch(ix.rmask + node, 1u)) atomicExch(dup, 1u);
    } else {
      node = (uint32_t)(g - (g > m0 ? 1 : 0) - (g > m1 ? 1 : 0));
      bool claimed = false;
      const uint32_t slot = table_find_or_claim(ix, ctr, key, &claimed);
      if (!claimed) {  // (a full table sets ctr->overflow instead)
        if (slot != SLOT_MISS) atomicExch(dup, 1u);
        continue;
      }
      ix.klog[node] = key;
      ix.node_of[slot] = node;
      ix.rmask[node] = 1u;
    }
    const uint32_t* src = rows + i * We;
    uint32_t* dst = ix.rows + ((uint64_t)node << ix.logW);
    uint32_t c = 0;
    for (uint32_t w = 0; w < We; ++w) {
      dst[w] = src[w];
      c += __popc(src[w]);
    }
    ix.cnt[node] = c;
  }
}

inline unsigned grid_for(uint64_t n) {
  uint64_t g = (n + 255) / 256;
  if (g > 132ull * 16) g = 132ull * 16;  // 16 CTAs per SM of an H100
  if (g == 0) g = 1;
  return (unsigned)g;
}

}  // namespace

cudaError_t launch_index_set(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t n, uint32_t ep_begin,
                             uint32_t ep_count, uint32_t rank, GossipLog log, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_set_kernel<false><<<grid_for(n), 256, 0, s>>>(ix, ctr, ops, nullptr, n, ep_begin, ep_count, rank, log);
  return cudaGetLastError();
}

cudaError_t launch_index_clear(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t n,
                               uint32_t ep_begin, uint32_t ep_count, uint32_t rank, GossipLog log, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_clear_kernel<false><<<grid_for(n), 256, 0, s>>>(ix, ctr, ops, nullptr, n, ep_begin, ep_count, rank, log, nullptr);
  return cudaGetLastError();
}

cudaError_t launch_index_clear_counted(IndexView ix, IndexCounters* ctr, const fi_index_op* ops, uint64_t cap,
                                       const unsigned long long* n_dev, uint32_t ep_begin, uint32_t ep_count, uint32_t rank,
                                       GossipLog log, cudaStream_t s) {
  if (cap == 0) return cudaSuccess;
  index_clear_kernel<false><<<grid_for(cap), 256, 0, s>>>(ix, ctr, ops, nullptr, cap, ep_begin, ep_count, rank, log, n_dev);
  return cudaGetLastError();
}

cudaError_t launch_index_remote_appear(IndexView ix, IndexCounters* ctr, const uint64_t* hashes, uint64_t n, uint32_t rank,
                                       cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_set_kernel<true><<<grid_for(n), 256, 0, s>>>(ix, ctr, nullptr, hashes, n, 0, 0, rank, GossipLog{});
  return cudaGetLastError();
}

cudaError_t launch_index_remote_vanish(IndexView ix, IndexCounters* ctr, const uint64_t* hashes, uint64_t n, uint32_t rank,
                                       cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_clear_kernel<true><<<grid_for(n), 256, 0, s>>>(ix, ctr, nullptr, hashes, n, 0, 0, rank, GossipLog{}, nullptr);
  return cudaGetLastError();
}

cudaError_t launch_index_rebuild(IndexView from, IndexView to, IndexCounters* ctr, cudaStream_t s) {
  index_rebuild_kernel<<<grid_for(from.C), 256, 0, s>>>(from, to, ctr);
  return cudaGetLastError();
}

cudaError_t launch_index_remove_sweep(IndexView ix, IndexCounters* ctr, const RemoveSet& rs, bool whole_rows, uint32_t rank,
                                      unsigned long long* removed, int sm_count, cudaStream_t s) {
  if (rs.m == 0) return cudaSuccess;
  // the node count is read on the device (ctr->used): one wave of resident CTAs strides over whatever it is
  auto kernel = whole_rows ? index_remove_rows_kernel : index_remove_words_kernel;
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0);
  if (e != cudaSuccess) return e;
  kernel<<<(unsigned)(sm_count * (per_sm > 0 ? per_sm : 1)), 256, 0, s>>>(ix, ctr, rs, 1u << rank, removed);
  return cudaGetLastError();
}

cudaError_t launch_index_contains(IndexView ix, const fi_index_op* q, uint64_t n, uint32_t ep_begin,
                                  uint32_t ep_count, uint8_t* out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_contains_kernel<<<grid_for(n), 256, 0, s>>>(ix, q, n, ep_begin, ep_count, out);
  return cudaGetLastError();
}

uint32_t index_snap_tiles(uint64_t n) { return (uint32_t)((n + 2 + kSnapTile - 1) / kSnapTile); }

cudaError_t launch_index_snap_count(IndexView ix, const IndexCounters* ctr, uint32_t* tile_live, cudaStream_t s) {
  index_snap_count_kernel<<<index_snap_tiles(ix.C), kSnapTile, 0, s>>>(ix, ctr, tile_live);
  return cudaGetLastError();
}

cudaError_t launch_index_snap_export(IndexView ix, uint64_t n, uint32_t t0, uint32_t t1, const uint64_t* tile_off, uint64_t base,
                                     uint32_t We, uint64_t* keys, uint32_t* rows, cudaStream_t s) {
  if (t1 <= t0) return cudaSuccess;
  index_snap_export_kernel<<<t1 - t0, kSnapTile, 0, s>>>(ix, n, t0, tile_off, base, We, keys, rows);
  return cudaGetLastError();
}

cudaError_t launch_index_snap_import(IndexView ix, IndexCounters* ctr, const uint64_t* keys, const uint32_t* rows, uint64_t n,
                                     uint64_t g0, uint64_t m0, uint64_t m1, uint32_t We, uint32_t* dup, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  index_snap_import_kernel<<<grid_for(n), 256, 0, s>>>(ix, ctr, keys, rows, n, g0, m0, m1, We, dup);
  return cudaGetLastError();
}

}  // namespace fi
