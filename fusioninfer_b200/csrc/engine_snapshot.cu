// engine_snapshot.cu — index snapshots (docs/SPEC.md S.2d): save, capture, read, load and info.
#include "engine.h"
#include "snapshot_format.h"

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
  int rc = check_whole_pool(h, what);
  if (rc != FI_OK) return rc;
  if (h->cfg.lru_capacity) {
    rc = choose_lru_mode(h);
    if (rc != FI_OK) return rc;
    if (h->lru_mode == 0) return fail(h, FI_ERR_STATE, std::string(what) + ": the host LRU serves the handle");
  }
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

extern "C" {

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
    return fail(h, alloc_status(e),
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
    if (e != cudaSuccess) return alloc_status(e);
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

  rc = replace_begin(h);
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
  if (e != cudaSuccess) return fail(h, alloc_status(e), std::string("snapshot staging: ") + cudaGetErrorString(e));
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
  h->ctr_used_known = regular;
  h->ctr_unchecked = 0;
  // (the host LRU sets are empty, lru_mode != 0: they only take the capacities)
  return replace_commit(h, &nix, nlru, caps);
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

}  // extern "C"
