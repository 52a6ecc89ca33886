// snapshot_format.h — the byte format of an index snapshot (fi_epp_snapshot_save / fi_epp_snapshot_load, docs/SPEC.md
// S.2d): its layout, size and checksum, and the structural check fi_epp_snapshot_info and the load run before anything
// reaches the device.  Pure C++ (unit-tested on the CPU through hostcheck.cpp).  Little-endian hosts only, like the
// rest of the C ABI.
//
// Version 1: a 64-byte header (SnapHeader), then the payload
//   caps[E] u32 | lru_len[E] u32 | lru_keys[n_lru] u64 (endpoint 0's keys LRU first, then endpoint 1's, ...)
//   | node_keys[n_nodes] u64 | node_rows[n_nodes][ceil(E / 32)] u32 (bit e % 32 of word e / 32: endpoint e holds it)
// The checksum is XXH64(header[0:56] ‖ LE64(XXH64(chunk_0)) ‖ LE64(XXH64(chunk_1)) ‖ ...) over the payload's 1 MiB
// chunks (seed 0 throughout), so that the chunks can be hashed in parallel.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "xxh64.cuh"

namespace fi {

constexpr char kSnapMagic[8] = {'F', 'I', 'E', 'P', 'P', 'S', 'N', 'P'};
constexpr uint32_t kSnapVersion = 1;
constexpr uint32_t kSnapHeaderBytes = 64;
constexpr uint64_t kSnapChunk = 1ull << 20;
constexpr uint64_t kSnapNone = ~0ull;  // snap_markers: no such key

struct SnapHeader {
  char magic[8];
  uint32_t version, header_bytes;
  uint32_t block_bytes, max_blocks, lru_capacity, num_endpoints;
  uint64_t n_nodes, n_lru, payload_bytes, checksum;
};
static_assert(sizeof(SnapHeader) == kSnapHeaderBytes, "the header is 64 bytes");
constexpr size_t kSnapHashedHeader = offsetof(SnapHeader, checksum);  // 56

// words per membership row in a snapshot: ceil(E / 32), not the handle's power-of-two width
inline uint32_t snap_row_words(uint32_t num_endpoints) { return (num_endpoints + 31) / 32; }

// byte offsets of the payload's sections (from the payload's start); `end` is the payload size
struct SnapLayout {
  uint64_t caps, lru_len, lru_keys, node_keys, node_rows, end;
};
inline SnapLayout snap_layout(uint32_t num_endpoints, uint64_t n_nodes, uint64_t n_lru) {
  SnapLayout l;
  l.caps = 0;
  l.lru_len = 4ull * num_endpoints;
  l.lru_keys = 8ull * num_endpoints;
  l.node_keys = l.lru_keys + 8 * n_lru;
  l.node_rows = l.node_keys + 8 * n_nodes;
  l.end = l.node_rows + 4ull * snap_row_words(num_endpoints) * n_nodes;
  return l;
}

inline uint64_t snap_rd64(const uint8_t* p) {
  uint64_t v;
  std::memcpy(&v, p, 8);
  return v;
}

// XXH64 (seed 0) of a byte string, with word loads (xxh64_bytes reads a virtual message byte by byte)
inline uint64_t snap_xxh64(const uint8_t* p, uint64_t len) {
  uint64_t i = 0, h;
  if (len >= 32) {
    XAcc a = xacc_init();
    do {
      xacc_stripe(a, snap_rd64(p + i), snap_rd64(p + i + 8), snap_rd64(p + i + 16), snap_rd64(p + i + 24));
      i += 32;
    } while (i + 32 <= len);
    h = xacc_finish(a, len);
  } else {
    h = XP5 + len;
  }
  for (; i + 8 <= len; i += 8) {
    h ^= xround(0, snap_rd64(p + i));
    h = rotl64(h, 27) * XP1 + XP4;
  }
  if (i + 4 <= len) {
    uint32_t v;
    std::memcpy(&v, p + i, 4);
    h ^= (uint64_t)v * XP1;
    h = rotl64(h, 23) * XP2 + XP3;
    i += 4;
  }
  for (; i < len; ++i) {
    h ^= (uint64_t)p[i] * XP5;
    h = rotl64(h, 11) * XP1;
  }
  return xavalanche(h);
}

// fn(i) for i in [0, n) on up to `threads` host threads, in contiguous ranges
template <class Fn>
void snap_parallel(uint64_t n, unsigned threads, Fn&& fn) {
  const uint64_t t = threads < 1 ? 1 : threads > n ? (n ? n : 1) : threads;
  if (t <= 1) {
    for (uint64_t i = 0; i < n; ++i) fn(i);
    return;
  }
  std::vector<std::thread> pool;
  for (uint64_t k = 0; k < t; ++k)
    pool.emplace_back([&, k] {
      for (uint64_t i = n * k / t; i < n * (k + 1) / t; ++i) fn(i);
    });
  for (auto& th : pool) th.join();
}

// the checksum of a snapshot whose header's first 56 bytes are `header` and whose payload is `payload`
inline uint64_t snap_checksum(const void* header, const void* payload, uint64_t payload_bytes, unsigned threads) {
  const uint64_t chunks = (payload_bytes + kSnapChunk - 1) / kSnapChunk;
  std::vector<uint8_t> outer(kSnapHashedHeader + 8 * chunks);
  std::memcpy(outer.data(), header, kSnapHashedHeader);
  const uint8_t* p = static_cast<const uint8_t*>(payload);
  snap_parallel(chunks, threads, [&](uint64_t c) {
    const uint64_t off = c * kSnapChunk, n = payload_bytes - off < kSnapChunk ? payload_bytes - off : kSnapChunk;
    const uint64_t v = snap_xxh64(p + off, n);
    std::memcpy(outer.data() + kSnapHashedHeader + 8 * c, &v, 8);
  });
  return snap_xxh64(outer.data(), outer.size());
}

// The structural check: everything S.2d asks of a well-formed blob except that keys are distinct.  On success *out is
// the header and *pairs the total popcount of the rows; else *why says what is wrong.
inline bool snap_check(const void* buf, uint64_t len, unsigned threads, SnapHeader* out, uint64_t* pairs, std::string* why) {
  SnapHeader hd;
  if (len < kSnapHeaderBytes) return *why = "snapshot shorter than its header", false;
  std::memcpy(&hd, buf, sizeof(hd));
  if (std::memcmp(hd.magic, kSnapMagic, 8) != 0) return *why = "not a snapshot (magic)", false;
  if (hd.version != kSnapVersion)
    return *why = "snapshot format version " + std::to_string(hd.version) + " (this library reads version 1)", false;
  if (hd.header_bytes != kSnapHeaderBytes) return *why = "snapshot header size is not 64", false;
  const uint32_t E = hd.num_endpoints;
  if (E == 0 || E > 4096) return *why = "snapshot num_endpoints out of range", false;
  const uint64_t room = len - kSnapHeaderBytes;
  if (hd.n_nodes > room / 8 || hd.n_lru > room / 8) return *why = "snapshot counts exceed its length", false;
  const SnapLayout l = snap_layout(E, hd.n_nodes, hd.n_lru);
  if (hd.payload_bytes != l.end) return *why = "snapshot payload size does not match its counts", false;
  if (room != l.end) return *why = "snapshot length does not match its header (truncated or padded)", false;
  const uint8_t* p = static_cast<const uint8_t*>(buf) + kSnapHeaderBytes;
  if (snap_checksum(buf, p, l.end, threads) != hd.checksum) return *why = "snapshot checksum mismatch", false;
  std::vector<uint32_t> caps(E), lens(E);
  std::memcpy(caps.data(), p + l.caps, 4ull * E);
  std::memcpy(lens.data(), p + l.lru_len, 4ull * E);
  uint64_t total = 0;
  for (uint32_t e = 0; e < E; ++e) {
    const bool cap_ok = hd.lru_capacity ? caps[e] >= hd.max_blocks && caps[e] <= hd.lru_capacity : caps[e] == 0;
    if (!cap_ok) return *why = "snapshot LRU capacity of endpoint " + std::to_string(e) + " out of range", false;
    if (lens[e] > caps[e]) return *why = "snapshot LRU of endpoint " + std::to_string(e) + " above its capacity", false;
    total += lens[e];
  }
  if (total != hd.n_lru) return *why = "snapshot LRU lengths do not add up to n_lru", false;
  // rows: non-empty, no bit at or above E
  const uint32_t We = snap_row_words(E);
  const uint32_t last = E % 32 ? (1u << (E % 32)) - 1u : ~0u;
  const uint64_t parts = threads ? threads : 1;
  std::vector<uint64_t> pc(parts, 0), bad(parts, kSnapNone);
  snap_parallel(parts, threads, [&](uint64_t k) {
    const uint8_t* rows = p + l.node_rows;
    for (uint64_t i = hd.n_nodes * k / parts; i < hd.n_nodes * (k + 1) / parts; ++i) {
      uint32_t row[128];
      std::memcpy(row, rows + 4ull * We * i, 4ull * We);
      uint64_t c = 0;
      for (uint32_t w = 0; w < We; ++w) c += (uint64_t)__builtin_popcount(row[w]);
      if (c == 0 || (row[We - 1] & ~last)) {
        bad[k] = i;
        return;
      }
      pc[k] += c;
    }
  });
  uint64_t sum = 0;
  for (uint64_t k = 0; k < parts; ++k) {
    if (bad[k] != kSnapNone) return *why = "snapshot row " + std::to_string(bad[k]) + " is empty or names an endpoint >= E", false;
    sum += pc[k];
  }
  *out = hd;
  *pairs = sum;
  return true;
}

// The positions of the keys 0 and ~0 (the index's marker keys) among n node keys; false if either appears twice
inline bool snap_markers(const uint8_t* node_keys, uint64_t n, uint64_t* pos0, uint64_t* pos1) {
  *pos0 = *pos1 = kSnapNone;
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t k = snap_rd64(node_keys + 8 * i);
    if (k != 0 && k != ~0ull) continue;
    uint64_t* at = k ? pos1 : pos0;
    if (*at != kSnapNone) return false;
    *at = i;
  }
  return true;
}

}  // namespace fi
