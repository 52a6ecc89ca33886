// xxh64.cuh — XXH64 arithmetic shared by the sm_90a kernels and the host side of
// libfi_epp (chain seed h0, host unit checks).  Pure integer; no tensor cores.
//
// Follows the public xxHash specification (SURVEY.md Appendix A.7), the function
// upstream's prefix plugin applies through github.com/cespare/xxhash/v2
// (/root/reference/go.mod:27).  The chain construction is SURVEY.md Appendix A.1.
//
// Split used by the GPU path for block_bytes % 32 == 0 (e.g. 64 B = 16 uint32
// tokens): the message of block i is  block_i ‖ LE64(h_{i-1})  (block_bytes + 8
// bytes).  All 32-byte stripes, the merge and "+= len" depend on block_i only
// (block_prestate — embarrassingly parallel, >85 % of the multiplies); h_{i-1}
// enters through one 8-byte tail step and the avalanche (chain_step — the only
// serial part).
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define FI_HD __host__ __device__ __forceinline__
#else
#define FI_HD inline
#endif

namespace fi {

constexpr uint64_t XP1 = 0x9E3779B185EBCA87ULL;
constexpr uint64_t XP2 = 0xC2B2AE3D27D4EB4FULL;
constexpr uint64_t XP3 = 0x165667B19E3779F9ULL;
constexpr uint64_t XP4 = 0x85EBCA77C2B2AE63ULL;
constexpr uint64_t XP5 = 0x27D4EB2F165667C5ULL;

FI_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
FI_HD uint64_t xround(uint64_t acc, uint64_t x) { return rotl64(acc + x * XP2, 31) * XP1; }
FI_HD uint64_t xmerge(uint64_t h, uint64_t v) { return (h ^ xround(0, v)) * XP1 + XP4; }
FI_HD uint64_t xavalanche(uint64_t h) {
  h ^= h >> 33;
  h *= XP2;
  h ^= h >> 29;
  h *= XP3;
  h ^= h >> 32;
  return h;
}

// Stripe accumulators for seed 0.
struct XAcc {
  uint64_t v1, v2, v3, v4;
};
FI_HD XAcc xacc_init() { return XAcc{XP1 + XP2, XP2, 0, 0 - XP1}; }
FI_HD void xacc_stripe(XAcc& a, uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3) {
  a.v1 = xround(a.v1, w0);
  a.v2 = xround(a.v2, w1);
  a.v3 = xround(a.v3, w2);
  a.v4 = xround(a.v4, w3);
}
// merge + "h += total_len": the state right before the tail of a message whose
// length is a multiple of 32 plus `tail` bytes (total_len counts the tail).
FI_HD uint64_t xacc_finish(const XAcc& a, uint64_t total_len) {
  uint64_t h = rotl64(a.v1, 1) + rotl64(a.v2, 7) + rotl64(a.v3, 12) + rotl64(a.v4, 18);
  h = xmerge(h, a.v1);
  h = xmerge(h, a.v2);
  h = xmerge(h, a.v3);
  h = xmerge(h, a.v4);
  return h + total_len;
}

// Serial link of the chain for block_bytes % 32 == 0:
//   h_i = avalanche( rotl(pre_i ^ round(0, h_{i-1}), 27)·P1 + P4 )
FI_HD uint64_t chain_step(uint64_t pre, uint64_t prev) {
  uint64_t h = pre ^ xround(0, prev);
  h = rotl64(h, 27) * XP1 + XP4;
  return xavalanche(h);
}

// Generic XXH64 (seed 0) over a "virtual" message  block ‖ LE64(prev)  read
// through byte loads; used for block sizes that are not a multiple of 32 (the
// reference's own blockSize: 5, /root/reference/pkg/router/strategy.go:57) and
// for h0 on the host.  `blk` may be unaligned.
struct ChainMsg {
  const uint8_t* blk;
  uint32_t blk_len;
  uint64_t prev;
  bool has_prev;
  FI_HD uint64_t len() const { return (uint64_t)blk_len + (has_prev ? 8u : 0u); }
  FI_HD uint32_t byte(uint64_t j) const {
    return j < blk_len ? (uint32_t)blk[j] : (uint32_t)((prev >> (8 * (j - blk_len))) & 0xFF);
  }
  FI_HD uint64_t rd64(uint64_t j) const {
    uint64_t v = 0;
    for (int t = 0; t < 8; ++t) v |= (uint64_t)byte(j + t) << (8 * t);
    return v;
  }
  FI_HD uint32_t rd32(uint64_t j) const {
    uint32_t v = 0;
    for (int t = 0; t < 4; ++t) v |= byte(j + t) << (8 * t);
    return v;
  }
};

FI_HD uint64_t xxh64_msg(const ChainMsg& m) {
  const uint64_t len = m.len();
  uint64_t p = 0, h;
  if (len >= 32) {
    XAcc a = xacc_init();
    do {
      xacc_stripe(a, m.rd64(p), m.rd64(p + 8), m.rd64(p + 16), m.rd64(p + 24));
      p += 32;
    } while (p + 32 <= len);
    h = xacc_finish(a, len);
  } else {
    h = XP5 + len;
  }
  while (p + 8 <= len) {
    h ^= xround(0, m.rd64(p));
    h = rotl64(h, 27) * XP1 + XP4;
    p += 8;
  }
  if (p + 4 <= len) {
    h ^= (uint64_t)m.rd32(p) * XP1;
    h = rotl64(h, 23) * XP2 + XP3;
    p += 4;
  }
  while (p < len) {
    h ^= (uint64_t)m.byte(p) * XP5;
    h = rotl64(h, 11) * XP1;
    ++p;
  }
  return xavalanche(h);
}

// plain XXH64(seed 0) of a byte string (host: chain seed h0 = XXH64(model ‖ salt))
FI_HD uint64_t xxh64_bytes(const uint8_t* p, uint32_t len) {
  ChainMsg m{p, len, 0, false};
  return xxh64_msg(m);
}

}  // namespace fi
