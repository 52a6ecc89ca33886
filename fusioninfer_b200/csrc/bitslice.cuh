// bitslice.cuh — per-endpoint match counters kept as bit-planes.
//
// One index row is a bitset over the local endpoints; a lane of the match kernel
// owns one 32-bit word of it (32 endpoints).  The per-endpoint match count
// (SURVEY.md Appendix A.3: res[p]++ for every block p holds) is accumulated for
// all 32 endpoints at once in NP bit-planes: plane j holds bit j of each of
// the 32 counters (NP = NPLANES = 10 counts up to 1023 blocks; the windowed match kernel
// keeps 12 for chains of up to FI_EPP_MAX_BLOCKS = 4095).  Words are added K at a time through a Harley–Seal
// carry-save tree: K-1 full adders (2 LOP3 each) plus one ripple of the final
// carry — ≈2.6 logic ops per row word at K=16 instead of 20 for a plain ripple.
#pragma once
#include <stdint.h>

#include "xxh64.cuh"  // FI_HD

namespace fi {

constexpr int NPLANES = 10;  // counts up to 1023 blocks: one match window (match_kernels.cu)

template <int NP = NPLANES>
struct BitCounter {
  uint32_t c[NP];
};

template <int NP>
FI_HD void bc_clear(BitCounter<NP>& b) {
#pragma unroll
  for (int i = 0; i < NP; ++i) b.c[i] = 0;
}

// add a carry word of weight 2^lvl
template <int LVL, int NP>
FI_HD void bc_ripple(BitCounter<NP>& b, uint32_t e) {
#pragma unroll
  for (int pl = LVL; pl < NP; ++pl) {
    uint32_t t = b.c[pl] & e;
    b.c[pl] ^= e;
    e = t;
  }
}

// Add K (power of two, 1..16) one-bit-per-endpoint words.  w is clobbered.
template <int K, int NP>
FI_HD void bc_add(BitCounter<NP>& b, uint32_t (&w)[K]) {
  static_assert(K == 1 || K == 2 || K == 4 || K == 8 || K == 16, "K must be a power of two <= 16");
  if (K >= 2) {
#pragma unroll
    for (int i = 0; i < K / 2; ++i) {
      uint32_t a = b.c[0], x = w[2 * i], y = w[(2 * i + 1) % K];
      b.c[0] = a ^ x ^ y;
      w[i] = (a & x) | (a & y) | (x & y);
    }
  }
  if (K >= 4) {
#pragma unroll
    for (int i = 0; i < K / 4; ++i) {
      uint32_t a = b.c[1], x = w[(2 * i) % K], y = w[(2 * i + 1) % K];
      b.c[1] = a ^ x ^ y;
      w[i] = (a & x) | (a & y) | (x & y);
    }
  }
  if (K >= 8) {
#pragma unroll
    for (int i = 0; i < K / 8; ++i) {
      uint32_t a = b.c[2], x = w[(2 * i) % K], y = w[(2 * i + 1) % K];
      b.c[2] = a ^ x ^ y;
      w[i] = (a & x) | (a & y) | (x & y);
    }
  }
  if (K >= 16) {
    uint32_t a = b.c[3], x = w[0], y = w[1 % K];
    b.c[3] = a ^ x ^ y;
    w[0] = (a & x) | (a & y) | (x & y);
  }
  if (K == 1) bc_ripple<0>(b, w[0]);
  if (K == 2) bc_ripple<1>(b, w[0]);
  if (K == 4) bc_ripple<2>(b, w[0]);
  if (K == 8) bc_ripple<3>(b, w[0]);
  if (K == 16) bc_ripple<4>(b, w[0]);
}

// b += o (bit-sliced ripple-carry addition of two counters)
template <int NP>
FI_HD void bc_merge(BitCounter<NP>& b, const BitCounter<NP>& o) {
  uint32_t carry = 0;
#pragma unroll
  for (int pl = 0; pl < NP; ++pl) {
    uint32_t x = b.c[pl], y = o.c[pl];
    b.c[pl] = x ^ y ^ carry;
    carry = (x & y) | (x & carry) | (y & carry);
  }
}

// endpoints (bits) whose count is non-zero
template <int NP>
FI_HD uint32_t bc_nonzero(const BitCounter<NP>& b) {
  uint32_t m = 0;
#pragma unroll
  for (int pl = 0; pl < NP; ++pl) m |= b.c[pl];
  return m;
}

// count of endpoint `bit` (0..31)
template <int NP>
FI_HD uint32_t bc_get(const BitCounter<NP>& b, uint32_t bit) {
  uint32_t v = 0;
#pragma unroll
  for (int pl = 0; pl < NP; ++pl) v |= ((b.c[pl] >> bit) & 1u) << pl;
  return v;
}

// out[j] = count of endpoint bit0 + j for j < NB (NB a power of two <= 32, bit0 + NB <= 32).  Two counts per pass
// over the planes: bit q and bit q + NB/2 are gathered into the low and high half of one word, so the transpose
// costs half of NB bc_get calls.
template <int NB, int NP>
FI_HD void bc_unpack(const BitCounter<NP>& b, uint32_t bit0, uint16_t* out) {
  static_assert(NB == 1 || NB == 2 || NB == 4 || NB == 8 || NB == 16 || NB == 32, "NB must be a power of two <= 32");
  if (NB == 1) {
    out[0] = (uint16_t)bc_get(b, bit0);
    return;
  }
  constexpr int H = NB > 1 ? NB / 2 : 1;
  uint32_t c[NP];
#pragma unroll
  for (int pl = 0; pl < NP; ++pl) c[pl] = b.c[pl] >> bit0;
#pragma unroll
  for (int q = 0; q < H; ++q) {
    uint32_t v = 0;
#pragma unroll
    for (int pl = 0; pl < NP; ++pl) {
      const uint32_t x = c[pl] >> q;
      v |= ((x & 1u) | ((x << (16 - H)) & 0x10000u)) << pl;
    }
    out[q] = (uint16_t)(v & 0xFFFFu);
    out[q + H] = (uint16_t)(v >> 16);
  }
}

}  // namespace fi
