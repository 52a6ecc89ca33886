// xxh64_sm100.cuh — the XXH64 arithmetic of xxh64.cuh (same functions, same results bit for bit) written on
// 32-bit halves for the SASS it should become on sm_90a.  Device only; xxh64.cuh stays the host/device
// definition the oracle-facing unit tests pin.
//
// Why: nvcc turns the 64-bit constant multiplies of a block into many more IMADs than they need (it splits the
// rotates into extra products and moves halves around with IMAD.MOV / IMAD.IADD), and the chain walk is
// issue-bound rather than latency-bound (tools/microbench/chainlat: two independent chains in one thread take
// twice as long as one).  Spelled as IMAD.WIDE + IMADs (addend folded in) and two funnel shifts per rotate, a
// block and a link take far fewer instructions.
#pragma once
#include <stdint.h>
#include "xxh64.cuh"

namespace fi {

// ---- products, rotates, the parallel part (stripes + merge) ---------------------------------------------
struct U2 {
  uint32_t lo, hi;
};
__device__ __forceinline__ U2 u2_of(uint64_t a) { return U2{(uint32_t)a, (uint32_t)(a >> 32)}; }
__device__ __forceinline__ uint64_t u64_of(U2 a) { return (uint64_t)a.lo | ((uint64_t)a.hi << 32); }
template <uint64_t P>
__device__ __forceinline__ U2 mulc(U2 x, U2 a) {  // x * P + a  (mod 2^64)
  U2 r;
  asm("{\n .reg .b64 t; .reg .b32 l, h;\n"
      " mov.b64 t, {%4, %5};\n"
      " mad.wide.u32 t, %2, %6, t;\n"
      " mov.b64 {l, h}, t;\n"
      " mad.lo.u32 h, %2, %7, h;\n"
      " mad.lo.u32 h, %3, %6, h;\n"
      " mov.b32 %0, l;\n mov.b32 %1, h;\n}"
      : "=r"(r.lo), "=r"(r.hi)
      : "r"(x.lo), "r"(x.hi), "r"(a.lo), "r"(a.hi), "n"((uint32_t)P), "n"((uint32_t)(P >> 32)));
  return r;
}
template <int R>
__device__ __forceinline__ U2 rotl2(U2 x) {
  static_assert(R > 0 && R < 32, "rotations used here are all below 32");
  return U2{__funnelshift_l(x.hi, x.lo, R), __funnelshift_l(x.lo, x.hi, R)};
}
__device__ __forceinline__ U2 xround2(U2 acc, U2 x) { return mulc<XP1>(rotl2<31>(mulc<XP2>(x, acc)), U2{0u, 0u}); }
__device__ __forceinline__ U2 xmerge2(U2 h, U2 v) {
  const U2 r = xround2(U2{0u, 0u}, v);
  return mulc<XP1>(U2{h.lo ^ r.lo, h.hi ^ r.hi}, u2_of(XP4));
}
struct XAcc2 {
  U2 v1, v2, v3, v4;
};
__device__ __forceinline__ XAcc2 xacc2_init() { return XAcc2{u2_of(XP1 + XP2), u2_of(XP2), u2_of(0), u2_of(0 - XP1)}; }
__device__ __forceinline__ uint64_t xacc2_finish(const XAcc2& a, uint64_t total_len) {
  const uint64_t s = u64_of(rotl2<1>(a.v1)) + u64_of(rotl2<7>(a.v2)) + u64_of(rotl2<12>(a.v3)) + u64_of(rotl2<18>(a.v4));
  U2 h = u2_of(s);
  h = xmerge2(h, a.v1);
  h = xmerge2(h, a.v2);
  h = xmerge2(h, a.v3);
  h = xmerge2(h, a.v4);
  return u64_of(h) + total_len;
}


// ---- the serial link --------------------------------------------------------------------------------------
// x * P + a with the high half as ONE three-input add of independent products: lo after 1 IMAD.WIDE, hi after
// IMAD + IADD3 (two dependent steps instead of three chained IMADs) — the form for the chain walker, where a lone
// warp per scheduler runs one dependency chain and the latency of every product is on the batch's critical path
template <uint64_t P>
__device__ __forceinline__ U2 mulc_par(U2 x, U2 a) {
  U2 r;
  asm("{\n .reg .b64 t; .reg .b32 l, h, c1, c2;\n"
      " mov.b64 t, {%4, %5};\n"
      " mad.wide.u32 t, %2, %6, t;\n"
      " mul.lo.u32 c1, %2, %7;\n"
      " mul.lo.u32 c2, %3, %6;\n"
      " mov.b64 {l, h}, t;\n"
      " add.u32 c1, c1, c2;\n"
      " add.u32 h, h, c1;\n"
      " mov.b32 %0, l;\n mov.b32 %1, h;\n}"
      : "=r"(r.lo), "=r"(r.hi)
      : "r"(x.lo), "r"(x.hi), "r"(a.lo), "r"(a.hi), "n"((uint32_t)P), "n"((uint32_t)(P >> 32)));
  return r;
}

//   h_i = avalanche( rotl(pre_i ^ round(0, h_{i-1}), 27)·P1 + P4 )      (xxh64.cuh chain_step)
__device__ __forceinline__ U2 chain_step2(U2 pre, U2 prev) {
  const U2 z{0u, 0u};
  U2 m = mulc_par<XP2>(prev, z);
  m = rotl2<31>(m);
  m = mulc_par<XP1>(m, z);
  U2 x{pre.lo ^ m.lo, pre.hi ^ m.hi};
  x = rotl2<27>(x);
  x = mulc_par<XP1>(x, u2_of(XP4));
  x.lo ^= x.hi >> 1;  // h ^= h >> 33
  x = mulc_par<XP2>(x, z);
  const uint32_t s_lo = __funnelshift_r(x.lo, x.hi, 29);  // h ^= h >> 29
  x.lo ^= s_lo;
  x.hi ^= x.hi >> 29;
  x = mulc_par<XP3>(x, z);
  x.lo ^= x.hi;  // h ^= h >> 32
  return x;
}

}  // namespace fi
