// hostcheck.cpp — host build of the arithmetic the kernels share with the CPU
// (xxh64.cuh, bitslice.cuh) and of the host LRU, exported for CPU unit tests
// (tests/test_host_logic.py).  Not part of libfi_epp.so and never used to serve a pick.
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <set>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "bitslice.cuh"
#include "lru.h"
#include "lru_batch.h"
#include "lru_plan.h"
#include "pool_shape.h"
#include "snapshot_format.h"
#include "tiebreak.cuh"
#include "xxh64.cuh"

namespace {

template <int NP>
void bitcount(const uint32_t* words, uint32_t n, uint32_t K, uint32_t* counts) {
  fi::BitCounter<NP> b;
  fi::bc_clear(b);
  for (uint32_t i = 0; i < n; i += K) {
    uint32_t w[16] = {0};
    for (uint32_t j = 0; j < K && i + j < n; ++j) w[j] = words[i + j];
    switch (K) {
      case 1: { uint32_t t[1] = {w[0]}; fi::bc_add<1>(b, t); break; }
      case 2: { uint32_t t[2] = {w[0], w[1]}; fi::bc_add<2>(b, t); break; }
      case 4: { uint32_t t[4]; std::memcpy(t, w, sizeof(t)); fi::bc_add<4>(b, t); break; }
      case 8: { uint32_t t[8]; std::memcpy(t, w, sizeof(t)); fi::bc_add<8>(b, t); break; }
      default: { uint32_t t[16]; std::memcpy(t, w, sizeof(t)); fi::bc_add<16>(b, t); break; }
    }
  }
  for (uint32_t bit = 0; bit < 32; ++bit) counts[bit] = fi::bc_get(b, bit);
}

template <int NP>
int bc_unpack_check(const uint32_t* planes, uint32_t bit0, uint32_t nb, uint16_t* out_unpack, uint16_t* out_get) {
  if (bit0 + nb > 32) return -1;
  fi::BitCounter<NP> b;
  for (int pl = 0; pl < NP; ++pl) b.c[pl] = planes[pl];
  switch (nb) {
    case 1: fi::bc_unpack<1>(b, bit0, out_unpack); break;
    case 2: fi::bc_unpack<2>(b, bit0, out_unpack); break;
    case 4: fi::bc_unpack<4>(b, bit0, out_unpack); break;
    case 8: fi::bc_unpack<8>(b, bit0, out_unpack); break;
    case 16: fi::bc_unpack<16>(b, bit0, out_unpack); break;
    case 32: fi::bc_unpack<32>(b, bit0, out_unpack); break;
    default: return -1;
  }
  for (uint32_t j = 0; j < nb; ++j) out_get[j] = (uint16_t)fi::bc_get(b, bit0 + j);
  return 0;
}

template <int NP>
void bitcount_merge(const uint32_t* wa, uint32_t na, const uint32_t* wb, uint32_t nb, uint32_t* counts, uint32_t* nonzero) {
  fi::BitCounter<NP> a, b;
  fi::bc_clear(a);
  fi::bc_clear(b);
  for (uint32_t i = 0; i < na; ++i) { uint32_t t[1] = {wa[i]}; fi::bc_add<1>(a, t); }
  for (uint32_t i = 0; i < nb; ++i) { uint32_t t[1] = {wb[i]}; fi::bc_add<1>(b, t); }
  fi::bc_merge(a, b);
  for (uint32_t bit = 0; bit < 32; ++bit) counts[bit] = fi::bc_get(a, bit);
  *nonzero = fi::bc_nonzero(a);
}

}  // namespace

extern "C" {

uint64_t fihc_xxh64(const uint8_t* p, uint32_t len) { return fi::xxh64_bytes(p, len); }

// chain via the generic virtual-message path (any block size)
uint32_t fihc_chain_generic(const uint8_t* p, uint64_t len, uint64_t h0, uint32_t B, uint32_t M, uint64_t* out) {
  uint64_t nb = len / B;
  if (nb > M) nb = M;
  uint64_t h = h0;
  for (uint64_t i = 0; i < nb; ++i) {
    fi::ChainMsg m{p + i * B, B, h, true};
    h = fi::xxh64_msg(m);
    out[i] = h;
  }
  return (uint32_t)nb;
}

// chain via the split pre-state / chain_step path (B % 32 == 0), as the GPU fast path does
uint32_t fihc_chain_split(const uint8_t* p, uint64_t len, uint64_t h0, uint32_t B, uint32_t M, uint64_t* out) {
  if (B % 32) return 0;
  uint64_t nb = len / B;
  if (nb > M) nb = M;
  uint64_t h = h0;
  for (uint64_t i = 0; i < nb; ++i) {
    fi::XAcc a = fi::xacc_init();
    for (uint32_t s = 0; s < B / 32; ++s) {
      uint64_t w[4];
      std::memcpy(w, p + i * B + 32 * s, 32);
      fi::xacc_stripe(a, w[0], w[1], w[2], w[3]);
    }
    const uint64_t pre = fi::xacc_finish(a, (uint64_t)B + 8);
    h = fi::chain_step(pre, h);
    out[i] = h;
  }
  return (uint32_t)nb;
}

// bit-sliced counting: add n words K at a time (zero padded), return the 32 counts
void fihc_bitcount(const uint32_t* words, uint32_t n, uint32_t K, uint32_t* counts) { bitcount<fi::NPLANES>(words, n, K, counts); }

// bc_unpack<nb>(planes, bit0) and bc_get of the same bits: out_unpack[j], out_get[j] for j < nb; -1 for an nb that is
// not a power of two <= 32 or a range past bit 31
int fihc_bc_unpack(const uint32_t* planes, uint32_t bit0, uint32_t nb, uint16_t* out_unpack, uint16_t* out_get) {
  return bc_unpack_check<fi::NPLANES>(planes, bit0, nb, out_unpack, out_get);
}

// merge of two counters built from two word streams
void fihc_bitcount_merge(const uint32_t* wa, uint32_t na, const uint32_t* wb, uint32_t nb, uint32_t* counts,
                         uint32_t* nonzero) {
  bitcount_merge<fi::NPLANES>(wa, na, wb, nb, counts, nonzero);
}

// the same three with the 12 bit-planes of the windowed match kernel (counts up to 4095)
void fihc_bitcount12(const uint32_t* words, uint32_t n, uint32_t K, uint32_t* counts) { bitcount<12>(words, n, K, counts); }
int fihc_bc_unpack12(const uint32_t* planes, uint32_t bit0, uint32_t nb, uint16_t* out_unpack, uint16_t* out_get) {
  return bc_unpack_check<12>(planes, bit0, nb, out_unpack, out_get);
}
void fihc_bitcount_merge12(const uint32_t* wa, uint32_t na, const uint32_t* wb, uint32_t nb, uint32_t* counts,
                           uint32_t* nonzero) {
  bitcount_merge<12>(wa, na, wb, nb, counts, nonzero);
}

// tie rotation (tiebreak.cuh): start of a request's rotation, rotated distance of an endpoint, and the first
// member of a local tie set (bit words) in rotation order — the per-word arithmetic the match kernel uses
uint32_t fihc_tie_start(uint32_t n_blocks, uint64_t first_hash, uint64_t h0, uint32_t r, uint32_t E) {
  return fi::tie_start(fi::tie_seed(n_blocks, first_hash, h0, r), E);
}
uint32_t fihc_tie_rot(uint32_t e, uint32_t start, uint32_t E) { return fi::tie_rot(e, start, E); }
uint32_t fihc_tie_first_local(const uint32_t* words, uint32_t W, uint32_t start, uint32_t ep_begin, uint32_t ep_count) {
  const uint32_t p = fi::tie_local_origin(start, ep_begin, ep_count);
  const uint32_t mask = W * 32u - 1u;
  uint32_t best = 0xFFFFFFFFu;
  for (uint32_t wi = 0; wi < W; ++wi) {
    const uint32_t d = fi::tie_word_min(words[wi], wi, p, mask);
    if (d < best) best = d;
  }
  return best == 0xFFFFFFFFu ? 0xFFFFFFFFu : ((best + p) & mask);
}

// LRU trace: for each key report (inserted, did_evict, evicted)
void* fihc_lru_new(uint32_t cap) { return new fi::LruSet(cap); }
void fihc_lru_free(void* l) { delete (fi::LruSet*)l; }
uint32_t fihc_lru_size(void* l) { return ((fi::LruSet*)l)->size(); }
int fihc_lru_contains(void* l, uint64_t k) { return ((fi::LruSet*)l)->contains(k) ? 1 : 0; }
void fihc_lru_clear(void* l) { ((fi::LruSet*)l)->clear(); }
void fihc_lru_touch(void* l, const uint64_t* keys, uint32_t n, uint8_t* inserted, uint8_t* did_evict, uint64_t* evicted) {
  fi::LruSet* s = (fi::LruSet*)l;
  for (uint32_t i = 0; i < n; ++i) {
    bool d = false;
    uint64_t ev = 0;
    inserted[i] = s->touch(keys[i], &ev, &d) ? 1 : 0;
    did_evict[i] = d ? 1 : 0;
    evicted[i] = ev;
  }
}

// LruSet::shrink: set the limit, write the evicted keys (oldest first, at most cap); returns how many were evicted
uint32_t fihc_lru_shrink(void* l, uint32_t limit, uint64_t* evicted, uint32_t cap) {
  uint32_t n = 0;
  ((fi::LruSet*)l)->shrink(limit, [&](uint64_t k) {
    if (n < cap) evicted[n] = k;
    ++n;
  });
  return n;
}
uint32_t fihc_lru_limit(void* l) { return ((fi::LruSet*)l)->limit(); }
// the keys, least recently used first (at most cap written); returns the size
uint32_t fihc_lru_dump(void* l, uint64_t* out, uint32_t cap) {
  uint32_t n = 0;
  ((fi::LruSet*)l)->for_each_oldest_first([&](uint64_t k) {
    if (n < cap) out[n] = k;
    ++n;
  });
  return n;
}

// A pool of host LRUs with per-endpoint limits, walked batch by batch with lru_walk_batch (fi_epp_index_add_chains'
// host phase) and resized with LruSet::shrink (fi_epp_set_lru_capacities): tests/test_lru_capacity_cpu.py drives it
// against a sequential model.
struct HcLruPool {
  std::vector<fi::LruSet> lrus;
  fi::WorkerPool pool;
  std::vector<fi::WorkerOps> outs;
  HcLruPool(uint32_t E, uint32_t cap, uint32_t workers) : lrus(E, fi::LruSet(cap)), pool(workers) {}
};
void* fihc_lrupool_new(uint32_t E, uint32_t cap, uint32_t workers) { return new HcLruPool(E, cap, workers); }
void fihc_lrupool_free(void* p) { delete (HcLruPool*)p; }
uint32_t fihc_lrupool_shrink(void* p, uint32_t e, uint32_t limit, uint64_t* evicted, uint32_t cap) {
  return fihc_lru_shrink(&((HcLruPool*)p)->lrus[e], limit, evicted, cap);
}
uint32_t fihc_lrupool_dump(void* p, uint32_t e, uint64_t* out, uint32_t cap) {
  return fihc_lru_dump(&((HcLruPool*)p)->lrus[e], out, cap);
}
// one batch of Adds; the ops in the order the engine applies them (segment by segment, a segment's SETs before its
// CLEARs), at most cap written; returns how many there are
uint64_t fihc_lrupool_walk(void* p, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch, const uint32_t* nblocks,
                           uint32_t R, fi_index_op* ops, uint64_t cap) {
  HcLruPool& hp = *(HcLruPool*)p;
  const size_t nseg = fi::lru_walk_batch(hp.lrus, 0, (uint32_t)hp.lrus.size(), endpoints, chains, pitch, nblocks, R, hp.pool, hp.outs);
  uint64_t n = 0;
  for (size_t s = 0; s < nseg; ++s)
    for (int kind = 0; kind < 2; ++kind)
      for (auto& o : hp.outs) {
        if (s >= o.nseg) continue;
        for (const fi_index_op& op : kind == 0 ? o.sets[s] : o.clears[s]) {
          if (n < cap) ops[n] = op;
          ++n;
        }
      }
  return n;
}

// plan_staging (lru_batch.h) of W workers' ops given by counts: worker w used wseg[w] <= nseg segments, and
// counts[(w * nseg + s) * 2 + kind] is how many SETs (kind 0) / CLEARs (kind 1) it has in segment s.  Writes each
// piece as 7 words (group, worker, seg, clear, src, n, dst), at most piece_cap of them, and each group's fill
// (n_sets, n_clears), at most group_cap groups; *n_pieces = pieces.  Returns the number of groups.
uint64_t fihc_plan_staging(uint32_t W, uint32_t nseg, const uint32_t* wseg, const uint64_t* counts, uint64_t ns0, uint64_t nc0,
                           uint64_t chunk, uint64_t* pieces, uint64_t piece_cap, uint64_t* fills, uint64_t group_cap,
                           uint64_t* n_pieces) {
  std::vector<fi::WorkerOps> outs(W);
  for (uint32_t w = 0; w < W; ++w)
    for (uint32_t s = 0; s < wseg[w]; ++s) {
      outs[w].sets_of(s).resize(counts[((size_t)w * nseg + s) * 2]);
      outs[w].clears_of(s).resize(counts[((size_t)w * nseg + s) * 2 + 1]);
    }
  const std::vector<fi::StageGroup> groups = fi::plan_staging(outs, nseg, ns0, nc0, chunk);
  uint64_t n = 0;
  for (size_t g = 0; g < groups.size(); ++g) {
    if (g < group_cap) {
      fills[2 * g] = groups[g].n_sets;
      fills[2 * g + 1] = groups[g].n_clears;
    }
    for (const fi::StagePiece& p : groups[g].pieces) {
      if (n < piece_cap) {
        const uint64_t row[7] = {g, p.worker, p.seg, p.clear, p.src, p.n, p.dst};
        std::memcpy(pieces + 7 * n, row, sizeof(row));
      }
      ++n;
    }
  }
  *n_pieces = n;
  return groups.size();
}

// One fi_epp_index_add_chains on a pool: walk the batch, plan its staging behind an open group of ns0 SETs and nc0
// CLEARs, and write the ops in the order they are staged, each with its group (ops[i], group[i]; at most cap).
// Returns how many ops there are; *n_groups = groups (the last one, the tail, stays open).
uint64_t fihc_lrupool_stage(void* p, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch, const uint32_t* nblocks,
                            uint32_t R, uint64_t ns0, uint64_t nc0, uint64_t chunk, fi_index_op* ops, uint32_t* group, uint64_t cap,
                            uint64_t* n_groups) {
  HcLruPool& hp = *(HcLruPool*)p;
  const size_t nseg = fi::lru_walk_batch(hp.lrus, 0, (uint32_t)hp.lrus.size(), endpoints, chains, pitch, nblocks, R, hp.pool, hp.outs);
  const std::vector<fi::StageGroup> groups = fi::plan_staging(hp.outs, nseg, ns0, nc0, chunk);
  uint64_t n = 0;
  for (uint32_t g = 0; g < groups.size(); ++g)
    for (const fi::StagePiece& sp : groups[g].pieces) {
      const fi::WorkerOps& o = hp.outs[sp.worker];
      const fi_index_op* src = (sp.clear ? o.clears : o.sets)[sp.seg].data() + sp.src;
      for (size_t i = 0; i < sp.n; ++i, ++n)
        if (n < cap) {
          ops[n] = src[i];
          group[n] = g;
        }
    }
  *n_groups = groups.size();
  return n;
}

// fi_epp_index_add_chains' host phase (lru_batch.h) against the sequential definition: walk the batch on
// `workers` threads, apply the resulting ops segment by segment (all SETs of a segment, then all its CLEARs — the
// way the GPU applies a group) to a membership set, and compare that set and the LRU contents with one LRU per
// endpoint touched request after request.  Returns 0 if identical, else a code; *segments = segments used.
int fihc_lru_batch_check(uint32_t E, uint32_t cap, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch,
                         const uint32_t* nblocks, uint32_t R, uint32_t batches, uint32_t workers, uint32_t* segments) {
  std::vector<fi::LruSet> par(E, fi::LruSet(cap)), seq(E, fi::LruSet(cap));
  fi::WorkerPool pool(workers);
  std::vector<fi::WorkerOps> outs;
  std::vector<std::vector<uint64_t>> member_par(E), member_seq(E);  // sorted membership per endpoint
  auto has = [](std::vector<uint64_t>& v, uint64_t k) { return std::binary_search(v.begin(), v.end(), k); };
  auto add = [&](std::vector<uint64_t>& v, uint64_t k) {
    auto it = std::lower_bound(v.begin(), v.end(), k);
    if (it == v.end() || *it != k) v.insert(it, k);
  };
  auto del = [&](std::vector<uint64_t>& v, uint64_t k) {
    auto it = std::lower_bound(v.begin(), v.end(), k);
    if (it != v.end() && *it == k) v.erase(it);
  };
  (void)has;
  uint32_t max_seg = 0;
  for (uint32_t b = 0; b < batches; ++b) {
    const uint32_t* ep = endpoints + (size_t)b * R;
    const uint64_t* ch = chains + (size_t)b * R * pitch;
    const uint32_t* nb = nblocks + (size_t)b * R;
    const size_t nseg = fi::lru_walk_batch(par, 0, E, ep, ch, pitch, nb, R, pool, outs);
    if (nseg > max_seg) max_seg = (uint32_t)nseg;
    for (size_t sgi = 0; sgi < nseg; ++sgi) {
      for (auto& o : outs)
        if (sgi < o.nseg)
          for (auto& op : o.sets[sgi]) add(member_par[op.endpoint], op.hash);
      for (auto& o : outs)
        if (sgi < o.nseg)
          for (auto& op : o.clears[sgi]) del(member_par[op.endpoint], op.hash);
    }
    for (uint32_t r = 0; r < R; ++r) {
      if (ep[r] == FI_NO_ENDPOINT || ep[r] >= E) continue;
      for (uint32_t i = 0; i < nb[r]; ++i) {
        uint64_t ev = 0;
        bool did = false;
        const uint64_t k = ch[(size_t)r * pitch + i];
        const bool ins = seq[ep[r]].touch(k, &ev, &did);
        if (ins) add(member_seq[ep[r]], k);
        if (did) del(member_seq[ep[r]], ev);
      }
    }
    for (uint32_t e = 0; e < E; ++e) {
      if (member_par[e] != member_seq[e]) return 1;
      if (par[e].size() != seq[e].size() || par[e].size() != member_seq[e].size()) return 2;
      for (uint64_t k : member_seq[e])
        if (!par[e].contains(k)) return 3;
    }
  }
  if (segments) *segments = max_seg;
  return 0;
}

// The device LRU's batch rule (lru_kernels.cu) on the CPU: plan the batch with lru_plan_batch (at most plan_cap
// touches per endpoint and sub-batch: the LRU capacity in the conservative pass, unlimited in the optimistic one),
// apply every sub-batch AT ONCE — per endpoint: the keys touched move behind everything else in the order of
// their LAST touch, then the oldest entries beyond the capacity go — and compare recency order and content with
// one LRU per endpoint touched request after request.  0 if identical; *subs = sub-batches of the last batch.
int fihc_lru_plan_check(uint32_t E, uint32_t cap, const uint32_t* endpoints, const uint64_t* chains, uint32_t pitch,
                        const uint32_t* nblocks, uint32_t R, uint32_t batches, uint32_t plan_cap, uint64_t cap_touches,
                        uint32_t cap_requests, uint32_t* subs) {
  std::vector<std::vector<uint64_t>> order(E);  // oldest first
  std::vector<fi::LruSet> seq(E, fi::LruSet(cap));
  std::vector<std::vector<uint64_t>> seq_order(E);
  fi::LruPlan pl;
  for (uint32_t b = 0; b < batches; ++b) {
    const uint32_t* ep = endpoints + (size_t)b * R;
    const uint64_t* ch = chains + (size_t)b * R * pitch;
    const uint32_t* nb = nblocks + (size_t)b * R;
    fi::lru_plan_batch(ep, nb, R, 0, E, plan_cap, cap_touches, cap_requests, &pl);
    if (subs) *subs = (uint32_t)pl.subs.size();
    size_t covered = 0;
    for (size_t sb = 0; sb < pl.subs.size(); ++sb) {
      const fi::LruSubBatch& s = pl.subs[sb];
      if (s.k_end - s.k_begin > cap_requests || s.touches > cap_touches) return 10;
      const uint32_t* st = pl.ep_start.data() + sb * ((size_t)E + 1);
      const uint32_t* inc = pl.inc.data() + sb * (size_t)E;
      for (uint32_t e = 0; e < E; ++e) {
        // touches of endpoint e in this sub-batch, in request order
        std::vector<uint64_t> t;
        uint32_t last_k = 0;
        for (uint32_t i = st[e]; i < st[e + 1]; ++i) {
          const uint32_t k = s.k_begin + pl.ep_list[s.k_begin + i];
          if (i > st[e] && k <= last_k) return 11;  // ascending
          last_k = k;
          if (pl.req_ep[k] != e) return 12;
          const uint64_t* c = ch + (size_t)pl.req_id[k] * pitch;
          t.insert(t.end(), c, c + pl.req_n[k]);
        }
        if (t.size() != inc[e] || t.size() > plan_cap) return 13;
        covered += t.size();
        std::unordered_set<uint64_t> seen;
        std::vector<uint64_t> winners;  // keys by last touch, newest first
        for (size_t i = t.size(); i-- > 0;)
          if (seen.insert(t[i]).second) winners.push_back(t[i]);
        std::vector<uint64_t>& o = order[e];
        o.erase(std::remove_if(o.begin(), o.end(), [&](uint64_t k) { return seen.count(k) != 0; }), o.end());
        o.insert(o.end(), winners.rbegin(), winners.rend());
        if (o.size() > cap) o.erase(o.begin(), o.begin() + (o.size() - cap));
      }
    }
    size_t want_cov = 0;
    for (uint32_t r = 0; r < R; ++r) {
      if (ep[r] >= E) continue;
      want_cov += nb[r];
      for (uint32_t i = 0; i < nb[r]; ++i) {
        const uint64_t k = ch[(size_t)r * pitch + i];
        uint64_t ev = 0;
        bool did = false;
        const bool ins = seq[ep[r]].touch(k, &ev, &did);
        std::vector<uint64_t>& so = seq_order[ep[r]];
        if (!ins) so.erase(std::find(so.begin(), so.end(), k));
        so.push_back(k);
        if (did) so.erase(std::find(so.begin(), so.end(), ev));
      }
    }
    if (covered != want_cov) return 14;
    for (uint32_t e = 0; e < E; ++e)
      if (order[e] != seq_order[e]) return 1;
  }
  return 0;
}

// lru_touch_bound (lru_plan.h): the per-endpoint touches a sub-batch of fi_epp_index_add_submitted may carry
uint32_t fihc_lru_touch_bound(uint32_t TS, uint32_t C) { return fi::lru_touch_bound(TS, C); }

// The packed plan (lru_plan.h) read back the way the engine hands it to the LRU kernels: plan each batch with
// lru_plan_batch, pack it with lru_plan_pack, and read every sub-batch's arrays through lru_plan_offsets.  They must
// equal the LruPlan vectors, and the sub-batches' sections must cover the lru_plan_words packed words exactly once.
// 0 if so, else a code; *subs = sub-batches in total.
int fihc_lru_plan_pack_check(uint32_t E, const uint32_t* endpoints, const uint32_t* nblocks, uint32_t R, uint32_t batches,
                             uint32_t plan_cap, uint64_t cap_touches, uint32_t cap_requests, uint32_t* subs) {
  const uint32_t kGuard = 0xA5A5A5A5u;
  fi::LruPlan pl;
  uint32_t nsubs = 0;
  for (uint32_t b = 0; b < batches; ++b) {
    fi::lru_plan_batch(endpoints + (size_t)b * R, nblocks + (size_t)b * R, R, 0, E, plan_cap, cap_touches, cap_requests, &pl);
    nsubs += (uint32_t)pl.subs.size();
    const size_t words = fi::lru_plan_words(pl, E);
    std::vector<uint32_t> packed(words + 1, kGuard);
    fi::lru_plan_pack(pl, packed.data());
    if (packed[words] != kGuard) return 1;  // wrote past the end
    std::vector<uint32_t> seen(words, 0);
    auto same = [&](size_t at, const uint32_t* want, size_t n) {
      for (size_t i = 0; i < n; ++i) {
        if (at + i >= words || packed[at + i] != want[i]) return false;
        seen[at + i]++;
      }
      return true;
    };
    for (size_t sb = 0; sb < pl.subs.size(); ++sb) {
      const uint32_t k0 = pl.subs[sb].k_begin, nk = pl.subs[sb].k_end - k0;
      const fi::LruPlanOffsets o = fi::lru_plan_offsets(pl, E, sb);
      if (!same(o.req_id, pl.req_id.data() + k0, nk)) return 2;
      if (!same(o.req_ep, pl.req_ep.data() + k0, nk)) return 3;
      if (!same(o.req_n, pl.req_n.data() + k0, nk)) return 4;
      if (!same(o.req_off, pl.req_off.data() + k0, nk)) return 5;
      if (!same(o.ep_list, pl.ep_list.data() + k0, nk)) return 6;
      if (!same(o.ep_start, pl.ep_start.data() + sb * ((size_t)E + 1), (size_t)E + 1)) return 7;
      if (!same(o.inc, pl.inc.data() + sb * (size_t)E, E)) return 8;
    }
    for (uint32_t s : seen)
      if (s != 1) return 9;
  }
  if (subs) *subs = nsubs;
  return 0;
}

// The device LRU's table occupancy under plans cut with lru_touch_bound: per endpoint, `used` (regular slots taken:
// entries + tombstones) follows lru_maintain_kernel's rule before every sub-batch (kept if (used + min(add, C)) * 10
// <= 6 TS, else rebuilt to the live entries), then every key the sub-batch touches that is not an entry takes a slot,
// and the LRU keeps the C most recent keys (what falls out becomes a tombstone: used stays).  The touch kernel reserves
// a slot before it looks further, so up to `add` reservations can be outstanding at once: it cannot fail iff
// used_before + add <= TS * 85 / 100.  Returns 0 if that holds for every endpoint and sub-batch, else 1; *max_pct =
// the highest used_before + add seen, in percent of TS; *subs = sub-batches in total.
int fihc_lru_bound_check(uint32_t E, uint32_t cap, uint32_t TS, const uint32_t* endpoints, const uint64_t* chains,
                         uint32_t pitch, const uint32_t* nblocks, uint32_t R, uint32_t batches, uint64_t cap_touches,
                         uint32_t cap_requests, double* max_pct, uint32_t* subs) {
  const uint64_t limit = (uint64_t)TS * 85 / 100;
  const uint32_t bound = fi::lru_touch_bound(TS, cap);
  std::vector<fi::LruSet> lru(E, fi::LruSet(cap));
  std::vector<uint64_t> used(E, 0);
  fi::LruPlan pl;
  uint64_t peak = 0, nsubs = 0;
  for (uint32_t b = 0; b < batches; ++b) {
    const uint32_t* ep = endpoints + (size_t)b * R;
    const uint64_t* ch = chains + (size_t)b * R * pitch;
    const uint32_t* nb = nblocks + (size_t)b * R;
    fi::lru_plan_batch(ep, nb, R, 0, E, bound, cap_touches, cap_requests, &pl);
    nsubs += pl.subs.size();
    for (size_t sb = 0; sb < pl.subs.size(); ++sb) {
      const uint32_t* inc = pl.inc.data() + sb * (size_t)E;
      const fi::LruSubBatch& s = pl.subs[sb];
      for (uint32_t e = 0; e < E; ++e) {
        const uint64_t add = inc[e];
        if (!add) continue;
        const uint64_t addc = std::min<uint64_t>(add, cap);
        if ((used[e] + addc) * 10 > (uint64_t)TS * 6) used[e] = lru[e].size();
        peak = std::max(peak, used[e] + add);
        if (used[e] + add > limit) return 1;
      }
      std::set<std::pair<uint32_t, uint64_t>> fresh;  // (endpoint, key) pairs new to their endpoint in this sub-batch
      for (uint32_t k = s.k_begin; k < s.k_end; ++k) {
        const uint32_t e = pl.req_ep[k];
        const uint64_t* c = ch + (size_t)pl.req_id[k] * pitch;
        for (uint32_t i = 0; i < pl.req_n[k]; ++i)
          if (!lru[e].contains(c[i]) && fresh.insert({e, c[i]}).second) used[e]++;
      }
      for (uint32_t k = s.k_begin; k < s.k_end; ++k) {
        const uint32_t e = pl.req_ep[k];
        const uint64_t* c = ch + (size_t)pl.req_id[k] * pitch;
        for (uint32_t i = 0; i < pl.req_n[k]; ++i) {
          uint64_t ev = 0;
          bool did = false;
          lru[e].touch(c[i], &ev, &did);
        }
      }
    }
  }
  if (max_pct) *max_pct = 100.0 * (double)peak / TS;
  if (subs) *subs = (uint32_t)nsubs;
  return 0;
}

// the index shape of a pool (pool_shape.h), as fi_epp_create and fi_epp_resize_pool derive it
uint32_t fihc_pool_row_words(uint32_t endpoint_count) { return fi::pool_row_words(endpoint_count); }
uint64_t fihc_pool_default_slots(uint32_t num_endpoints, uint32_t lru_capacity) {
  return fi::pool_default_slots(num_endpoints, lru_capacity);
}
uint64_t fihc_pool_resized_slots(uint64_t pinned, uint32_t num_endpoints, uint32_t lru_capacity, uint64_t live_keys) {
  return fi::pool_resized_slots(pinned, num_endpoints, lru_capacity, live_keys);
}
int fihc_pool_needs_rebuild(uint32_t W, uint64_t slots, uint32_t new_W, uint64_t new_slots) {
  return fi::pool_needs_rebuild(W, slots, new_W, new_slots) ? 1 : 0;
}

// the snapshot format (snapshot_format.h): its checksum and its structural check (0: well-formed; *pairs = popcount)
uint64_t fihc_snap_xxh64(const uint8_t* p, uint64_t len) { return fi::snap_xxh64(p, len); }
uint64_t fihc_snap_checksum(const uint8_t* blob, uint64_t len, unsigned threads) {
  return fi::snap_checksum(blob, blob + fi::kSnapHeaderBytes, len - fi::kSnapHeaderBytes, threads);
}
int fihc_snap_check(const uint8_t* blob, uint64_t len, unsigned threads, uint64_t* pairs) {
  fi::SnapHeader hd;
  std::string why;
  return fi::snap_check(blob, len, threads, &hd, pairs, &why) ? 0 : -1;
}
int fihc_snap_markers(const uint8_t* keys, uint64_t n, uint64_t* pos) { return fi::snap_markers(keys, n, pos, pos + 1) ? 0 : -1; }

}  // extern "C"
