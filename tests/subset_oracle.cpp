// subset_oracle.cpp — CPU reference of the subset pick (docs/SPEC.md S.5a), test infrastructure only.
//
// It compiles the CPU oracle (oracle/epp_oracle.cpp) into the same translation unit and adds one entry point,
// epo_pick_batch_subset: the ranked pick of S.6a over each request's candidate subset, built from the oracle's own
// hashing, index, eligibility, scoring and tie-rotation pieces.  The oracle itself is left as it is.
#include "../oracle/epp_oracle.cpp"

#include <algorithm>

namespace {

struct Ranked {
  double total;
  uint32_t dist;  // tie rotation distance (smaller first among equal totals)
  uint32_t e;
  uint32_t match;
};

inline bool in_subset(const uint32_t* row, uint32_t e) { return !row || ((row[e >> 5] >> (e & 31)) & 1u); }

// One request: hash → match (A.3) over the WHOLE pool, exactly as pick_one does (the walk stops at the first block
// no endpoint of the pool holds, whatever the subset).  Then per profile: the eligible endpoints of the subset, the
// queue scorer's min / max over them (S.4 per request), their totals (A.4), ordered by (total desc, rotation
// distance asc), and the PD rule on the decode profile's entry 0 (A.6).
void subset_one(const Oracle& o, const uint8_t* prompt, uint64_t len, uint64_t h0, uint64_t adapter,
                const uint32_t* row, uint32_t r, uint32_t k, fi_pick* out, Scratch& sc, std::vector<Ranked>& cand) {
  const fi_epp_config& cfg = o.cfg;
  const uint32_t E = cfg.num_endpoints;
  sc.chain.resize(cfg.max_blocks);
  const uint32_t n = hash_prompt(prompt, len, h0, cfg.block_bytes, cfg.max_blocks, sc.chain.data(), sc.tmp);
  if (sc.match.size() != E) sc.match.assign(E, 0);
  sc.touched.clear();
  if (cfg.match_mode == FI_MATCH_UPSTREAM) {
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t* m = nullptr;
      const uint32_t cnt = o.index.get(sc.chain[i], &m);
      if (cnt == 0) break;
      for (uint32_t j = 0; j < cnt; ++j)
        if (sc.match[m[j]]++ == 0) sc.touched.push_back(m[j]);
    }
  } else {
    sc.alive.clear();
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t* m = nullptr;
      const uint32_t cnt = o.index.get(sc.chain[i], &m);
      if (cnt == 0) break;
      if (i == 0) {
        sc.alive.assign(m, m + cnt);
      } else {
        sc.alive2.clear();
        for (uint32_t a : sc.alive)
          if (std::find(m, m + cnt, a) != m + cnt) sc.alive2.push_back(a);
        sc.alive.swap(sc.alive2);
      }
      if (sc.alive.empty()) break;
      for (uint32_t a : sc.alive)
        if (sc.match[a]++ == 0) sc.touched.push_back(a);
    }
  }

  const uint32_t start = tie_rotation_start(n, n ? sc.chain[0] : 0, h0, r, E);
  for (uint32_t p = 0; p < cfg.n_profiles; ++p) {
    const fi_profile& prof = cfg.profiles[p];
    ProfileCtx ctx;  // make_ctx over the request's eligible candidates
    for (uint32_t e = 0; e < E; ++e) {
      const EpState& es = o.eps[e];
      if (!eligible(es, prof) || !in_subset(row, e)) continue;
      if (!ctx.any) {
        ctx.min_q = ctx.max_q = es.queue_depth;
        ctx.any = true;
      } else {
        ctx.min_q = std::min(ctx.min_q, es.queue_depth);
        ctx.max_q = std::max(ctx.max_q, es.queue_depth);
      }
    }
    cand.clear();
    for (uint32_t e = 0; e < E; ++e) {
      const EpState& es = o.eps[e];
      if (!eligible(es, prof) || !in_subset(row, e)) continue;
      cand.push_back({total_score(prof, ctx, es, sc.match[e], n, adapter), tie_distance(e, start, E), e, sc.match[e]});
    }
    const size_t kk = std::min<size_t>(k, cand.size());
    std::partial_sort(cand.begin(), cand.begin() + kk, cand.end(), [](const Ranked& a, const Ranked& b) {
      return a.total > b.total || (a.total == b.total && a.dist < b.dist);
    });
    for (uint32_t j = 0; j < k; ++j) {
      fi_pick& pk = out[(size_t)p * k + j];
      pk.n_blocks = (uint16_t)n;
      if (j < kk) {
        pk.endpoint = cand[j].e;
        pk.match_blocks = (uint16_t)cand[j].match;
        pk.score = cand[j].total;
      } else {
        pk.endpoint = FI_NO_ENDPOINT;
        pk.match_blocks = 0;
        pk.score = 0.0;
      }
    }
  }
  if (cfg.pd_enabled) {
    const fi_pick& d = out[(size_t)cfg.pd_decode_profile * k];
    const double hit = (d.endpoint != FI_NO_ENDPOINT && n) ? (double)d.match_blocks / (double)n : 0.0;
    const double miss_bytes = (1.0 - hit) * (double)len;
    if (!(miss_bytes >= cfg.pd_threshold)) {
      for (uint32_t j = 0; j < k; ++j) {
        fi_pick& pf = out[(size_t)cfg.pd_prefill_profile * k + j];
        pf.endpoint = FI_NO_ENDPOINT;
        pf.match_blocks = 0;
        pf.score = 0.0;
      }
    }
  }
  for (uint32_t e : sc.touched) sc.match[e] = 0;
}

}  // namespace

extern "C" {

// subsets: R rows of ceil(num_endpoints / 32) words (bit e of row r: e is a candidate of request r), or NULL
// (every request unrestricted).  out: R*n_profiles*k picks, out[(r*n_profiles + p)*k + j]; adapters may be NULL.
int epo_pick_batch_subset(void* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0,
                          const uint64_t* adapters, const uint32_t* subsets, uint32_t R, uint32_t k, fi_pick* out) {
  if (!h || k == 0) return FI_ERR_INVALID;
  const Oracle* o = (const Oracle*)h;
  const uint32_t P = o->cfg.n_profiles;
  const size_t pitch = (o->cfg.num_endpoints + 31) / 32;
  Scratch sc;
  std::vector<Ranked> cand;
  for (uint32_t r = 0; r < R; ++r)
    subset_one(*o, prompts + offsets[r], offsets[r + 1] - offsets[r], h0[r], adapters ? adapters[r] : 0,
               subsets ? subsets + r * pitch : nullptr, r, k, out + (size_t)r * P * k, sc, cand);
  return FI_OK;
}

}  // extern "C"
