// counts_oracle.cpp — the CPU oracle's extension (tests/ext_oracle.cpp) with fi_epp_match_counts, test infrastructure
// only.
//
// It compiles the extension (and through it oracle/epp_oracle.cpp) into the same translation unit and adds the match
// counts of docs/SPEC.md S.3a.  Every epo_* and epx_* function works on its handles.  The counts come from the
// extension's own ranked pick (rank_one), so the walk of S.3 is the one the ranked and subset tests already check
// against, not a third copy of it: a probe that makes every endpoint a candidate and ranks all of the shard's
// endpoints reports each one's match_blocks.
#include "ext_oracle.cpp"

extern "C" {

// fi_epp_match_counts (S.3a): counts[r * cnt + j] = match[lo + j] of request r, nblocks[r] = N.  For the call the
// handle's configuration is one profile without filters or PD and its endpoints are all alive, so rank_one's one
// list holds every endpoint of the shard; configuration and states are restored before the call returns.  The count
// reads neither, as S.3a says.
int epx_match_counts(void* h, const uint8_t* prompts, const uint64_t* offsets, const uint64_t* h0, uint32_t R,
                     uint16_t* counts, uint32_t* nblocks) {
  if (!h) return FI_ERR_INVALID;
  ExtOracle* o = ext_of(h);
  const fi_epp_config saved_cfg = o->cfg;
  std::vector<EpState> saved_eps;
  saved_eps.swap(o->eps);
  o->eps.assign(saved_cfg.num_endpoints, EpState{});
  for (EpState& s : o->eps) s.flags = FI_ENDPOINT_ALIVE;
  fi_profile probe{};
  probe.n_scorers = 1;
  probe.scorers[0].kind = FI_SCORER_PREFIX;
  probe.scorers[0].weight = 1;
  o->cfg.n_profiles = 1;
  o->cfg.profiles[0] = probe;
  o->cfg.pd_enabled = 0;
  Scratch sc;
  std::vector<Ranked> cand;
  std::vector<fi_pick> list(o->cnt);
  for (uint32_t r = 0; r < R; ++r) {
    rank_one(*o, prompts + offsets[r], offsets[r + 1] - offsets[r], h0[r], 0, nullptr, r, o->cnt, list.data(), sc, cand);
    for (const fi_pick& pk : list) counts[(size_t)r * o->cnt + (pk.endpoint - o->lo)] = pk.match_blocks;
    nblocks[r] = list[0].n_blocks;
  }
  o->cfg = saved_cfg;
  o->eps.swap(saved_eps);
  return FI_OK;
}

}  // extern "C"
