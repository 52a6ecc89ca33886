"""CPU: the shard view of the oracle (docs/SPEC.md S.2e) — what a single-rank handle over endpoints [b, b + c) of the
pool computes, the yardstick of tests/test_gpu_shard_handle.py.

  * The C++ view (tests/ext_oracle.cpp, ExtOracle(cfg, shard=...)) equals the independent Python restatement's
    (tests/restate.py), in both match modes, with PD, LoRA, label filters, dead endpoints and the LRU.
  * Composition: the shard views of a partition of the pool, merged by (score desc, rotation asc) — the rule of the
    sharded mode's merge — equal the unsharded oracle, single and ranked picks, queue scorer included, in LPM mode and
    in UPSTREAM mode on a prefix-closed index.  On an UPSTREAM index with holes they need not: a shard's walk stops at
    the first block no endpoint OF THE SHARD holds, which is why a sharded pool keeps a directory of the whole pool.
"""
import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests import restate
from tests import shard_view as SV
from tests.ext_oracle import ExtOracle

P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
PROFILES = [{"name": "a", "scorers": [(P, 100), (K, 10), (Q, 10)]},
            {"name": "b", "role_mask": 3, "more_filters": [6], "scorers": [(P, 20), (Q, 7)]},
            {"name": "c", "role_mask": 4, "scorers": [(K, 3), (P, 50)]}]


def _lora(E, rng):
    lo = np.zeros(E, dtype=abi.lora_dtype())
    lo["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 3)), int(rng.integers(0, 2))
        ids = rng.permutation(6)[: na + nw] + 1000
        lo[e]["n_active"], lo[e]["n_waiting"], lo[e]["max_active"] = na, nw, int(rng.integers(0, 4))
        lo[e]["active"][:na] = ids[:na]
        lo[e]["waiting"][:nw] = ids[na:]
    return lo


def _cold(offs, n=12, nbytes=20):
    """the first n requests become prompts shorter than one block"""
    offs = offs.copy()
    offs[1:n + 1] = offs[0] + np.arange(1, n + 1, dtype=np.uint64) * nbytes
    return offs


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", ["plain", "pd", "lora"])
def test_shard_view_equals_restatement(mode, variant):
    rng = np.random.default_rng(11 + mode)
    wl = H.small_workload(E=37, R=64, T=256, holes=True, lru_capacity=40, groups_per_endpoint=2)
    profiles = [dict(p) for p in PROFILES]
    pd = None
    if variant == "pd":
        pd = {"decode": 0, "prefill": 2, "threshold": 0.5 * wl.T * 4}
    if variant == "lora":
        profiles[0] = {"name": "a", "scorers": [(P, 60), (L, 30), (Q, 10)]}
    cfg = H.config_for(wl, profiles=profiles, pd=pd, match_mode=mode, lru_capacity=40)
    st = SV.tie_states(wl.E, rng)
    lo = _lora(wl.E, rng) if variant == "lora" else None
    ops = list(wl.index_ops())
    tok, offs = wl.prompts()
    offs = _cold(offs)
    ad = (rng.integers(0, 8, wl.R) + 1000).astype(np.uint64) if lo is not None else None
    full = ExtOracle(cfg)
    full.update_endpoints(st)
    for o in ops:
        full.index_apply(o)
    chains, nb = full.hash_batch(tok, offs, wl.h0)
    for b, c in [(0, 1), (1, 32), (33, 4), (5, 12), (0, 37), (36, 1)]:
        cpp = ExtOracle(cfg, shard=(b, c))
        py = restate.from_config(cfg, shard=(b, c))
        for x in (cpp, py):
            x.update_endpoints(st)
        if lo is not None:
            cpp.update_endpoints_lora(lo)
            py.update_lora(lo)
        for o in ops:
            cpp.index_apply(o)
            py.apply(o)
        got, want = cpp.pick_batch(tok, offs, wl.h0, adapters=ad), py.pick(tok, offs, wl.h0, ad)
        assert H.picks_equal(got, want), f"shard {(b, c)}\n" + H.describe_diff(got, want)
        real = got["endpoint"][got["endpoint"] != abi.FI_NO_ENDPOINT]
        assert ((real >= b) & (real < b + c)).all()
        # Adds across the pool: only the shard's own endpoints learn
        dest = rng.integers(0, wl.E, wl.R).astype(np.uint32)
        cpp.index_add_chains(dest, chains, nb)
        for r in range(wl.R):
            py.add_chain(int(dest[r]), chains[r, : nb[r]])
        for e in range(wl.E):
            assert len(cpp.lru(e)) == (len(py.lru.get(e, ())) if b <= e < b + c else 0)
            assert cpp.lru(e).tolist() == list(py.lru.get(e, {}).keys())
        got = cpp.pick_batch(tok, offs, wl.h0, adapters=ad)
        assert H.picks_equal(got, py.pick(tok, offs, wl.h0, ad)), f"shard {(b, c)} after Adds"
        cpp.close()


def _composition_setup(mode, holes, E=70, seed=3):
    rng = np.random.default_rng(seed)
    wl = H.small_workload(E=E, R=96, T=256, holes=holes, lru_capacity=64, groups_per_endpoint=2)
    cfg = H.config_for(wl, profiles=PROFILES, match_mode=mode, lru_capacity=64)
    st = SV.tie_states(wl.E, rng)
    st["queue_depth"] = rng.integers(0, 40, wl.E)  # the queue scorer's min / max sit in some shard, not in others
    ops = list(wl.index_ops())
    tok, offs = wl.prompts()
    return wl, cfg, st, ops, tok, _cold(offs)


@pytest.mark.parametrize("mode", MODES)
def test_shard_views_compose_into_the_pool(mode):
    """LPM, and UPSTREAM on a prefix-closed index: the merged shard views equal the unsharded oracle, single picks and
    ranked lists, with the queue scorer, before and after Adds aimed across the pool"""
    wl, cfg, st, ops, tok, offs = _composition_setup(mode, holes=mode == abi.FI_MATCH_LPM)
    dest = np.random.default_rng(5).integers(0, wl.E, wl.R).astype(np.uint32)
    for parts in SV.splits(wl.E):
        assert [b for b, _ in parts] == [0] + list(np.cumsum([c for _, c in parts]))[:-1]
        assert sum(c for _, c in parts) == wl.E
        full = ExtOracle(cfg)
        views = [ExtOracle(cfg, shard=bc) for bc in parts]
        for x in [full] + views:
            x.update_endpoints(st)
            for o in ops:
                x.index_apply(o)
        chains, nb = full.hash_batch(tok, offs, wl.h0)
        starts = SV.starts(chains, nb, wl.h0, wl.E)
        for step in ("before", "after the Adds"):
            want = full.pick_batch(tok, offs, wl.h0)
            got = SV.merge_single([v.pick_batch(tok, offs, wl.h0) for v in views], starts, wl.E)
            assert H.picks_equal(got, want), f"{parts} {step}\n" + H.describe_diff(got, want)
            for k in (1, 5, 16):
                want = full.pick_batch_ranked(tok, offs, wl.h0, k)
                got = SV.merge_ranked([v.pick_batch_ranked(tok, offs, wl.h0, k) for v in views], starts, wl.E)
                assert H.picks_equal(got, want), f"{parts} k {k} {step}\n" + H.describe_diff(got, want)
            for x in [full] + views:
                x.index_add_chains(dest, chains, nb)
        for x in [full] + views:
            x.close()


def test_upstream_holes_do_not_compose():
    """e0 holds blocks 0 and 2 of a prompt, e1 (another shard) blocks 0 and 1.  The pool's UPSTREAM walk reaches block
    2 through e1's block 1, so e0 matches 2 blocks; e0's shard stops at block 1, which no endpoint of its own holds,
    and matches 1.  The merged shard views then differ from the pool: the sharded mode needs its directory."""
    wl = H.small_workload(E=2, R=1, T=64, max_blocks=4)
    cfg = H.config_for(wl, profiles=[{"name": "d", "scorers": [(P, 100)]}])
    full = ExtOracle(cfg)
    tok, offs = wl.prompts()
    chains, nb = full.hash_batch(tok, offs, wl.h0)
    assert nb[0] == 4
    ops = H.ops_array([(int(chains[0, 0]), 0, 1), (int(chains[0, 2]), 0, 1),
                       (int(chains[0, 0]), 1, 1), (int(chains[0, 1]), 1, 1)])
    st = H.states_array(2)
    views = [ExtOracle(cfg, shard=(0, 1)), ExtOracle(cfg, shard=(1, 1))]
    for x in [full] + views:
        x.update_endpoints(st)
        x.index_apply(ops)
    want = full.pick_batch(tok, offs, wl.h0)
    assert [int(x) for x in want[0]["match_blocks"]] == [2]
    starts = SV.starts(chains, nb, wl.h0, 2)
    got = SV.merge_single([v.pick_batch(tok, offs, wl.h0) for v in views], starts, 2)
    assert views[0].pick_batch(tok, offs, wl.h0)[0, 0]["match_blocks"] == 1
    assert not H.picks_equal(got, want)
    # the LPM walk is per endpoint: there the views compose
    cfg.match_mode = abi.FI_MATCH_LPM
    full, views = ExtOracle(cfg), [ExtOracle(cfg, shard=(0, 1)), ExtOracle(cfg, shard=(1, 1))]
    for x in [full] + views:
        x.update_endpoints(st)
        x.index_apply(ops)
    got = SV.merge_single([v.pick_batch(tok, offs, wl.h0) for v in views], starts, 2)
    assert H.picks_equal(got, full.pick_batch(tok, offs, wl.h0))


def test_shard_view_drops_what_is_addressed_elsewhere():
    """ops, Adds, capacity changes and removals aimed outside the shard leave it as it was; a range outside the pool
    is refused, and so are a resize and the snapshot state (the product refuses them on a handle over part of the
    pool)"""
    wl = H.small_workload(E=40, R=8, T=1024, lru_capacity=80, groups_per_endpoint=1)
    cfg = H.config_for(wl, lru_capacity=80)
    with pytest.raises(ValueError):
        ExtOracle(cfg, shard=(30, 11))
    with pytest.raises(ValueError):
        ExtOracle(cfg, shard=(3, 0))
    v = ExtOracle(cfg, shard=(10, 5), track_removal=True)
    v.update_endpoints(H.states_array(wl.E))
    tok, offs = wl.prompts()
    chains, nb = v.hash_batch(tok, offs, wl.h0)
    assert (nb == wl.max_blocks).all()
    v.index_apply(H.ops_array([(int(chains[0, 0]), 3, 1), (int(chains[0, 0]), 12, 1)]))
    assert not v.index_contains(3, int(chains[0, 0])) and v.index_contains(12, int(chains[0, 0]))
    v.index_add_chain(30, chains[1])
    assert v.lru_size(30) == 0 and not v.index_contains(30, int(chains[1, 0]))
    v.index_add_chains([11, 30, 11], chains[1:4], nb[1:4])
    assert v.lru_size(11) == 2 * wl.max_blocks and v.lru_size(30) == 0
    assert v.set_lru_capacities([30, 11], [wl.max_blocks, wl.max_blocks]) == [(int(h), 11) for h in chains[1]]
    v.remove_endpoints([3, 30])
    assert v.index_contains(12, int(chains[0, 0])) and v.lru_size(11) == min(nb[1], wl.max_blocks)
    v.remove_endpoints([12])
    assert not v.index_contains(12, int(chains[0, 0]))
    for call in (lambda: v.resize(wl.E + 1), v.state, lambda: v.load_state(set(), [[]] * wl.E, [80] * wl.E)):
        with pytest.raises(ValueError):
            call()
    assert v._lib.epx_resize(v._h, wl.E + 1) == abi.FI_ERR_STATE
    assert v._lib.epx_load_state(v._h, 0, None, None, None, None, None) == abi.FI_ERR_STATE
    assert v.lru_size(11) == min(nb[1], wl.max_blocks) and v.capacities()[11] == wl.max_blocks
    v.close()
