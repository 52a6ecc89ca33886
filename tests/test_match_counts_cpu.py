"""CPU: the oracle of fi_epp_match_counts (docs/SPEC.md S.3a), the yardstick of tests/test_gpu_match_counts.py.

  * ExtOracle.match_counts equals the independent restatement's match (tests/restate.py) in both match modes, on
    indices built from SET / CLEAR ops with holes, from LRU Adds that evict chain fronts and from removals, at block
    sizes 5 and 64, on the whole pool and on shard views.
  * Every pick and ranked entry of the oracle, over filters, every scorer kind, LoRA and PD, reports the matrix's
    count at its endpoint.
  * Shard-view matrices of a partition, side by side, are the pool's matrix in LPM mode and in UPSTREAM mode on a
    prefix-closed index; on an UPSTREAM index with a hole they need not be.
  * bc_unpack (bitslice.cuh), the kernel's transpose of the bit-plane counters, equals bc_get.
"""
import ctypes as C
import os

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests import match_counts_cases as MC
from tests import restate
from tests import shard_view as SV
from tests.ext_oracle import ExtOracle

P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
NO = abi.FI_NO_ENDPOINT


def _cfg(E, B, M, R, mode, lru=0, profiles=None, pd=None, **kw):
    return H.make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=lru, max_batch=R, index_slots=1 << 14,
                         match_mode=mode, profiles=profiles or [{"name": "d", "scorers": [(P, 100)]}], pd=pd, **kw)


def _restated_matrix(py, chains, nb, cols):
    out = np.zeros((len(nb), len(cols)), dtype=np.uint16)
    for r in range(len(nb)):
        m = py.match([int(h) for h in chains[r, : nb[r]]])
        out[r] = [m.get(e, 0) for e in cols]
    return out


def _build(x, how, chains, nb, E, seed, py=False):
    """apply one of the index constructions of tests/match_counts_cases.py to an oracle (py: the restatement)"""
    rng = np.random.default_rng(seed)
    if how in ("ops", "ops+remove"):
        for o in MC.family_ops(chains, nb, E, rng):
            x.apply(o) if py else x.index_apply(o)
    else:
        for dest, ch, n in MC.add_batches(chains, nb, E, rng):
            for r in range(len(n)):
                if dest[r] == NO:
                    continue
                x.add_chain(int(dest[r]), ch[r, : n[r]]) if py else x.index_add_chain(int(dest[r]), ch[r, : n[r]])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [5, 64])
@pytest.mark.parametrize("how", ["ops", "adds", "ops+remove"])
@pytest.mark.parametrize("shard", [None, (0, 1), (3, 33), (20, 17)])
def test_matrix_equals_restatement(mode, B, how, shard):
    E, R, M = 37, 96, 24
    rng = np.random.default_rng(7 + B)
    tok, offs = MC.prompts(R, B, M, rng)
    lru = 2 * M if how != "ops" else 0  # below what three batches of Adds touch: chain fronts are evicted
    cfg = _cfg(E, B, M, R, mode, lru=lru)
    o = ExtOracle(cfg, shard=shard, track_removal=how == "ops+remove")
    py = restate.from_config(cfg, shard=shard)
    chains, nb = o.hash_batch(tok, offs, 0x1234)
    _build(o, how, chains, nb, E, seed=B + mode)
    _build(py, how, chains, nb, E, seed=B + mode, py=True)
    if how == "ops+remove":
        gone = [1, 4, 20, 36]
        o.remove_endpoints(gone)
        for h in py.index.values():
            h.difference_update(gone)
    counts, n = o.match_counts(tok, offs, 0x1234)
    cols = list(py.own)
    assert (n == nb).all()
    want = _restated_matrix(py, chains, nb, cols)
    assert counts.shape == (R, len(cols))
    assert np.array_equal(counts, want), np.argwhere(counts != want)[:5]
    if shard is None:
        assert MC.unique_counts(counts) > 3 and (counts == 0).any()
    o.close()


PROFILE_SETS = {
    "filters": ([{"name": "a", "scorers": [(P, 100), (K, 10), (Q, 10)]},
                 {"name": "b", "role_mask": 3, "more_filters": [6], "scorers": [(P, 20), (Q, 7)]},
                 {"name": "c", "role_mask": 4, "scorers": [(K, 3), (P, 50)]}], None),
    "kv-queue-only": ([{"name": "a", "scorers": [(K, 10), (Q, 10)]}], None),
    "lora": ([{"name": "a", "scorers": [(P, 60), (L, 30), (Q, 10)]}, {"name": "b", "scorers": [(L, 5), (P, 1)]}], None),
    "pd": ([{"name": "prefill", "role_mask": 2, "scorers": [(P, 50), (K, 25), (Q, 25)]},
            {"name": "decode", "role_mask": 4, "scorers": [(P, 50), (K, 25), (Q, 25)]}], {"decode": 1, "prefill": 0}),
}


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


def check_picks_against_matrix(picks, counts, begin=0):
    """every entry with an endpoint reports the matrix's count at that endpoint ([R, P] or [R, P, k] picks)"""
    p = picks.reshape(picks.shape[0], -1)
    real = p["endpoint"] != NO
    r, _ = np.nonzero(real)
    assert real.any()
    assert np.array_equal(p["match_blocks"][real], counts[r, p["endpoint"][real].astype(np.int64) - begin])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("profiles", sorted(PROFILE_SETS))
@pytest.mark.parametrize("shard", [None, (5, 30)])
def test_picks_agree_with_the_matrix(mode, profiles, shard):
    E, R, M, B = 70, 96, 24, 64
    rng = np.random.default_rng(3)
    tok, offs = MC.prompts(R, B, M, rng)
    prof, pd = PROFILE_SETS[profiles]
    if pd is not None:
        pd = dict(pd, threshold=float(B * M // 3))
    cfg = _cfg(E, B, M, R, mode, profiles=prof, pd=pd)
    o = ExtOracle(cfg, shard=shard)
    o.update_endpoints(SV.tie_states(E, rng))
    ad = None
    if profiles == "lora":
        o.update_endpoints_lora(_lora(E, rng))
        ad = (rng.integers(0, 8, R) + 1000).astype(np.uint64)
    chains, nb = o.hash_batch(tok, offs, 9)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=4):
        o.index_apply(ops)
    before = o.pick_batch_ranked(tok, offs, 9, 16, adapters=ad)
    counts, n = o.match_counts(tok, offs, 9)
    begin = 0 if shard is None else shard[0]
    check_picks_against_matrix(o.pick_batch(tok, offs, 9, adapters=ad), counts, begin)
    ranked = o.pick_batch_ranked(tok, offs, 9, 16, adapters=ad)
    assert H.picks_equal(ranked, before)  # the counts leave the configuration and endpoint states as they were
    check_picks_against_matrix(ranked, counts, begin)
    assert (ranked["n_blocks"] == n[:, None, None]).all()
    o.close()


@pytest.mark.parametrize("mode", MODES)
def test_shard_matrices_join_into_the_pool(mode):
    """LPM (holes included), and UPSTREAM on a prefix-closed index: the columns of a partition's shard views, side by
    side, are the pool's matrix"""
    E, R, M, B = 70, 64, 24, 64
    rng = np.random.default_rng(21)
    tok, offs = MC.prompts(R, B, M, rng)
    cfg = _cfg(E, B, M, R, mode)
    full = ExtOracle(cfg)
    chains, nb = full.hash_batch(tok, offs, 5)
    ops = MC.family_ops(chains, nb, E, rng, holes=0.1 if mode == abi.FI_MATCH_LPM else 0.0)
    if mode == abi.FI_MATCH_UPSTREAM:
        ops = ops[:1]  # no CLEAR: every endpoint's keys of a chain are a prefix of it
    for o in ops:
        full.index_apply(o)
    want, _ = full.match_counts(tok, offs, 5)
    for parts in SV.splits(E):
        views = [ExtOracle(cfg, shard=bc) for bc in parts]
        for v in views:
            for o in ops:
                v.index_apply(o)
        got = np.concatenate([v.match_counts(tok, offs, 5)[0] for v in views], axis=1)
        assert np.array_equal(got, want), parts
        for v in views:
            v.close()
    full.close()


def test_upstream_hole_does_not_join():
    """e0 holds blocks 0 and 2, e1 (another shard) blocks 0 and 1: the pool's UPSTREAM walk counts 2 for e0, e0's
    shard walk stops at block 1 and counts 1; in LPM mode both count 1"""
    wl = H.small_workload(E=2, R=1, T=64, max_blocks=4)
    tok, offs = wl.prompts()
    for mode, e0 in ((abi.FI_MATCH_UPSTREAM, (2, 1)), (abi.FI_MATCH_LPM, (1, 1))):
        cfg = H.config_for(wl, match_mode=mode)
        full = ExtOracle(cfg)
        chains, nb = full.hash_batch(tok, offs, wl.h0)
        ops = H.ops_array([(int(chains[0, 0]), 0, 1), (int(chains[0, 2]), 0, 1),
                           (int(chains[0, 0]), 1, 1), (int(chains[0, 1]), 1, 1)])
        views = [ExtOracle(cfg, shard=(0, 1)), ExtOracle(cfg, shard=(1, 1))]
        for x in [full] + views:
            x.index_apply(ops)
        whole = full.match_counts(tok, offs, wl.h0)[0]
        joined = np.concatenate([v.match_counts(tok, offs, wl.h0)[0] for v in views], axis=1)
        assert whole.tolist() == [[e0[0], 2]]
        assert joined.tolist() == [[e0[1], 2]]


def test_zero_requests_and_the_matrix_layout():
    wl = H.small_workload(E=3, R=4, T=128, max_blocks=8)
    cfg = H.config_for(wl)
    o = ExtOracle(cfg)
    tok, offs = wl.prompts()
    counts, nb = o.match_counts(tok, offs[:1], wl.h0)
    assert counts.shape == (0, 3) and nb.shape == (0,)
    chains, nb = o.hash_batch(tok, offs, wl.h0)
    o.index_apply(H.ops_array([(int(h), 2, 1) for h in chains[1, :5]]))
    counts, _ = o.match_counts(tok, offs, wl.h0)
    assert counts.dtype == np.uint16 and counts[1].tolist() == [0, 0, 5]


# ---- the bit-plane unpack of the COUNTS epilogue --------------------------------------------------------------------
@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    lib.fihc_bc_unpack.restype = C.c_int
    lib.fihc_bc_unpack.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return lib


def test_bc_unpack_equals_bc_get(hc):
    rng = np.random.default_rng(1)
    for trial in range(400):
        planes = rng.integers(0, 2**32, size=10, dtype=np.uint64).astype(np.uint32)
        if trial % 4 == 0:
            planes[rng.random(10) < 0.5] = 0
        if trial % 4 == 1:
            planes[:] = 0xFFFFFFFF  # every count 1023
        planes = np.ascontiguousarray(planes)
        for nbits in (1, 2, 4, 8, 16, 32):
            for bit0 in range(0, 33 - nbits, nbits):
                a = np.zeros(nbits, dtype=np.uint16)
                b = np.zeros(nbits, dtype=np.uint16)
                assert hc.fihc_bc_unpack(planes.ctypes.data, bit0, nbits, a.ctypes.data, b.ctypes.data) == 0
                assert np.array_equal(a, b), (trial, nbits, bit0)
                want = [sum(((int(planes[pl]) >> (bit0 + j)) & 1) << pl for pl in range(10)) for j in range(nbits)]
                assert a.tolist() == want
    z = np.zeros(10, dtype=np.uint32)
    a = np.zeros(32, dtype=np.uint16)
    assert hc.fihc_bc_unpack(z.ctypes.data, 16, 32, a.ctypes.data, a.ctypes.data) == -1
    assert hc.fihc_bc_unpack(z.ctypes.data, 0, 3, a.ctypes.data, a.ctypes.data) == -1
