"""GPU (-m gpu): handles over part of the pool (endpoint_begin / endpoint_count, docs/SPEC.md S.2e) on one GPU,
bit-exact against the oracle's shard view (tests/ext_oracle.py, ExtOracle(cfg, shard=(b, c))), and several of them
merged on the host against the unsharded oracle.

Such a handle runs the kernels of the sharded pool with ep_begin != 0: every endpoint offset by ep_begin, rows sized
by the shard, the queue scorer's min / max over the whole pool, zero-match ties found in local bit words
(tie_local_origin / tie_first_local), device-LRU CLEARs written as ep_begin + e.  The cases reach each of those: every
match row width of 1 .. 128 words, shards that start at 0, 1, 31, 32, 33 and end at the pool's end, shard sizes that
leave padded bits in the last word, tie rotations that start before, at, inside, at the end of and after the shard,
queue extremes inside and outside it, and updates addressed across the whole pool.
"""
import functools

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import craft
from tests import helpers as H
from tests import shard_view as SV
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
UP, LPM = abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM
NO = abi.FI_NO_ENDPOINT
PROFILES = [{"name": "a", "scorers": [(P, 100), (K, 10), (Q, 10)]},
            {"name": "b", "role_mask": 3, "more_filters": [6], "scorers": [(P, 20), (Q, 7)]},
            {"name": "c", "role_mask": 4, "scorers": [(K, 3), (P, 50)]}]


def row_words(c):
    """match_pick's row width over c local endpoints (pool_shape.h)"""
    w = 1
    while w < (c + 31) // 32:
        w *= 2
    return w


# (E, b, c): every row width 1 .. 128, b in {0, 1, 31, 32, 33, E - c}, c in {1, 31, 32, 33, 100, 1025, 3000} and
# widths 8, 16, 32 with c not a multiple of 32
GEOMETRY = [(40, 0, 1), (64, 1, 31), (96, 32, 32), (37, 36, 1), (100, 33, 33), (300, 31, 100), (300, 100, 200),
            (700, 1, 300), (1000, 300, 700), (2100, 33, 1025), (4096, 1096, 3000), (3100, 0, 3000)]
assert sorted({row_words(c) for _, _, c in GEOMETRY}) == [1, 2, 4, 8, 16, 32, 64, 128]


def _eq(got, want, what):
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)


def _inside(picks, b, c):
    e = picks["endpoint"][picks["endpoint"] != NO]
    assert ((e >= b) & (e < b + c)).all(), "a pick outside the shard"


@functools.lru_cache(maxsize=None)
def _workload(E, holes):
    wl = H.small_workload(E=E, R=128, T=512, holes=holes, lru_capacity=64, groups_per_endpoint=2)
    return wl, tuple(wl.index_ops()), wl.prompts()


def _cold(offs, n=16, nbytes=20):
    offs = offs.copy()
    offs[1:n + 1] = offs[0] + np.arange(1, n + 1, dtype=np.uint64) * nbytes
    return offs


def _pair(cfg, b, c, st, ops=(), lora=None, track=False):
    """the handle over [b, b + c) and its shard view, fed the same states and whole-pool ops"""
    cfg = abi.fi_epp_config.from_buffer_copy(cfg)
    cfg.endpoint_begin, cfg.endpoint_count = b, c
    g, o = EndpointPicker(cfg), ExtOracle(cfg, shard=(b, c), track_removal=track)
    for x in (g, o):
        x.update_endpoints(st)
        if lora is not None:
            x.update_endpoints_lora(lora)
        for op in ops:
            x.index_apply(op)
    return g, o


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


@pytest.mark.parametrize("mode,holes", [(UP, False), (UP, True), (LPM, True)], ids=["upstream", "upstream-holes", "lpm-holes"])
@pytest.mark.parametrize("geom", GEOMETRY, ids=[f"E{E}-b{b}-c{c}" for E, b, c in GEOMETRY])
def test_shard_geometry(geom, mode, holes):
    """single and ranked picks (k = 1, 5, 16) of a handle over [b, b + c), with label filters, dead endpoints, the
    queue scorer and many zero-match ties"""
    E, b, c = geom
    wl, ops, (tok, offs) = _workload(E, holes)
    rng = np.random.default_rng(E + b + mode)
    st = SV.tie_states(E, rng)
    st["flags"][b], st["role_mask"][b] = abi.FI_ENDPOINT_ALIVE, 7  # a shard of one endpoint still picks
    cfg = H.config_for(wl, profiles=PROFILES, match_mode=mode)
    g, o = _pair(cfg, b, c, st, ops)
    offs = _cold(offs)
    got = g.pick_batch(tok, offs, wl.h0)
    _eq(got, o.pick_batch(tok, offs, wl.h0), "single pick")
    _inside(got, b, c)
    assert (got[:, 0]["endpoint"] != NO).any()
    for k in (1, 5, 16):
        got = g.pick_batch_ranked(tok, offs, wl.h0, k)
        _eq(got, o.pick_batch_ranked(tok, offs, wl.h0, k), f"ranked k = {k}")
        _inside(got, b, c)
    g.close()


def _start_requests(E, b, c, rng, block_bytes=64):
    """requests whose tie rotation starts before b, at b, inside, at b + c - 1 and at or after b + c: each once
    without blocks and once with one block the index does not hold -> (tok, offs, h0, starts)"""
    starts = sorted({s % E for s in (b - 1, b, b + 1, b + c // 2, b + c - 2, b + c - 1, b + c, b + c + 7, 0)})
    blobs, h0 = [], []
    for s in starts:
        r = len(blobs)
        blobs.append(b"\x11" * 20)
        h0.append(craft.h0_for_start(s, E, r, low=int(rng.integers(0, 1 << 32))))
        blk = rng.integers(0, 256, block_bytes, dtype=np.uint8).tobytes()
        blobs.append(blk)
        h0.append(craft.h0_for_start(s, E, r + 1, blocks=[blk], low=int(rng.integers(0, 1 << 32))))
    tok, offs = H.pack_prompts(blobs)
    return tok, offs, np.asarray(h0, dtype=np.uint64), [s for s in starts for _ in (0, 1)]


@pytest.mark.parametrize("alive", ["all", "sparse"])
@pytest.mark.parametrize("geom", [(64, 1, 31), (100, 33, 33), (300, 100, 200), (2100, 33, 1025), (4096, 1096, 3000),
                                  (40, 0, 1)], ids=lambda g: f"E{g[0]}-b{g[1]}-c{g[2]}")
def test_tie_rotation_starts(geom, alive):
    """zero-match ties among several shard endpoints: the winner is the first tied endpoint from the request's start,
    wrapping from the shard's tail to its head; the ranked list continues in that order"""
    E, b, c = geom
    rng = np.random.default_rng(c)
    wl = H.small_workload(E=E, R=32, T=64)
    st = H.states_array(E, kv=0.25, queue=3)
    if alive == "sparse":  # a head, a middle, nothing at the tail: a start past the middle wraps to b
        st["flags"] = 0
        st["flags"][[b, b + c // 2]] = abi.FI_ENDPOINT_ALIVE
        st["flags"][rng.integers(0, E, 5)] = abi.FI_ENDPOINT_ALIVE
        st["flags"][b + c // 2 + 1: b + c] = 0
    cfg = H.config_for(wl, profiles=[{"name": "a", "scorers": [(P, 100), (K, 10), (Q, 10)]}], max_batch=64)
    g, o = _pair(cfg, b, c, st)
    tok, offs, h0, starts = _start_requests(E, b, c, rng)
    got = g.pick_batch(tok, offs, h0)
    _eq(got, o.pick_batch(tok, offs, h0), "single pick")
    tied = [e for e in range(b, b + c) if st["flags"][e]]
    for r, s in enumerate(starts):  # the rule itself, stated once more
        assert got[r, 0]["endpoint"] == min(tied, key=lambda e: (e - s) % E)
    for k in (5, 16):
        _eq(g.pick_batch_ranked(tok, offs, h0, k), o.pick_batch_ranked(tok, offs, h0, k), f"ranked k = {k}")
    g.close()


@pytest.mark.parametrize("where", ["outside", "inside", "no-eligible"])
def test_queue_extremes_and_empty_shard(where):
    """the queue scorer normalises over the eligible endpoints of the WHOLE pool; a shard without an eligible
    endpoint answers FI_NO_ENDPOINT"""
    E, b, c = 300, 100, 70
    wl, ops, (tok, offs) = _workload(E, True)
    rng = np.random.default_rng(9)
    st = SV.tie_states(E, rng)
    st["queue_depth"] = rng.integers(10, 20, E)
    lo_e, hi_e = (3, 290) if where == "outside" else (b + 5, b + 60)
    st["queue_depth"][lo_e], st["queue_depth"][hi_e] = 0, 100
    st["flags"][[lo_e, hi_e]] = abi.FI_ENDPOINT_ALIVE
    st["role_mask"][[lo_e, hi_e]] = 7
    if where == "no-eligible":
        st["flags"][b:b + c] = 0
    for mode in (UP, LPM):
        cfg = H.config_for(wl, profiles=PROFILES, match_mode=mode)
        g, o = _pair(cfg, b, c, st, ops)
        got = g.pick_batch(tok, offs, wl.h0)
        _eq(got, o.pick_batch(tok, offs, wl.h0), "single pick")
        for k in (1, 5, 16):
            _eq(g.pick_batch_ranked(tok, offs, wl.h0, k), o.pick_batch_ranked(tok, offs, wl.h0, k), f"ranked k = {k}")
        if where == "no-eligible":
            assert (got["endpoint"] == NO).all() and (got["score"] == 0).all()
        g.close()


def _torch():
    import torch

    return torch


def _dev(a, dtype=np.int64):
    return _torch().from_numpy(np.ascontiguousarray(a).view(dtype)).cuda()


def _picks(t, R, Pn, k):
    return t.cpu().numpy().view(H.PICK_DTYPE).reshape((R, Pn, k) if k else (R, Pn))


@pytest.mark.parametrize("case", ["lora", "pd"])
def test_entry_points(case):
    """host and device single, LoRA and ranked picks, pick_submit, pick_submit_ex (k = 0 and ranked) with
    wait_batch and index_add_submitted, and early-exit hashing on a handle without an LRU"""
    torch = _torch()
    E, b, c = 300, 33, 100
    wl, ops, (tok, offs) = _workload(E, True)
    rng = np.random.default_rng(17)
    st = SV.tie_states(E, rng)
    if case == "lora":
        profiles, pd, lo = [{"name": "a", "scorers": [(P, 60), (L, 30), (Q, 10)]}], None, _lora(E, rng)
    else:
        profiles = [{"name": "prefill", "role_mask": 1, "scorers": [(P, 50), (K, 5)]},
                    {"name": "decode", "role_mask": 2, "scorers": [(P, 50), (Q, 5)]}]
        pd, lo = {"prefill": 0, "decode": 1, "threshold": 0.6 * wl.T * 4}, None
    ad = (rng.integers(0, 8, wl.R) + 1000).astype(np.uint64)
    Pn = len(profiles)
    offs = _cold(offs)
    cfg = H.config_for(wl, profiles=profiles, pd=pd, lru_capacity=64, max_prompt_bytes=wl.R * wl.T * 4)
    g, o = _pair(cfg, b, c, st, ops, lora=lo)
    want1 = o.pick_batch(tok, offs, wl.h0, adapters=ad)
    if case == "pd":
        assert (want1[:, 0]["endpoint"] == NO).any() and (want1[:, 0]["endpoint"] != NO).any()
    _eq(g.pick_batch(tok, offs, wl.h0, adapters=ad), want1, "host single / LoRA")
    _eq(g.pick_batch_ranked(tok, offs, wl.h0, 5, adapters=ad), o.pick_batch_ranked(tok, offs, wl.h0, 5, adapters=ad),
        "host ranked")
    s = torch.cuda.current_stream().cuda_stream
    d_tok, d_off, d_ad = _dev(tok, np.int32), _dev(offs), _dev(ad)
    d_h0 = torch.full((wl.R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    p = (d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr())
    out = torch.zeros(wl.R * Pn * 16 * 16, dtype=torch.uint8, device="cuda")
    rc = abi.load().fi_epp_pick_batch_device_lora(g._h, *p, d_ad.data_ptr(), wl.R, tok.nbytes, out.data_ptr(), None, s)
    g._check(rc, "fi_epp_pick_batch_device_lora")
    _eq(_picks(out[: wl.R * Pn * 16], wl.R, Pn, 0), want1, "device single / LoRA")
    g.pick_batch_device_ranked(*p, wl.R, tok.nbytes, 16, out.data_ptr(), stream=s, d_adapters=d_ad.data_ptr())
    _eq(_picks(out, wl.R, Pn, 16), o.pick_batch_ranked(tok, offs, wl.h0, 16, adapters=ad), "device ranked")
    # the pipelined calls: submit, submit_ex k = 0 and ranked, wait_batch, add_submitted
    out2 = torch.zeros_like(out)
    g.pick_submit(*p, wl.R, tok.nbytes, out2.data_ptr(), s)
    g.pick_wait(s)
    _eq(_picks(out2[: wl.R * Pn * 16], wl.R, Pn, 0), o.pick_batch(tok, offs, wl.h0), "pick_submit")
    chains, nb = o.hash_batch(tok, offs, wl.h0)
    t0 = g.pick_submit_ex(*p, wl.R, tok.nbytes, out.data_ptr(), k=0, d_adapters=d_ad.data_ptr(), stream=s)
    g.pick_wait_batch(t0, s)
    _eq(_picks(out[: wl.R * Pn * 16], wl.R, Pn, 0), want1, "pick_submit_ex k = 0")
    dest = rng.integers(0, E, wl.R).astype(np.uint32)  # decisions across the pool: only the shard's own are added
    g.index_add_submitted(t0, dest, nb)
    o.index_add_chains(dest, chains, nb)
    t1 = g.pick_submit_ex(*p, wl.R, tok.nbytes, out.data_ptr(), k=5, d_adapters=d_ad.data_ptr(), stream=s)
    g.pick_wait_batch(t1, s)
    torch.cuda.synchronize()
    _eq(_picks(out[: wl.R * Pn * 5 * 16], wl.R, Pn, 5), o.pick_batch_ranked(tok, offs, wl.h0, 5, adapters=ad),
        "pick_submit_ex ranked after add_submitted")
    g.index_add_submitted(t1, dest[::-1].copy(), nb)
    o.index_add_chains(dest[::-1].copy(), chains, nb)
    for e in range(b, b + c, 7):
        assert g.lru_dump(e).tolist() == o.lru(e).tolist(), e
    _eq(g.pick_batch(tok, offs, wl.h0, adapters=ad), o.pick_batch(tok, offs, wl.h0, adapters=ad), "after the Adds")
    g.close()
    # early-exit hashing (device buffers, no LRU, no chains_out): a shard that holds none of the keys stops every
    # request early, although the other endpoints' ops named those keys.  (It runs on batches of half-SM hashing tiles,
    # more than 64 requests per SM; a host-buffer pick that large hashes in slices of whole-SM tiles.)
    R = 64 * torch.cuda.get_device_properties(0).multi_processor_count + 200
    wl = H.small_workload(E=E, R=R, T=16 * 256 + 21, max_blocks=256, lru_capacity=0, groups_per_endpoint=2)
    tok, offs = wl.prompts()
    ad = (rng.integers(0, 8, R) + 1000).astype(np.uint64)
    cfg0 = H.config_for(wl, profiles=profiles, pd=pd, lru_capacity=0, max_prompt_bytes=wl.R * wl.T * 4)
    elsewhere = [op[(op["endpoint"] < b) | (op["endpoint"] >= b + c)] for op in wl.index_ops()]
    g, o = _pair(cfg0, b, c, st, elsewhere, lora=lo)
    total = int(o.hash_batch(tok, offs, wl.h0)[1].sum())
    d_tok, d_off, d_ad = _dev(tok, np.int32), _dev(offs), _dev(ad)
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    out = torch.zeros(R * Pn * 16, dtype=torch.uint8, device="cuda")

    def device_pick():
        rc = abi.load().fi_epp_pick_batch_device_lora(g._h, d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(),
                                                       d_ad.data_ptr(), R, tok.nbytes, out.data_ptr(), None, s)
        g._check(rc, "fi_epp_pick_batch_device_lora")
        return _picks(out, R, Pn, 0)

    g.set_profiling(True)
    _eq(device_pick(), o.pick_batch(tok, offs, wl.h0, adapters=ad), "early exit")
    assert g.stats().hashed_blocks < total // 2, (g.stats().hashed_blocks, total)
    for op in wl.index_ops(b, b + c):  # and with the shard's own keys
        g.index_apply(op)
        o.index_apply(op)
    _eq(device_pick(), o.pick_batch(tok, offs, wl.h0, adapters=ad), "early exit, held keys")
    g.close()


def _members(g, o, hashes, eps):
    """index_contains over every (endpoint, hash) pair, on the handle and in the view"""
    q = np.zeros(len(hashes) * len(eps), dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(np.asarray(hashes, dtype=np.uint64), len(eps))
    q["endpoint"] = np.tile(np.asarray(eps, dtype=np.uint32), len(hashes))
    got = g.index_contains(q)
    want = np.array([o.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
    assert np.array_equal(got, want), f"{int((got != want).sum())} memberships differ"
    return got


@pytest.mark.parametrize("lru", ["device", "host"])
def test_updates_across_the_pool(lru):
    """index_apply, Adds, evicting Adds, capacity changes and removals addressed across the whole pool change only the
    shard; picks, memberships and LRUs equal the view after every step"""
    torch = _torch()
    E, b, c = 200, 40, 70
    wl = H.small_workload(E=E, R=96, T=1024, holes=True, lru_capacity=80, groups_per_endpoint=1)
    ops = list(wl.index_ops())
    tok, offs = wl.prompts()
    rng = np.random.default_rng(23)
    st = SV.tie_states(E, rng, roles=False)
    cfg = H.config_for(wl, profiles=PROFILES[:1], lru_capacity=80, max_prompt_bytes=wl.R * wl.T * 4)
    cfg.endpoint_begin, cfg.endpoint_count = b, c
    g = EndpointPicker(cfg)
    if lru == "host":
        g.set_option("device_lru", 0)
    o = ExtOracle(cfg, shard=(b, c), track_removal=True)
    for x in (g, o):
        x.update_endpoints(st)
        for op in ops:
            x.index_apply(op)
    outside = [0, 1, b - 1, b + c, E - 1]
    inside = [b, b + 1, b + 31, b + 32, b + c - 1]
    chains, nb = o.hash_batch(tok, offs, wl.h0)
    probe = np.unique(chains[:, :4])

    def check(what):
        _eq(g.pick_batch(tok, offs, wl.h0), o.pick_batch(tok, offs, wl.h0), what)
        _eq(g.pick_batch_ranked(tok, offs, wl.h0, 5), o.pick_batch_ranked(tok, offs, wl.h0, 5), what + " (ranked)")
        m = _members(g, o, probe, inside + outside)
        assert not m.reshape(len(probe), -1)[:, len(inside):].any(), "an endpoint outside the shard holds a key"
        if lru == "device":
            for e in range(b, b + c):
                assert g.lru_dump(e).tolist() == o.lru(e).tolist(), (what, e)

    check("after index_apply")
    # Adds across the pool; the eviction pressure is two chains per endpoint against a capacity of 80
    dest = rng.integers(0, E, wl.R).astype(np.uint32)
    dest[: len(inside)] = inside
    g.index_add_chains(dest, chains, nb)
    o.index_add_chains(dest, chains, nb)
    check("after index_add_chains")
    g.index_add_chain(outside[0], chains[0, : nb[0]])  # another shard's endpoint: FI_OK, nothing changes
    o.index_add_chain(outside[0], chains[0, : nb[0]])
    g.index_add_chain(inside[0], chains[1, : nb[1]])
    o.index_add_chain(inside[0], chains[1, : nb[1]])
    check("after index_add_chain")
    if lru == "device":
        got, _ = g.pick_batch(tok, offs, wl.h0, want_chains=True)
        d2 = dest[::-1].copy()
        g.index_add_chains_device(d2, 0, 0, nb)  # the chains of the pick just made
        o.index_add_chains(d2, chains, nb)
        torch.cuda.synchronize()
        check("after index_add_chains_device(NULL)")
        for e in outside:
            with pytest.raises(FiEppError) as ei:
                g.lru_dump(e)
            assert ei.value.status == abi.FI_ERR_INVALID
    caps = [wl.max_blocks, 0, wl.max_blocks, 40, wl.max_blocks]
    g.set_lru_capacities(outside[:2] + inside[:3], caps)
    o.set_lru_capacities(outside[:2] + inside[:3], caps)
    check("after set_lru_capacities")
    g.index_add_chains(dest, chains, nb)  # evicting against the new capacities
    o.index_add_chains(dest, chains, nb)
    check("after Adds against the new capacities")
    g.remove_endpoints(outside + inside[1:3])
    o.remove_endpoints(outside + inside[1:3])
    check("after remove_endpoints")
    g.close()


@pytest.mark.parametrize("mode", [UP, LPM])
def test_shard_handles_compose_into_the_pool(mode):
    """2 .. 5 handles over a partition of the pool on one GPU, merged on the host by (score desc, rotation asc):
    the unsharded oracle's single picks and ranked lists"""
    E = 150
    wl, ops, (tok, offs) = _workload(E, mode == LPM)
    rng = np.random.default_rng(31)
    st = SV.tie_states(E, rng)
    st["queue_depth"] = rng.integers(0, 40, E)
    offs = _cold(offs)
    cfg = H.config_for(wl, profiles=PROFILES, match_mode=mode)
    full = ExtOracle(cfg)
    full.update_endpoints(st)
    for op in ops:
        full.index_apply(op)
    chains, nb = full.hash_batch(tok, offs, wl.h0)
    starts = SV.starts(chains, nb, wl.h0, E)
    want1 = full.pick_batch(tok, offs, wl.h0)
    want5 = full.pick_batch_ranked(tok, offs, wl.h0, 5)
    for parts in SV.splits(E):
        hs = [_pair(cfg, b, c, st, ops)[0] for b, c in parts]
        _eq(SV.merge_single([h.pick_batch(tok, offs, wl.h0) for h in hs], starts, E), want1, f"{parts} single")
        _eq(SV.merge_ranked([h.pick_batch_ranked(tok, offs, wl.h0, 5) for h in hs], starts, E), want5, f"{parts} ranked")
        for h in hs:
            h.close()
    full.close()


def test_resize_and_snapshots_are_refused():
    """a handle over part of the pool refuses fi_epp_resize_pool, fi_epp_snapshot_save and fi_epp_snapshot_load with
    FI_ERR_STATE and stays as it was"""
    E, b, c = 100, 33, 33
    wl, ops, (tok, offs) = _workload(E, True)
    st = SV.tie_states(E, np.random.default_rng(2))
    cfg = H.config_for(wl, profiles=PROFILES, lru_capacity=64)
    g, o = _pair(cfg, b, c, st, ops)
    chains, nb = o.hash_batch(tok, offs, wl.h0)
    dest = np.arange(wl.R, dtype=np.uint32) % E
    g.index_add_chains(dest, chains, nb)
    o.index_add_chains(dest, chains, nb)
    full = EndpointPicker(cfg)
    full.index_add_chains(dest, chains, nb)
    blob = full.save_snapshot()
    full.close()
    before = g.pick_batch_ranked(tok, offs, wl.h0, 5)
    for call in (lambda: g.resize_pool(E + 10), lambda: g.resize_pool(b + c), g.save_snapshot,
                 lambda: g.load_snapshot(blob)):
        with pytest.raises(FiEppError) as ei:
            call()
        assert ei.value.status == abi.FI_ERR_STATE
    _eq(g.pick_batch_ranked(tok, offs, wl.h0, 5), before, "after the refusals")
    _eq(before, o.pick_batch_ranked(tok, offs, wl.h0, 5), "the view")
    for e in range(b, b + c):
        assert g.lru_dump(e).tolist() == o.lru(e).tolist()
    g.close()
