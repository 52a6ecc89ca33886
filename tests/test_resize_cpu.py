"""CPU: fi_epp_resize_pool's reference and its shape rule.

The tests' oracle resizes a pool with ExtOracle.resize (tests/ext_oracle.py).  docs/SPEC.md S.2c defines a resize by a
history: the resized pool behaves like one created at the new size and fed the same calls, with everything ever aimed
at an endpoint a shrink dropped left out.  Here ExtOracle.resize is held to that definition (tests/resize_ref.py replays
the filtered history into a fresh oracle) over random call streams with interleaved grows and shrinks.  The shape rule
(pool_shape.h: row words, default slots and their floor, when a resize rebuilds) is checked through libfi_hostcheck.so.
"""
import ctypes as C
import os

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests import resize_ref as RR
from tests.ext_oracle import ExtOracle


def _compare(ora, ref, cs, E, what):
    tok, offs, h0 = cs.tok, cs.offs, cs.h0
    ad = cs.adapters()
    got, want = ora.pick_batch(tok, offs, h0, adapters=ad), ref.pick_batch(tok, offs, h0, adapters=ad)
    assert H.picks_equal(got, want), what + " (single)\n" + H.describe_diff(got, want)
    got, want = ora.pick_batch_ranked(tok, offs, h0, 4, adapters=ad), ref.pick_batch_ranked(tok, offs, h0, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (ranked)\n" + H.describe_diff(got, want)
    sub = cs.subsets(E)
    assert sub.shape == (cs.R, (E + 31) // 32)
    got, want = ora.pick_batch_subset(tok, offs, h0, sub, 4), ref.pick_batch_subset(tok, offs, h0, sub, 4)
    assert H.picks_equal(got, want), what + " (subset)\n" + H.describe_diff(got, want)
    for e in range(E):
        for h in cs.hashes:
            assert ora.index_contains(e, int(h)) == ref.index_contains(e, int(h)), (what, e, h)
        assert np.array_equal(ora.lru(e), ref.lru(e)), (what, e)


def _capacities(ora, E, C_):
    """every endpoint's LRU capacity, observed: the size its LRU settles at under a chain of fresh keys"""
    fresh = np.arange(1 << 40, (1 << 40) + C_, dtype=np.uint64)
    for e in range(E):
        ora.index_add_chain(e, fresh)
    return [ora.lru_size(e) for e in range(E)]


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_resize_matches_the_filtered_history(mode, seed):
    sizes = [40, 33, 70, 5, 64, 1, 37, 37, 100, 31, 45]  # shrinks, grows (dropped endpoints come back), a no-op
    cfg = RR.config(sizes[0], match_mode=mode)
    cs = RR.CallStream(seed, cfg)
    ora = ExtOracle(cfg, track_removal=True)
    hist = RR.History(cfg)
    E = sizes[0]
    for En in sizes[1:]:
        for entry in cs.calls(E, n=8):
            RR.apply(ora, entry)
            hist.record(entry)
        before = {(e, int(h)) for e in range(En, E) for h in cs.hashes if ora.index_contains(e, int(h))}
        removed = ora.resize(En)
        assert removed == len(before)
        if En < E:
            hist.shrink(En)
        E = En
        ref = hist.replay(E)
        _compare(ora, ref, cs, E, f"after the resize to {E}")
        ref.close()
    caps = _capacities(ora, E, cfg.lru_capacity)
    ref = hist.replay(E)
    assert caps == _capacities(ref, E, cfg.lru_capacity)
    ref.close()
    ora.close()


def test_grown_endpoints_start_fresh():
    """A grown endpoint is not alive, has no adapters, an empty LRU and capacity lru_capacity, even one that held all
    of these before a shrink dropped it."""
    cfg = RR.config(8)
    ora = ExtOracle(cfg, track_removal=True)
    ora.update_endpoints(H.states_array(8))
    ora.index_add_chain(7, np.arange(1, 31, dtype=np.uint64))
    ora.set_lru_capacities([7], [16])
    assert ora.lru_size(7) == 16
    assert ora.resize(4) == 16
    assert ora.resize(8) == 0
    assert ora.lru_size(7) == 0 and not ora.index_contains(7, 30)
    assert _capacities(ora, 8, cfg.lru_capacity)[7] == cfg.lru_capacity
    data, offs = H.pack_prompts([bytes(range(64))])
    assert ora.pick_batch(data, offs, 1)[0, 0]["endpoint"] != 7
    ora.close()


# ---- the shape rule (pool_shape.h) -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    lib.fihc_pool_row_words.restype = C.c_uint32
    lib.fihc_pool_row_words.argtypes = [C.c_uint32]
    lib.fihc_pool_default_slots.restype = C.c_uint64
    lib.fihc_pool_default_slots.argtypes = [C.c_uint32, C.c_uint32]
    lib.fihc_pool_resized_slots.restype = C.c_uint64
    lib.fihc_pool_resized_slots.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint64]
    lib.fihc_pool_needs_rebuild.restype = C.c_int
    lib.fihc_pool_needs_rebuild.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64]
    return lib


def _pow2_ceil(x):
    p = 1
    while p < x:
        p *= 2
    return p


def test_row_words_for_every_pool_size(hc):
    for E in range(1, 4097):
        assert hc.fihc_pool_row_words(E) == _pow2_ceil((E + 31) // 32), E
    for k in range(8):  # the boundaries 32 * 2^k +- 1
        b = 32 << k
        assert hc.fihc_pool_row_words(b) == 1 << k
        assert hc.fihc_pool_row_words(b + 1) == 2 << k
        assert hc.fihc_pool_row_words(b - 1) == 1 << k


def test_default_slots_and_their_floor(hc):
    for E in (1, 2, 3, 31, 100, 1000, 1024, 4096):
        for cap in (0, 1, 300, 31250):
            want = min(max(_pow2_ceil(2 * E * (cap or 1024)), 4096), 1 << 31)
            assert hc.fihc_pool_default_slots(E, cap) == want, (E, cap)
            # no live keys, or as many as the default holds: the default
            assert hc.fihc_pool_resized_slots(0, E, cap, 0) == want
            assert hc.fihc_pool_resized_slots(0, E, cap, want * 6 // 10) == want
            # more: doubled until they are at most 60% of the slots
            for live in (want * 6 // 10 + 1, want, 5 * want):
                got = hc.fihc_pool_resized_slots(0, E, cap, live)
                assert live * 10 <= got * 6 and (got // 2) * 6 < live * 10 and got & (got - 1) == 0, (E, cap, live)


def test_pinned_slots_are_kept(hc):
    for pinned in (64, 4096, 1 << 20):
        for live in (0, pinned // 2):
            assert hc.fihc_pool_resized_slots(pinned, 7, 300, live) == pinned


def test_rebuild_exactly_when_the_shape_changes(hc):
    for W, S, W2, S2 in [(1, 4096, 1, 4096), (2, 4096, 2, 8192), (2, 4096, 4, 4096), (4, 1 << 20, 2, 1 << 19)]:
        assert hc.fihc_pool_needs_rebuild(W, S, W2, S2) == (W != W2 or S != S2)
    # 33 -> 60 endpoints without an LRU: the same row width and default slots, so no rebuild; 60 -> 200: wider rows
    shape = [(hc.fihc_pool_row_words(E), hc.fihc_pool_default_slots(E, 0)) for E in (33, 60, 200)]
    assert shape[0] == shape[1] == (2, 1 << 17)
    assert not hc.fihc_pool_needs_rebuild(*shape[0], *shape[1])
    assert hc.fihc_pool_needs_rebuild(*shape[1], *shape[2])
