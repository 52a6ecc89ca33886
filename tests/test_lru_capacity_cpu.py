"""CPU: per-endpoint LRU capacities (fi_epp_set_lru_capacities, SPEC S.2b) in the CPU oracle and in the host LRU.

The oracle's extension (tests/ext_oracle.cpp, the CPU oracle with a capacity per endpoint) is what the GPU tests
compare against; here it is checked against the oracle's own Adds (uniform capacities) and against an ordered-dict
model of the same calls (random capacities).  The host LRU's LruSet::shrink and the
batched host walk (lru_batch.h) with mixed limits are driven through libfi_hostcheck.so against the same model.
"""
import ctypes as C
import os
import random

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import helpers as H
from tests.ext_oracle import ExtOracle


def _universe(rng, n):
    return [0, 0xFFFFFFFFFFFFFFFF] + [rng.randrange(1, 2**63) for _ in range(n)]


def test_reference_with_uniform_capacities_is_the_oracle():
    """Never set, set to lru_capacity and set to 0: the reference's index equals the oracle's own Adds."""
    E, cap, mb = 6, 12, 4
    cfg = H.make_config(num_endpoints=E, max_batch=8, max_blocks=mb, lru_capacity=cap)
    rng = random.Random(3)
    universe = _universe(rng, 40)
    for variant in ("never", "lru_capacity", "zero"):
        ref, cpu = ExtOracle(cfg), eo.Oracle(cfg)
        if variant != "never":
            assert ref.set_lru_capacities(list(range(E)), [cap if variant == "lru_capacity" else 0] * E) == []
        for _ in range(40):
            ops = H.ops_array([(rng.choice(universe), rng.randrange(E), rng.choice([abi.FI_OP_SET, abi.FI_OP_CLEAR]))
                               for _ in range(5)])
            ref.index_apply(ops)
            cpu.index_apply(ops)
            R = 4
            eps = np.array([rng.randrange(E) for _ in range(R)], dtype=np.uint32)
            chains = np.array([[rng.choice(universe) for _ in range(mb)] for _ in range(R)], dtype=np.uint64)
            nb = np.array([rng.randrange(0, mb + 1) for _ in range(R)], dtype=np.uint32)
            ref.index_add_chains(eps, chains, nb)
            cpu.index_add_chains(eps, chains, nb)
        for e in range(E):
            for h in universe:
                assert ref.index_contains(e, h) == cpu.index_contains(e, h), (variant, e, h)
        ref.close()
        cpu.close()


def test_reference_with_random_capacities_matches_model():
    """Membership, recency order and the CLEARs of every shrink, after every step, with capacities changed at random
    (shrinks, grows, duplicates in one call) between random Adds and direct ops."""
    E, cap, mb = 8, 24, 4
    cfg = H.make_config(num_endpoints=E, max_batch=8, max_blocks=mb, lru_capacity=cap)
    ref, model = ExtOracle(cfg), H.OrderedLrus(E, cap)
    rng = random.Random(11)
    universe = _universe(rng, 120)
    for step in range(60):
        ops = [(rng.choice(universe), rng.randrange(E), rng.choice([abi.FI_OP_SET, abi.FI_OP_SET, abi.FI_OP_CLEAR]))
               for _ in range(6)]
        ref.index_apply(H.ops_array(ops))
        model.apply(ops)
        for _ in range(5):
            e = rng.randrange(E)
            keys = [rng.choice(universe) for _ in range(rng.randrange(0, 3 * cap))]  # hot: up to 3x its capacity
            ref.index_add_chain(e, np.array(keys, dtype=np.uint64))
            model.add_chain(e, keys)
        eps = [rng.randrange(E) for _ in range(rng.randrange(0, 4))]
        caps = [rng.choice([0, mb, cap, rng.randrange(mb, cap + 1)]) for _ in eps]
        got = ref.set_lru_capacities(eps, caps)
        last = {}
        for e, c in zip(eps, caps):
            last[e] = c
        want = []
        for e in dict.fromkeys(eps):
            want += [(h, e) for h in model.resize(e, last[e])]
        assert got == want, step
        for e in range(E):
            assert list(ref.lru(e)) == list(model.lru[e]), (step, e)
            for h in universe[:: 3]:
                assert ref.index_contains(e, h) == ((e, h) in model.pairs), (step, e, h)
    with pytest.raises(ValueError):
        ref.set_lru_capacities([1], [cap + 1])
    with pytest.raises(ValueError):
        ref.set_lru_capacities([1], [mb - 1])
    ref.close()


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
    lib.fihc_lru_new.restype = V
    lib.fihc_lru_new.argtypes = [U32]
    lib.fihc_lru_free.argtypes = [V]
    lib.fihc_lru_size.restype = U32
    lib.fihc_lru_size.argtypes = [V]
    lib.fihc_lru_touch.argtypes = [V, V, U32, V, V, V]
    lib.fihc_lru_shrink.restype = U32
    lib.fihc_lru_shrink.argtypes = [V, U32, V, U32]
    lib.fihc_lru_limit.restype = U32
    lib.fihc_lru_limit.argtypes = [V]
    lib.fihc_lru_dump.restype = U32
    lib.fihc_lru_dump.argtypes = [V, V, U32]
    lib.fihc_lrupool_new.restype = V
    lib.fihc_lrupool_new.argtypes = [U32, U32, U32]
    lib.fihc_lrupool_free.argtypes = [V]
    lib.fihc_lrupool_shrink.restype = U32
    lib.fihc_lrupool_shrink.argtypes = [V, U32, U32, V, U32]
    lib.fihc_lrupool_dump.restype = U32
    lib.fihc_lrupool_dump.argtypes = [V, U32, V, U32]
    lib.fihc_lrupool_walk.restype = U64
    lib.fihc_lrupool_walk.argtypes = [V, V, V, U32, V, U32, V, U64]
    return lib


def _touch(hc, l, keys):
    ka = np.ascontiguousarray(keys, dtype=np.uint64)
    ins = np.zeros(len(ka), np.uint8)
    did = np.zeros(len(ka), np.uint8)
    ev = np.zeros(len(ka), np.uint64)
    hc.fihc_lru_touch(l, ka.ctypes.data, len(ka), ins.ctypes.data, did.ctypes.data, ev.ctypes.data)
    return ins, did, ev


def _keys(fn, *args, cap):
    """the keys fn writes to an array of cap + 1 (an LRU dump or a shrink's evictions)"""
    out = np.zeros(cap + 1, dtype=np.uint64)
    n = fn(*args, out.ctypes.data, cap + 1)
    return [int(x) for x in out[:n]]


def test_host_lru_shrink_and_grow(hc):
    """LruSet::shrink evicts the oldest keys down to the limit (reported oldest first), raising the limit evicts
    nothing, and touches afterwards (reusing the nodes the shrink gave back) follow the model at every limit."""
    cap = 64
    l = hc.fihc_lru_new(cap)
    model = H.OrderedLrus(1, cap)
    rng = random.Random(5)
    assert _keys(hc.fihc_lru_shrink, l, 10, cap=cap) == [] and hc.fihc_lru_limit(l) == 10  # never used
    model.resize(0, 10)
    for step in range(200):
        keys = [rng.randrange(1, 200) for _ in range(rng.randrange(0, 90))]
        ins, did, ev = _touch(hc, l, keys)
        for k, i, d, x in zip(keys, ins, did, ev):
            before = set(model.lru[0])
            model.add_chain(0, [k])
            assert bool(i) == (k not in before)
            if d:
                assert int(x) in before and int(x) not in model.lru[0]
        limit = rng.choice([1, 10, 32, 63, cap, rng.randrange(1, cap + 1)])
        assert _keys(hc.fihc_lru_shrink, l, limit, cap=cap) == model.resize(0, limit), step
        assert hc.fihc_lru_limit(l) == limit
        assert _keys(hc.fihc_lru_dump, l, cap=cap) == list(model.lru[0]), step
        assert hc.fihc_lru_size(l) == len(model.lru[0])
    hc.fihc_lru_free(l)


@pytest.mark.parametrize("workers", [1, 4])
def test_host_batch_walk_with_mixed_limits(hc, workers):
    """The batched host Add (lru_batch.h) with a different limit per endpoint, hot endpoints receiving several times
    their limit in one batch, and limits changed between batches: the ops applied in the engine's order give the
    model's membership, and every LRU's recency order is the model's."""
    E, cap, mb, R = 9, 48, 8, 40
    p = hc.fihc_lrupool_new(E, cap, workers)
    model = H.OrderedLrus(E, cap)
    rng = np.random.default_rng(workers)
    pairs = set()
    for e in range(E):
        c = int(rng.integers(mb, cap + 1))
        assert _keys(hc.fihc_lrupool_shrink, p, e, c, cap=cap) == model.resize(e, c) == []
    for batch in range(30):
        hot = int(rng.integers(0, E))
        eps = np.where(rng.random(R) < 0.5, hot, rng.integers(0, E, size=R)).astype(np.uint32)
        eps[rng.random(R) < 0.05] = abi.FI_NO_ENDPOINT
        chains = rng.integers(1, 400, size=(R, mb), dtype=np.uint64)
        nb = rng.integers(0, mb + 1, size=R).astype(np.uint32)
        ops = np.zeros(4 * R * mb, dtype=H.OP_DTYPE)
        n = hc.fihc_lrupool_walk(p, eps.ctypes.data, chains.ctypes.data, mb, nb.ctypes.data, R, ops.ctypes.data, len(ops))
        assert n <= len(ops)
        for h, e, o in ops[:n]:
            (pairs.add if o == abi.FI_OP_SET else pairs.discard)((int(e), int(h)))
        for r in range(R):
            if eps[r] != abi.FI_NO_ENDPOINT:
                model.add_chain(int(eps[r]), chains[r, : nb[r]])
        assert pairs == model.pairs, batch
        for e in range(E):
            assert _keys(hc.fihc_lrupool_dump, p, e, cap=cap) == list(model.lru[e]), (batch, e)
        for e in rng.choice(E, size=2, replace=False):
            c = int(rng.choice([mb, cap, int(rng.integers(mb, cap + 1))]))
            gone = _keys(hc.fihc_lrupool_shrink, p, int(e), c, cap=cap)
            assert gone == model.resize(int(e), c)
            pairs -= {(int(e), h) for h in gone}
    hc.fihc_lrupool_free(p)
