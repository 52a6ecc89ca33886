"""CPU: removal of whole endpoints (upstream indexer.RemovePod) in the tests' reference and in the host LRU.

tests/remove_ref.py (the oracle's calls replayed without the removed endpoints) is what the GPU tests of
fi_epp_index_remove_endpoints compare against, so its removal is checked here against a plain-Python model of the
same calls: membership, LRU content and the count of removed pairs.
"""
import ctypes as C
import os
import random
from collections import OrderedDict

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.remove_ref import RemovalOracle


class _Model:
    """index = {(endpoint, hash)}, one ordered-dict LRU per endpoint"""

    def __init__(self, E, cap):
        self.cap = cap
        self.pairs = set()
        self.lru = [OrderedDict() for _ in range(E)]

    def apply(self, ops):
        for h, e, o in ops:
            (self.pairs.add if o == abi.FI_OP_SET else self.pairs.discard)((int(e), int(h)))

    def add_chain(self, e, keys):
        d = self.lru[e]
        for k in (int(x) for x in keys):
            if k in d:
                d.move_to_end(k)
                continue
            d[k] = True
            self.pairs.add((e, k))
            if len(d) > self.cap:
                old, _ = d.popitem(last=False)
                self.pairs.discard((e, old))

    def remove(self, eps):
        drop = set(int(e) for e in eps)
        gone = {p for p in self.pairs if p[0] in drop}
        self.pairs -= gone
        for e in drop:
            self.lru[e].clear()
        return len(gone)


def _check(cpu, model, E, universe):
    for h in universe:
        for e in range(E):
            assert cpu.index_contains(e, int(h)) == ((e, int(h)) in model.pairs), (e, h)


def test_reference_remove_endpoints_matches_model():
    E, cap = 12, 10
    cfg = H.make_config(num_endpoints=E, max_batch=8, lru_capacity=cap)
    cpu = RemovalOracle(cfg)
    model = _Model(E, cap)
    rng = random.Random(7)
    universe = [0, 0xFFFFFFFFFFFFFFFF] + [rng.randrange(1, 2**63) for _ in range(60)]
    for step in range(30):
        # direct SET / CLEAR ops (the hashes 0 and ~0 included) and LRU Adds, then a removal
        ops = [(rng.choice(universe), rng.randrange(E), rng.choice([abi.FI_OP_SET, abi.FI_OP_SET, abi.FI_OP_CLEAR]))
               for _ in range(40)]
        cpu.index_apply(H.ops_array(ops))
        model.apply(ops)
        for _ in range(4):
            e = rng.randrange(E)
            keys = np.array([rng.choice(universe) for _ in range(rng.randrange(0, 14))], dtype=np.uint64)
            cpu.index_add_chain(e, keys)
            model.add_chain(e, keys)
        kind = step % 5
        if kind == 0:
            eps = [rng.randrange(E)]
        elif kind == 1:
            eps = [rng.randrange(E) for _ in range(3)] * 2  # duplicates
        elif kind == 2:
            eps = list(range(E))
        elif kind == 3:
            eps = []
        else:
            eps = rng.sample(range(E), 5)
        assert cpu.remove_endpoints(eps) == model.remove(eps)
        _check(cpu, model, E, universe)
        # a removed endpoint's LRU is empty: re-adding a key it held is an insertion (SET) again, and eviction
        # order starts fresh
        for e in eps[:1]:
            keys = np.array(universe[2 : 2 + cap + 3], dtype=np.uint64)
            cpu.index_add_chain(e, keys)
            model.add_chain(e, keys)
            _check(cpu, model, E, universe)
    cpu.close()


def test_reference_remove_rejects_out_of_range_and_changes_nothing():
    cfg = H.make_config(num_endpoints=4, max_batch=8, lru_capacity=8)
    cpu = RemovalOracle(cfg)
    cpu.index_apply(H.ops_array([(5, 1, abi.FI_OP_SET)]))
    with pytest.raises(ValueError):
        cpu.remove_endpoints([1, 4])
    assert cpu.index_contains(1, 5)
    assert cpu.remove_endpoints([1]) == 1 and not cpu.index_contains(1, 5)
    cpu.close()


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    lib.fihc_lru_new.restype = C.c_void_p
    lib.fihc_lru_new.argtypes = [C.c_uint32]
    lib.fihc_lru_free.argtypes = [C.c_void_p]
    lib.fihc_lru_clear.argtypes = [C.c_void_p]
    lib.fihc_lru_size.restype = C.c_uint32
    lib.fihc_lru_size.argtypes = [C.c_void_p]
    lib.fihc_lru_contains.argtypes = [C.c_void_p, C.c_uint64]
    lib.fihc_lru_touch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _touch(hc, l, keys):
    ka = np.ascontiguousarray(keys, dtype=np.uint64)
    ins = np.zeros(len(ka), np.uint8)
    did = np.zeros(len(ka), np.uint8)
    ev = np.zeros(len(ka), np.uint64)
    hc.fihc_lru_touch(l, ka.ctypes.data, len(ka), ins.ctypes.data, did.ctypes.data, ev.ctypes.data)
    return ins, did, ev


def test_host_lru_clear_starts_fresh(hc):
    """LruSet::clear (the host LRU's part of fi_epp_index_remove_endpoints): empty, every key inserts anew, and
    eviction order is that of the touches after the clear."""
    cap = 8
    l = hc.fihc_lru_new(cap)
    hc.fihc_lru_clear(l)  # never used: nothing to do
    _touch(hc, l, np.arange(1, 21, dtype=np.uint64))
    assert hc.fihc_lru_size(l) == cap
    hc.fihc_lru_clear(l)
    assert hc.fihc_lru_size(l) == 0
    assert not any(hc.fihc_lru_contains(l, k) for k in range(1, 21))
    ins, did, _ = _touch(hc, l, np.arange(13, 21, dtype=np.uint64))  # the last 8 keys it held: all new again
    assert ins.all() and not did.any()
    _touch(hc, l, np.array([13], dtype=np.uint64))  # 13 becomes the most recent
    ins, did, ev = _touch(hc, l, np.array([100, 101], dtype=np.uint64))
    assert ins.all() and did.all() and list(ev) == [14, 15]
    hc.fihc_lru_free(l)
