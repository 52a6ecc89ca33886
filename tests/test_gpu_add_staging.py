"""GPU (-m gpu): indexer.Add calls in a row, with no pick or sync between them, against the CPU oracle.

On the host LRU (device_lru = 0) the Adds stage their index ops in an open group that the GPU applies as all SETs, then
all CLEARs.  A CLEAR staged by one call and a SET of the same pair staged by the next must not share a group, whichever
entry points staged them.  Membership is read once at the end with index_contains (which flushes the open group) over
every key ever added, at every endpoint.  The device-LRU case runs a batch whose hot endpoint overflows its table in the
optimistic pass, so that its requests are deferred to the conservative pass.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu


class _Pair:
    """a handle and the CPU oracle (tests/ext_oracle.cpp) fed the same Adds; `ever` = every key added so far"""

    def __init__(self, device_lru, E=4, cap=8, max_blocks=4, table_slots=0):
        wl = H.small_workload(E=E, R=8, T=max_blocks * 16, max_blocks=max_blocks, lru_capacity=0)
        self.cfg = H.config_for(wl, lru_capacity=cap, index_slots=1 << 17, max_batch=256)
        self.gpu = EndpointPicker(self.cfg)
        self.gpu.set_option("device_lru", device_lru)
        if table_slots:
            self.gpu.set_option("lru_table_slots", table_slots)
        self.ref = ExtOracle(self.cfg)
        self.E, self.mb, self.ever = E, max_blocks, set()

    def add_chains(self, eps, chains):
        """chains: one list of keys per request (at most max_blocks each)"""
        rows = np.zeros((len(chains), self.mb), np.uint64)
        nb = np.array([len(c) for c in chains], np.uint32)
        for r, c in enumerate(chains):
            rows[r, : len(c)] = c
            self.ever.update(int(k) for k in c)
        eps = np.asarray(eps, np.uint32)
        self.gpu.index_add_chains(eps, rows, nb)
        self.ref.index_add_chains(eps, rows, nb)

    def add_chain(self, e, keys):
        self.ever.update(keys)
        self.gpu.index_add_chain(e, np.asarray(keys, np.uint64))
        self.ref.index_add_chain(e, keys)

    def check(self):
        keys = np.array(sorted(self.ever), dtype=np.uint64)
        q = np.zeros(len(keys) * self.E, dtype=H.OP_DTYPE)
        q["hash"] = np.repeat(keys, self.E)
        q["endpoint"] = np.tile(np.arange(self.E, dtype=np.uint32), len(keys))
        got = self.gpu.index_contains(q)
        want = np.array([self.ref.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], np.uint8)
        bad = [(int(h), int(e)) for h, e, g, w in zip(q["hash"], q["endpoint"], got, want) if g != w]
        assert not bad, f"{len(bad)} of {len(q)} memberships differ, e.g. {bad[:4]}"
        assert self.gpu.index_stats().lru_entries == sum(self.ref.lru_size(e) for e in range(self.E))

    def close(self):
        self.gpu.close()
        self.ref.close()


# keys 1..9 on endpoint 0 (capacity 8): key 1 is evicted and its CLEAR stays staged in the call's tail
FIRST = ([0, 0, 0, 2], [[1, 2, 3, 4], [5, 6, 7, 8], [9], [11, 12]])


def test_add_chains_then_add_chains_re_adding_an_evicted_key():
    p = _Pair(device_lru=0)
    p.add_chains(*FIRST)
    p.add_chains([0, 1], [[1], [13, 14]])
    p.check()
    p.close()


def test_add_chains_then_add_chain():
    p = _Pair(device_lru=0)
    p.add_chains(*FIRST)
    p.add_chain(0, [1, 10])
    p.check()
    p.close()


def test_add_chains_then_index_apply_set():
    p = _Pair(device_lru=0)
    p.add_chains(*FIRST)
    ops = H.ops_array([(1, 0, abi.FI_OP_SET), (12, 2, abi.FI_OP_CLEAR)])
    p.gpu.index_apply(ops)
    p.ref.index_apply(ops)
    p.check()
    p.close()


def test_set_lru_capacities_then_add_chains():
    """the shrink's CLEARs (no count asked: nothing flushed) and a later batched Add that re-adds a key it evicted"""
    p = _Pair(device_lru=0)
    p.add_chains([0, 0], [[1, 2, 3, 4], [5, 6, 7, 8]])
    p.gpu.set_lru_capacities([0], [4])
    assert p.ref.set_lru_capacities([0], [4]) == [(k, 0) for k in (1, 2, 3, 4)]
    p.add_chains([0, 3], [[2], [20, 21]])
    p.check()
    p.close()


# lru_counters() after test_device_lru_deferral's batches, pinned: the Adds keep the same sub-batches, deferrals and
# maintenance runs
DEFERRAL_COUNTERS = {"sets": 3603, "clears": 4598, "doomed": 1600, "maintained": 25, "deferred_requests": 189, "sub_batches": 33}


def test_device_lru_deferral():
    """A hot endpoint receives most of a batch and overflows its (minimum-size) table in the optimistic pass: its
    requests run again in the conservative pass.  Membership, every LRU's recency order and the LRU counters."""
    E, M, cap = 6, 24, 90
    p = _Pair(device_lru=1, E=E, cap=cap, max_blocks=M, table_slots=1)
    rng = np.random.default_rng(7)
    prefixes = rng.integers(1, 1 << 62, size=(30, M), dtype=np.uint64)
    for step in range(4):
        R = 120
        eps = rng.integers(0, E, size=R)
        if step % 2 == 1:
            eps[rng.random(R) < 0.8] = step % E  # the hot endpoint
        chains = []
        for r in range(R):
            cut, n = int(rng.integers(0, M + 1)), int(rng.integers(0, M + 1))
            c = np.concatenate([prefixes[rng.integers(0, len(prefixes))][:cut], rng.integers(1, 1 << 62, size=M, dtype=np.uint64)])
            chains.append([int(k) for k in c[:n]])
        p.add_chains(eps, chains)
    p.check()
    for e in range(E):
        assert np.array_equal(p.gpu.lru_dump(e), p.ref.lru(e)), f"LRU of endpoint {e}"
    assert p.gpu.lru_counters() == DEFERRAL_COUNTERS
    p.close()
