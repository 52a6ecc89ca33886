"""The key constructors and table models of tests/collide.py, on the CPU: every constructor hits the home it was asked
for under the kernels' formulas, the LRU home's inverse round-trips, keys are distinct and never 0 or ~0, and the models
reproduce hand-worked layouts."""
import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import collide as X
from tests.helpers import ops_array

SET, CLEAR = abi.FI_OP_SET, abi.FI_OP_CLEAR
M64 = X.MASK64


@pytest.mark.parametrize("slots", [64, 4096, 1 << 20])
def test_index_keys_hit_their_bucket(slots):
    rng = np.random.default_rng(slots)
    nb = slots // 4
    for b in (0, 1, nb - 2, nb - 1, int(rng.integers(0, nb))):
        ks = X.index_keys(b, 300, slots, rng)
        assert len(set(ks)) == 300
        assert all(k & (nb - 1) == b for k in ks)
        assert all(k not in (0, M64) and 0 < k <= M64 for k in ks)
    h = int(rng.integers(1, 1 << 63))
    f = X.index_fillers_for(h, 40, slots, rng)
    assert h not in f and len(set(f)) == 40 and all(X.index_home(k, slots) == X.index_home(h, slots) for k in f)


def test_index_keys_exclude_the_markers():
    """bucket 0 with every free bit 0 would be the hash 0, the last bucket with every free bit 1 the hash ~0: a
    Generator that only draws those must never get them through"""

    class Stuck:
        def __init__(self, v):
            self.v, self.calls = v, 0

        def integers(self, lo, hi):
            self.calls += 1
            if self.calls <= 8:  # four keys' worth of the marker, then ordinary draws
                return self.v if hi > 2 else self.v & 1
            return (self.calls * 0x9E3779B97F4A7C15 & ((1 << 63) - 1)) if hi > 2 else self.calls & 1

    assert X.index_keys(0, 3, 64, Stuck(0)).count(0) == 0
    assert M64 not in X.index_keys(15, 3, 64, Stuck((1 << 63) - 1))
    assert 0 not in X.dlru_keys(0, 3, 256, Stuck(0))


@pytest.mark.parametrize("TS", [256, 512, 1 << 16, 1 << 24])
def test_dlru_keys_hit_their_slot(TS):
    rng = np.random.default_rng(TS)
    for s in (0, 1, TS - 2, TS - 1, int(rng.integers(0, TS))):
        ks = X.dlru_keys(s, 200, TS, rng)
        assert len(set(ks)) == 200
        assert all(k not in (0, M64) for k in ks)
        # the kernel's formula, in uint64 arithmetic: ((key * PHI) >> 40) & (TS - 1)
        a = np.array(ks, dtype=np.uint64)
        with np.errstate(over="ignore"):
            home = ((a * np.uint64(X.PHI)) >> np.uint64(40)) & np.uint64(TS - 1)
        assert (home == s).all()
        assert all(X.dlru_home(k, TS) == s for k in ks)


def test_dlru_inverse_round_trips():
    rng = np.random.default_rng(7)
    assert X.PHI * X.PHI_INV & M64 == 1
    for _ in range(2000):
        x = int(rng.integers(0, 1 << 63)) << 1 | int(rng.integers(0, 2))
        assert X.dlru_key_of(x) * X.PHI & M64 == x
        assert X.dlru_key_of(x * X.PHI & M64) == x


def test_table_sizes_follow_alloc_dev_lru():
    assert X.dlru_table_slots(64, 1) == 256      # the minimum: L = pow2_ceil(4 C)
    assert X.dlru_table_slots(64, 300) == 512
    assert X.dlru_table_slots(10, 1) == 64       # L is at least 64
    assert X.dlru_table_slots(100, 4096) == 4096
    assert X.dlru_log_records(64, 256) == 256 and X.dlru_log_records(64, 4096) == 1024


def test_index_model_wrapped_run():
    """16 buckets of 4: six keys homed at the last bucket fill it and wrap into bucket 0; a key of bucket 0 then
    lands behind them, and a lookup of a missing key homed at 15 crosses the end of the table"""
    rng = np.random.default_rng(1)
    m = X.IndexModel(64)
    run = X.index_keys(15, 6, 64, rng)
    m.apply(ops_array([(k, 0, SET) for k in run]))
    assert sorted(m.keys.index(k) for k in run) == [0, 1, 60, 61, 62, 63]
    late = X.index_keys(0, 1, 64, rng)[0]
    m.apply(ops_array([(late, 1, SET)]))
    p = m.probe(late)
    assert p.found == 2 and p.distance == 0 and not p.wrapped
    p = m.probe(run[5]) if m.keys.index(run[5]) < 4 else m.probe(run[0] if m.keys.index(run[0]) < 4 else run[1])
    assert p.wrapped and p.distance == 1 and p.steps == [15, 0]
    miss = m.probe(X.index_keys(15, 1, 64, rng, avoid=run)[0])
    assert miss.found is None and miss.steps == [15, 0] and miss.wrapped
    assert m.run_at(15) == [15, 0] and m.used == 7 and m.tombstones == 0


def test_index_model_tombstone_in_a_run_and_reinsert():
    """a run of 12 keys from bucket 3 (buckets 3, 4, 5); CLEAR one key of bucket 4 (its slot becomes a tombstone);
    a key added in a later call lands past the run and its lookup passes the tombstone; SET of the retired key again
    claims a new slot past the run instead of the tombstone"""
    rng = np.random.default_rng(2)
    m = X.IndexModel(64)
    first = X.index_keys(3, 12, 64, rng)
    m.apply(ops_array([(k, 0, SET) for k in first]))
    assert sorted(m.keys.index(k) for k in first) == list(range(12, 24))
    gone = next(k for k in first if m.keys.index(k) == 17)
    m.apply(ops_array([(gone, 0, CLEAR)]))
    assert m.keys[17] == X.TOMB and m.tombstones == 1 and not m.contains(0, gone)
    late = X.index_keys(3, 1, 64, rng, avoid=first)[0]
    m.apply(ops_array([(late, 0, SET)]))
    p = m.probe(late)
    assert p.found == 24 and p.steps == [3, 4, 5, 6] and p.tombs == 1
    m.apply(ops_array([(gone, 2, SET)]))
    assert m.keys.index(gone) == 25 and m.keys[17] == X.TOMB and m.used == 14 and m.contains(2, gone)
    assert m.live_regular() == 13 == m.used - m.tombstones


def test_index_model_groups_like_the_engine():
    """within one call SETs apply before CLEARs; a SET of a pair the open group CLEARs starts a new group"""
    rng = np.random.default_rng(3)
    m = X.IndexModel(64)
    a, b = X.index_keys(5, 2, 64, rng)
    m.apply(ops_array([(a, 0, SET), (a, 0, CLEAR), (b, 1, CLEAR), (b, 1, SET)]))
    # group 1: SET a, CLEAR a, CLEAR b (a retired); group 2: SET b
    assert not m.contains(0, a) and m.contains(1, b) and m.tombstones == 1 and m.used == 2
    m.apply(ops_array([(b, 3, SET), (b, 1, CLEAR)]))
    assert m.contains(3, b) and not m.contains(1, b)


def test_lru_model_wrapped_run_and_tombstones():
    """TS = 256: five keys homed at 254 and three at 255 fill 254, 255, 0..5; the two oldest leave as tombstones; a
    key homed at 255 inserted later sits at 6 and its lookup wraps past both tombstones"""
    rng = np.random.default_rng(4)
    TS = 256
    m = X.LruModel(TS, 64)
    a = X.dlru_keys(254, 5, TS, rng)
    b = X.dlru_keys(255, 3, TS, rng)
    m.insert(a + b + [0, M64])
    assert sorted(m.probe(k).found for k in a + b) == [0, 1, 2, 3, 4, 5, 254, 255] and m.used == 8
    at = {m.probe(k).found: k for k in a + b}
    m.retire([at[255], at[0]])
    assert m.tombstones() == 2 and m.used == 8
    late = X.dlru_keys(255, 1, TS, rng, avoid=a + b)[0]
    m.insert([late])
    p = m.probe(late)
    assert p.found == 6 and p.tombs == 2 and p.wrapped and p.distance == 7
    # re-inserting a retired key takes a new slot past the run
    m.insert([at[0]])
    assert m.probe(at[0]).found == 7 and m.used == 10


def test_lru_model_maintain_decision():
    """lru_maintain_kernel: compaction when the log cannot take the sub-batch, rebuild when used + min(touches, C) is
    above 60 % of TS; a rebuild keeps exactly the live keys"""
    TS, C = 256, 64
    rng = np.random.default_rng(5)
    m = X.LruModel(TS, C)
    ks = X.dlru_keys(10, 100, TS, rng)
    m.insert(ks)
    m.appended(100)
    assert m.maintain(53, ks) == (False, False)          # (100 + 53) * 10 = 1530 <= 1536
    assert m.maintain(54, ks) == (True, True)            # 1540 > 1536
    assert m.used == 100 and m.tombstones() == 0 and m.head == 100
    m.retire(ks[:60])
    m.appended(150)                                       # head 250
    assert m.maintain(7, ks[60:]) == (True, False)       # log: 250 + 7 > 256; table: (100 + 7) * 10 <= 1536
    assert m.head == 40 and m.tombstones() == 60
