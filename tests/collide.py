"""Keys placed on purpose in the two GPU open-addressed tables, and models of those tables' probing rules (test
helper, not collected).

The index (fusioninfer_b200/csrc/index_kernels.cu, index_device.cuh) keeps `slots` keys in buckets of 4 and homes a
key at bucket `h & (slots / 4 - 1)`; the device LRU (lru_kernels.cu) keeps TS 16-byte slots per endpoint and homes a
key at slot `((h * PHI) mod 2^64 >> 40) & (TS - 1)`.  Both probe linearly (over buckets, over slots) and wrap from the
last bucket / slot to the first; a retired key becomes a tombstone (~0) that a lookup has to probe past and an insert
never reuses.  The index home is a bit mask and the LRU home a multiplication by an odd constant, which has an inverse
mod 2^64, so both can be hit exactly: the constructors below return distinct keys with the home asked for, never the
hashes 0 or ~0 (the tables' EMPTY / TOMB markers, which live outside the tables), with their free bits drawn from a
seeded numpy Generator.

IndexModel and LruModel replay the inserts and retirements a test makes and say where every key sits.  Inside one
kernel launch, keys with the same home claim slots in an order set by the race; linear probing fills the same SET of
slots whatever that order is, so the models predict which slots a run occupies, and which slot a key takes when it is
the only new key of its run in its call.  The tests use them only to check that a crafted layout really happened.
"""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi

MASK64 = (1 << 64) - 1
EMPTY = 0
TOMB = MASK64
BUCKET_KEYS = 4
PHI = 0x9E3779B97F4A7C15  # lru_home's multiplier (lru_kernels.cu)
PHI_INV = pow(PHI, -1, 1 << 64)


def _special(h: int) -> bool:
    return h == EMPTY or h == TOMB


def _fresh(make, n, rng, avoid=()):
    """n distinct keys make(rng) that are neither 0, ~0 nor in `avoid`"""
    seen, out = set(int(a) for a in avoid), []
    while len(out) < n:
        k = make(int(rng.integers(0, 1 << 63)) << 1 | int(rng.integers(0, 2))) & MASK64
        if _special(k) or k in seen:
            continue
        seen.add(k)
        out.append(k)
    return out


# ---- the index -------------------------------------------------------------------------------------------------
def index_bmask(slots: int) -> int:
    return slots // BUCKET_KEYS - 1


def index_home(h: int, slots: int) -> int:
    return int(h) & index_bmask(slots)


def index_keys(bucket: int, n: int, slots: int, rng, avoid=()) -> list:
    """n distinct keys homed at index bucket `bucket` of a table of `slots` keys"""
    bm = index_bmask(slots)
    assert 0 <= bucket <= bm
    return _fresh(lambda r: (r & ~bm) | bucket, n, rng, avoid)


def index_fillers_for(h: int, n: int, slots: int, rng, avoid=()) -> list:
    """n distinct keys other than h sharing the home bucket of the chain hash h"""
    return index_keys(index_home(h, slots), n, slots, rng, avoid=set(avoid) | {int(h)})


# ---- the device LRU --------------------------------------------------------------------------------------------
def pow2_ceil(x: int) -> int:
    return 1 << max(0, (int(x) - 1).bit_length())


def dlru_table_slots(C: int, lru_table_slots: int) -> int:
    """TS of a device LRU of capacity C with the option lru_table_slots pinned (engine_lru.cu, alloc_dev_lru:
    L = max(pow2_ceil(4 C), 64); TS = max(L, pow2_ceil(lru_table_slots)))"""
    assert lru_table_slots > 0, "the tests pin lru_table_slots: unpinned, TS depends on the free HBM"
    return max(max(pow2_ceil(4 * C), 64), pow2_ceil(lru_table_slots))


def dlru_log_records(C: int, TS: int) -> int:
    """L of the same LRU (alloc_dev_lru: max(pow2_ceil(4 C), 64), then at least TS / 4)"""
    return max(max(pow2_ceil(4 * C), 64), TS // 4)


def dlru_home(key: int, TS: int) -> int:
    return ((int(key) * PHI & MASK64) >> 40) & (TS - 1)


def dlru_key_of(x: int) -> int:
    """the key whose product with PHI is x (mod 2^64): dlru_home(dlru_key_of(x)) = (x >> 40) & (TS - 1)"""
    return int(x) * PHI_INV & MASK64


def dlru_keys(slot: int, n: int, TS: int, rng, avoid=()) -> list:
    """n distinct keys homed at slot `slot` of an LRU table of TS slots: k = X * PHI^-1 with the slot in bits 40 and up
    of X, every other bit of X random"""
    assert TS & (TS - 1) == 0 and 0 <= slot < TS
    field = (TS - 1) << 40
    return _fresh(lambda r: dlru_key_of((r & ~field) | (slot << 40)), n, rng, avoid)


# ---- models ----------------------------------------------------------------------------------------------------
class Probe:
    """where a lookup went: the slot found (None: a miss), the slots / buckets it visited from the home on, the
    tombstones it passed, and whether it wrapped past the end of the table"""

    def __init__(self, found, steps, tombs, wrapped):
        self.found, self.steps, self.tombs, self.wrapped = found, steps, tombs, wrapped

    @property
    def distance(self) -> int:
        return len(self.steps) - 1

    def __repr__(self):
        return f"Probe(found={self.found}, distance={self.distance}, tombs={self.tombs}, wrapped={self.wrapped})"


class IndexModel:
    """The index table and membership of one handle, for calls below the rebuild threshold.  apply() takes what
    fi_epp_index_apply takes and applies it like the engine: op groups of SETs, then CLEARs, with a new group started
    by a SET of a pair the open group CLEARs.  used / tombstones follow the device counters (a claim, a retirement)."""

    def __init__(self, slots: int):
        self.slots = slots
        self.bmask = index_bmask(slots)
        self.keys = [EMPTY] * slots
        self.rows = {}  # present key -> set of endpoints
        self.used = 0
        self.tombstones = 0

    # lookups follow bucket_scan: a bucket holding h ends the probe with a hit, one holding EMPTY with a miss
    def probe(self, h: int) -> Probe:
        h = int(h)
        b = h & self.bmask
        steps, tombs, wrapped = [], 0, False
        for _ in range(self.bmask + 1):
            steps.append(b)
            ks = self.keys[b * BUCKET_KEYS:(b + 1) * BUCKET_KEYS]
            if h in ks:
                return Probe(b * BUCKET_KEYS + ks.index(h), steps, tombs, wrapped)
            tombs += ks.count(TOMB)
            if EMPTY in ks:
                return Probe(None, steps, tombs, wrapped)
            wrapped |= b == self.bmask
            b = (b + 1) & self.bmask
        return Probe(None, steps, tombs, wrapped)

    def _claim(self, h: int) -> int:
        b = h & self.bmask
        for _ in range(self.bmask + 1):
            for j in range(BUCKET_KEYS):
                s = b * BUCKET_KEYS + j
                if self.keys[s] == h:
                    return s
                if self.keys[s] == EMPTY:
                    self.keys[s] = h
                    self.used += 1
                    return s
            b = (b + 1) & self.bmask
        raise AssertionError("model: index full")

    def _flush(self, sets, clears):
        for h, e in sets:
            if not _special(h):
                self._claim(h)
            self.rows.setdefault(h, set()).add(e)
        for h, e in clears:
            row = self.rows.get(h)
            if row is None or e not in row:
                continue
            row.discard(e)
            if not row:
                del self.rows[h]
                if not _special(h):
                    self.keys[self.probe(h).found] = TOMB
                    self.tombstones += 1

    def apply(self, ops):
        sets, clears, cleared = [], [], set()
        for h, e, op in ((int(o["hash"]), int(o["endpoint"]), int(o["op"])) for o in np.atleast_1d(ops)):
            if op == abi.FI_OP_SET:
                if (h, e) in cleared:
                    self._flush(sets, clears)
                    sets, clears, cleared = [], [], set()
                sets.append((h, e))
            else:
                clears.append((h, e))
                cleared.add((h, e))
        self._flush(sets, clears)

    def rebuilt(self):
        """index_rebuild_kernel ran: a fresh table holding the live keys (which key takes which slot of a run is up to
        the race; the slots the runs fill are not), used = live keys, no tombstones"""
        live = [h for h in self.rows if not _special(h)]
        self.keys = [EMPTY] * self.slots
        self.used = self.tombstones = 0
        for h in live:
            self._claim(h)

    def remove_endpoints(self, endpoints):
        """fi_epp_index_remove_endpoints: their bits leave every row, keys nobody holds any more are retired"""
        drop = {int(e) for e in endpoints}
        for h in list(self.rows):
            row = self.rows[h]
            if row & drop:
                row -= drop
                if not row:
                    del self.rows[h]
                    if not _special(h):
                        self.keys[self.probe(h).found] = TOMB
                        self.tombstones += 1

    def contains(self, e: int, h: int) -> bool:
        return int(e) in self.rows.get(int(h), ())

    def live_regular(self) -> int:
        return sum(1 for h in self.rows if not _special(h))

    def run_at(self, bucket: int) -> list:
        """the buckets of the run that starts at `bucket`: it and the full buckets that follow it, up to the first
        bucket with an EMPTY key (included)"""
        out, b = [], bucket
        for _ in range(self.bmask + 1):
            out.append(b)
            if EMPTY in self.keys[b * BUCKET_KEYS:(b + 1) * BUCKET_KEYS]:
                break
            b = (b + 1) & self.bmask
        return out


class LruModel:
    """One endpoint's device-LRU table: linear probing over TS slots from dlru_home, evictions and rolled-back inserts
    leave tombstones, `used` counts entries + tombstones like the device's.  The hashes 0 and ~0 have slots of their
    own and never enter the table.  The test tells it what the LRU did (which keys a sub-batch inserted, which left);
    maintain() replays lru_maintain_kernel's decision for a sub-batch of `touches` touches and rebuilds the table from
    the live keys when the kernel would."""

    def __init__(self, TS: int, C: int):
        self.TS, self.C, self.L = TS, C, dlru_log_records(C, TS)
        self.keys = [EMPTY] * TS
        self.used = 0
        self.head = 0  # log records since the last compaction

    def probe(self, key: int) -> Probe:
        key = int(key)
        i = dlru_home(key, self.TS)
        steps, tombs, wrapped = [], 0, False
        for _ in range(self.TS):
            steps.append(i)
            k = self.keys[i]
            if k == key:
                return Probe(i, steps, tombs, wrapped)
            if k == EMPTY:
                return Probe(None, steps, tombs, wrapped)
            tombs += k == TOMB
            wrapped |= i == self.TS - 1
            i = (i + 1) & (self.TS - 1)
        return Probe(None, steps, tombs, wrapped)

    def insert(self, keys):
        """the new keys of one sub-batch (any order: the slots they fill do not depend on it)"""
        for key in keys:
            key = int(key)
            if _special(key) or self.probe(key).found is not None:
                continue
            i = dlru_home(key, self.TS)
            while self.keys[i] != EMPTY:
                i = (i + 1) & (self.TS - 1)
            self.keys[i] = key
            self.used += 1

    def retire(self, keys):
        for key in keys:
            if not _special(int(key)):
                s = self.probe(key).found
                assert s is not None, f"model: retiring {key:#x}, which is not in the table"
                self.keys[s] = TOMB

    def maintain(self, touches: int, live_in_order) -> tuple:
        """-> (ran, rebuilt) for a sub-batch bringing `touches` touches to this endpoint; live_in_order = its entries,
        oldest first, before the sub-batch (the compacted log a rebuild re-inserts)"""
        addc = min(touches, self.C)
        log_tight = self.head + addc > self.L
        tab_tight = (self.used + addc) * 10 > self.TS * 6
        if not (log_tight or tab_tight):
            return False, False
        live = [int(k) for k in live_in_order]
        self.head = len(live)
        if not tab_tight:
            return True, False
        self.keys = [EMPTY] * self.TS
        self.used = 0
        self.insert(live)
        return True, True

    def appended(self, records: int):
        self.head += records

    def tombstones(self) -> int:
        return self.keys.count(TOMB)
