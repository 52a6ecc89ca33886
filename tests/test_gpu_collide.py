"""GPU (-m gpu): the index and the device LRU under crafted key collisions, bit for bit against the CPU references.

tests/collide.py places keys exactly where a test wants them: full home buckets, runs that wrap from the last bucket
(slot) to the first, runs that merge, tombstones at the start, middle and end of runs, one new key claimed by several
CTAs at once.  Its models replay every call and the tests assert that each crafted layout really happened (a probe
that wraps, a key behind tombstones, a miss decided past its home), so a drift between a constructor and the kernels
cannot leave a test checking nothing.  Membership is compared with oracle/epp_oracle.cpp, picks with the ranked
oracle, removals with tests/remove_ref.py, and the device LRU's recency order with tests/capacity_oracle.py.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, make_config
from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import collide as X
from tests import helpers as H
from tests.capacity_oracle import CapacityOracle
from tests.ranked_oracle import RankedOracle
from tests.remove_ref import RemovalOracle

pytestmark = pytest.mark.gpu
SET, CLEAR = abi.FI_OP_SET, abi.FI_OP_CLEAR
MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
WEIGHTED = [{"name": "default", "scorers": [(H.P, 100), (H.K, 13), (H.Q, 7)]}]
M64 = X.MASK64


def _ops(pairs, op):
    return H.ops_array([(int(h), int(e), op) for h, e in pairs])


def _membership(gpu, ref, keys, endpoints, what=""):
    """index_contains over every (key, endpoint) pair against the reference (endpoints: a count or a list)"""
    keys = sorted({int(k) for k in keys})
    eps = np.arange(endpoints) if np.isscalar(endpoints) else np.asarray(sorted(endpoints))
    q = np.zeros(len(keys) * len(eps), dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(np.asarray(keys, dtype=np.uint64), len(eps))
    q["endpoint"] = np.tile(eps.astype(np.uint32), len(keys))
    got = gpu.index_contains(q)
    want = np.array([ref.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
    bad = np.flatnonzero(got != want)
    assert not len(bad), f"{what}: {len(bad)} of {len(q)} memberships differ, first " + ", ".join(
        f"({int(q['hash'][i]):#x}, {int(q['endpoint'][i])}): got {got[i]}" for i in bad[:4])


# ---- a. index membership -------------------------------------------------------------------------------------------
class _Index:
    """a handle, the oracle and the table model fed the same fi_epp_index_apply calls"""

    def __init__(self, slots, E=8):
        self.E = E
        self.cfg = make_config(num_endpoints=E, max_blocks=32, lru_capacity=0, max_batch=64, index_slots=slots)
        self.gpu, self.ref, self.model = EndpointPicker(self.cfg), eo.Oracle(self.cfg), X.IndexModel(slots)
        self.rng = np.random.default_rng(slots)
        self.ever = set()
        self.probes = set()  # keys never SET, sharing homes with the runs: their lookups are misses through runs

    def close(self):
        self.gpu.close()
        self.ref.close()

    def keys(self, bucket, n):
        ks = X.index_keys(bucket, n, self.model.slots, self.rng, avoid=self.ever | self.probes)
        self.probes.update(X.index_keys(bucket, 2, self.model.slots, self.rng, avoid=self.ever | self.probes | set(ks)))
        return ks

    def apply(self, ops, model=True):
        self.gpu.index_apply(ops)
        self.ref.index_apply(ops)
        if model:
            self.model.apply(ops)
        self.ever.update(int(h) for h in ops["hash"])

    def set(self, keys, eps=None):
        """SET each key on one or two endpoints (eps[i] or random), in one call"""
        pairs = []
        for i, k in enumerate(keys):
            es = eps[i] if eps is not None else self.rng.choice(self.E, size=int(self.rng.integers(1, 3)), replace=False)
            pairs += [(k, e) for e in np.atleast_1d(es)]
        self.apply(_ops(pairs, SET))
        return keys

    def retire(self, keys):
        """CLEAR every endpoint of each key: the keys become tombstones"""
        self.apply(_ops([(k, e) for k in keys for e in sorted(self.model.rows[int(k)])], CLEAR))

    def bucket(self, b):
        return self.model.keys[b * 4:(b + 1) * 4]

    def check(self, what, layout=True):
        st = self.gpu.index_stats()
        live = self.model.live_regular()
        assert st.used - st.tombstones == live, f"{what}: used - tombstones = {st.used - st.tombstones}, live keys {live}"
        if layout:
            assert st.rebuilds == 0, f"{what}: an index rebuild would void the layout"
            assert (st.used, st.tombstones) == (self.model.used, self.model.tombstones), what
        _membership(self.gpu, self.ref, self.ever | self.probes, self.E, what)


def test_index_membership_through_runs_64_slots():
    """The smallest table, 16 buckets, driven to one empty slot and through a rebuild (hand-worked layout in the
    comments; the model asserts each step)."""
    t = _Index(64)
    m = t.model
    # one home bucket holding 4·2 keys: bucket 5, then 6
    a1 = t.set(t.keys(5, 4))
    a2 = t.set(t.keys(5, 4))
    assert all(m.probe(k).steps == [5, 6] for k in a2)
    # runs homed at the last and second-to-last bucket, wrapping into bucket 0
    b1 = t.set(t.keys(15, 4))
    b2 = t.set(t.keys(15, 2))
    c1 = t.set(t.keys(14, 4))
    c2 = t.set(t.keys(14, 2))
    assert all(m.probe(k).wrapped and m.probe(k).steps == [15, 0] for k in b2)
    assert all(m.probe(k).wrapped and m.probe(k).steps == [14, 15, 0] for k in c2)
    assert X.EMPTY not in t.bucket(0)
    t.check("wrapped runs")
    # two runs that merge: a run homed at 7 fills the bucket behind run 5-6, and keys homed at 5 then probe through it
    d1 = t.set(t.keys(7, 4))
    d2 = t.set(t.keys(5, 2))
    assert all(m.probe(k).steps == [5, 6, 7, 8] for k in d2)
    assert all(X.index_home(k, 64) == 7 for k in t.bucket(7))
    t.check("merged runs")
    # tombstones at the start, middle and end of both runs; one more key only loses an endpoint (no tombstone)
    two = next(k for k in a1 + a2 + c1 if len(m.rows[k]) == 2 and k not in (a1[0], a2[0], c1[0]))
    t.apply(_ops([(two, min(m.rows[two]))], CLEAR))
    t.retire([a1[0], a2[0], d2[0], c1[0], b1[0], b2[0]])
    assert t.bucket(5).count(X.TOMB) == t.bucket(6).count(X.TOMB) == t.bucket(8).count(X.TOMB) == 1
    assert t.bucket(14).count(X.TOMB) == t.bucket(15).count(X.TOMB) == t.bucket(0).count(X.TOMB) == 1
    assert m.probe(d2[1]).tombs == 2 and m.probe(c2[0]).tombs == 2 and m.probe(c2[0]).wrapped
    t.check("tombstones in runs")
    # re-SETs of retired keys claim new slots past their runs
    t.set([a1[0], b2[0]], eps=[[3], [6]])
    p, q = m.probe(a1[0]), m.probe(b2[0])
    assert p.steps == [5, 6, 7, 8] and p.tombs == 2 and q.steps == [15, 0, 1] and q.tombs == 2 and q.wrapped
    t.check("re-SET of retired keys")
    # one new key at op positions 257 apart: eight CTAs race to claim it (two such keys); the ops in between are SETs
    # of pairs already present
    k1, k2 = t.keys(5, 1)[0], t.keys(14, 1)[0]
    present = [(h, e) for h, row in m.rows.items() for e in row if h not in (0, M64)]
    pairs = [present[i % len(present)] for i in range(8 * 257)]
    for i in range(8):
        pairs[i * 257] = (k1, i % t.E)
        pairs[i * 257 + 1] = (k2, (i + 3) % t.E)
    t.apply(_ops(pairs, SET))
    assert m.probe(k1).steps == [5, 6, 7, 8] and m.probe(k2).steps == [14, 15, 0, 1]
    t.check("one key claimed by several CTAs")
    # churn: 14 keys homed at 10 come and go, five more keys leave: 25 tombstones, 19 live keys, 44 slots used
    churn = t.set(t.keys(10, 14))
    t.retire(churn + [a1[1], a2[1], b1[1], c1[1], d1[0]])
    assert (m.used, m.tombstones, m.live_regular()) == (44, 25, 19)
    t.check("churn")
    # 19 distinct new keys homed at 10 in one call fill every empty slot but one; three of them sit in bucket 9, a full
    # lap from their home (index_resolve_overflow's last bucket)
    last = t.set(t.keys(10, 19))
    assert m.keys.count(X.EMPTY) == 1 and m.live_regular() == 38
    far = [k for k in last if m.probe(k).distance == m.bmask]
    assert len(far) == 3 and all(m.probe(k).wrapped for k in far)
    t.check("one empty slot left")
    # the next call finds 63 of 64 slots used: a rebuild with every run live
    t.set([last[0]], eps=[[7]])
    st = t.gpu.index_stats()
    assert st.rebuilds >= 1 and st.tombstones == 0 and st.used == m.live_regular()
    m.rebuilt()
    t.check("after the rebuild", layout=False)
    t.retire(last[:10])
    t.set(t.keys(9, 6), eps=None)
    t.check("after the rebuild, more calls", layout=False)
    t.close()


def test_index_membership_through_runs_4096_slots():
    t = _Index(4096)
    m = t.model
    last = m.bmask
    # one home bucket holding 4·40 keys, in four calls of 40 (distinct new keys with one home in a single call)
    home = [t.set(t.keys(100, 40)) for _ in range(4)]
    assert all(m.probe(k).distance >= 30 for k in home[3])
    # runs homed at the last and second-to-last bucket, wrapping
    r1 = t.set(t.keys(last, 30))
    r2 = t.set(t.keys(last - 1, 30))
    assert sum(m.probe(k).wrapped for k in r1) == 26 and sum(m.probe(k).wrapped for k in r2) == 26
    t.check("home bucket and wrapped runs")
    # runs homed at 3 and 5 merge with the wrapped one (it ends in bucket 13)
    t.set(t.keys(3, 12))
    mid = t.set(t.keys(5, 12))
    assert m.run_at(last - 1)[-1] > 13 and all(m.probe(k).distance >= 10 for k in mid)
    t.check("merged runs")
    # tombstones at the start, middle and end of the run homed at 100, then a late key and re-SETs past it
    t.retire([home[0][0], home[1][5], home[2][7], home[3][-1]] + r1[:3] + r2[-3:])
    late = t.set(t.keys(100, 3))
    assert all(m.probe(k).tombs >= 3 for k in late)
    t.set([home[0][0], r1[0]], eps=[[1], [2]])
    assert m.probe(home[0][0]).tombs >= 4 and m.probe(r1[0]).tombs >= 3 and m.probe(r1[0]).wrapped
    t.check("tombstones in runs, re-SETs")
    # new keys at op positions 257 apart, each claimed by eight CTAs at once, behind the long runs
    new = [t.keys(100, 1)[0], t.keys(last, 1)[0], t.keys(last - 1, 1)[0]]
    present = [(h, e) for h, row in m.rows.items() for e in row]
    pairs = [present[i % len(present)] for i in range(8 * 257)]
    for i in range(8):
        for j, k in enumerate(new):
            pairs[i * 257 + j] = (k, (i + j) % t.E)
    t.apply(_ops(pairs, SET))
    assert all(m.probe(k).found is not None and m.probe(k).distance >= 10 for k in new)
    t.check("keys claimed by several CTAs")
    t.close()


# ---- b. picks through runs; c. removal through runs ------------------------------------------------------------------
class _PickScene:
    """Requests whose chains sit in crafted runs of a 4096-slot index.  Before the chains are added, filler keys (on
    endpoints, none of them in any chain) fill the home bucket of every request's first block, of the first block no
    endpoint holds, and of a few held blocks: from there to the last bucket (so those blocks wrap) or just their home
    bucket, CLEARed after the chains are added (tombstones between those blocks and their homes)."""

    SLOTS, R, MB, BB, BATCH = 4096, 48, 32, 64, 4800

    def __init__(self, E, mode, shuffled, seed=11, ref_cls=RankedOracle):
        self.E, self.mode = E, mode
        self.cfg = make_config(num_endpoints=E, block_bytes=self.BB, max_blocks=self.MB, lru_capacity=0, max_batch=self.BATCH,
                               profiles=WEIGHTED, match_mode=mode, index_slots=self.SLOTS)
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.gpu, self.ref, self.model = EndpointPicker(self.cfg), ref_cls(self.cfg), X.IndexModel(self.SLOTS)
        st = H.states_array(E, kv=rng.integers(0, 1024, size=E) / 1024.0, queue=rng.integers(0, 32, size=E))
        self.gpu.update_endpoints(st)
        self.ref.update_endpoints(st)
        self.h0 = 0x5EED
        S = self.SLOTS
        home = lambda h: X.index_home(h, S)
        # requests: at least four have a held block past the fourth (the lazy probe's range) homed in the last buckets
        blobs, held, wraps = [], [], []
        while len(blobs) < self.R:
            n = int(rng.integers(12, self.MB + 1))
            blob = rng.integers(0, 256, size=n * self.BB, dtype=np.uint8).tobytes()
            ch = self._chain(blob)
            eps = rng.choice(E, size=int(rng.integers(1, 4)), replace=False)
            lens = {int(e): int(rng.integers(6, n + 1)) for e in eps}
            if rng.random() < 0.15:
                lens = {}  # nobody holds it: the very first lookup is the miss
            m_held = max(lens.values(), default=0)
            w = [j for j in range(5, m_held) if home(ch[j]) >= S // 4 - 6]
            if len(wraps) < 4 and not w and len(blobs) >= self.R - 4:
                continue
            if w:
                wraps.append((len(blobs), w[0]))
            blobs.append(blob)
            held.append(lens)
        self.tok, self.offs = H.pack_prompts(blobs)
        self.chains, self.nb = self.ref.hash_batch(self.tok, self.offs, self.h0)
        self.held, self.wraps = held, wraps
        self.m = [max(h.values(), default=0) for h in held]
        chain_keys = {int(k) for r in range(self.R) for k in self.chains[r, : self.nb[r]]}
        used = set(chain_keys)
        fill, tomb_fill = [], []

        def fillers(h, n):
            f = X.index_fillers_for(h, n, S, rng, avoid=used)
            used.update(f)
            return f

        for r in range(self.R):
            fill += fillers(self.chains[r, 0], 4)                       # h_1's home bucket full
            if self.m[r] < self.nb[r]:
                fill += fillers(self.chains[r, self.m[r]], 4)           # the miss decided past its home
        for r, j in wraps:                                              # buckets home .. last full: the block wraps
            fill += fillers(self.chains[r, j], 4 * (S // 4 - home(self.chains[r, j])))
        self.tomb_blocks = []
        for r in range(0, self.R, 5):                                   # tombstones between a held block and its home
            if self.m[r] > 8:
                j = int(rng.integers(4, self.m[r]))
                self.tomb_blocks.append((r, j))
                tomb_fill += fillers(self.chains[r, j], 4)
        self.fill_pairs = [(f, int(rng.integers(0, E))) for f in fill + tomb_fill]
        self.tomb_pairs = [p for p in self.fill_pairs if p[0] in set(tomb_fill)]
        self.chain_pairs = [(int(self.chains[r, j]), e) for r in range(self.R) for j in range(self.nb[r])
                            for e, L in sorted(held[r].items()) if j < L]
        if shuffled:
            rng.shuffle(self.chain_pairs)
        self.apply(_ops(self.fill_pairs, SET))
        self.apply(_ops(self.chain_pairs, SET))
        self.apply(_ops(self.tomb_pairs, CLEAR))
        self.ever = chain_keys | {f for f, _ in self.fill_pairs}
        self.endpoints = {e for _, e in self.fill_pairs} | {e for h in held for e in h} | {0, E - 1}

    def _chain(self, blob):
        tok, offs = H.pack_prompts([blob])
        ch, nb = self.ref.hash_batch(tok, offs, 0x5EED)
        return [int(x) for x in ch[0, : nb[0]]]

    def apply(self, ops):
        self.gpu.index_apply(ops)
        self.ref.index_apply(ops)
        self.model.apply(ops)

    def assert_layout(self):
        """race-free properties: they hold whichever slots the keys of one call took"""
        m, S = self.model, self.SLOTS
        st = self.gpu.index_stats()
        assert st.rebuilds == 0 and (st.used, st.tombstones) == (m.used, m.tombstones)
        for r in range(self.R):
            h1 = int(self.chains[r, 0])
            b = m.keys[X.index_home(h1, S) * 4:][:4]
            assert h1 not in b and X.EMPTY not in b, f"request {r}: h_1's home bucket is not full without it"
            if self.m[r] < self.nb[r]:
                p = m.probe(self.chains[r, self.m[r]])
                assert p.found is None and p.distance >= 1, f"request {r}: miss decided at home"
        assert len(self.wraps) >= 4
        for r, j in self.wraps:
            p = m.probe(self.chains[r, j])
            assert p.found is not None and p.wrapped, f"request {r} block {j} does not wrap"
        assert len(self.tomb_blocks) >= 4
        for r, j in self.tomb_blocks:
            assert m.probe(self.chains[r, j]).tombs >= 1, f"request {r} block {j}: no tombstone before it"

    def close(self):
        self.gpu.close()
        self.ref.close()


def _eq(got, want, what):
    assert got.tobytes() == want.tobytes(), what + "\n" + H.describe_diff(got, want)


@pytest.mark.parametrize("shuffled", [False, True], ids=["chain_order", "shuffled"])
@pytest.mark.parametrize("mode", MODES, ids=["upstream", "lpm"])
@pytest.mark.parametrize("E", [40, 2048])
def test_picks_through_runs(E, mode, shuffled):
    import torch

    s = _PickScene(E, mode, shuffled)
    s.assert_layout()
    # the requests repeated until the launch has more requests than warps: a warp that takes a second request finds
    # its first block's home bucket prefetched (full without the block, so the lookup continues in the table)
    copies = 100
    blobs = [bytes(s.tok[int(s.offs[r]):int(s.offs[r + 1])]) for r in range(s.R)]
    tok, offs = H.pack_prompts(blobs * copies)
    h0, R = s.h0, s.R * copies
    single = s.gpu.pick_batch(tok, offs, h0)
    want = s.ref.pick_batch(tok, offs, h0)
    _eq(single, want, "pick_batch vs the oracle")
    assert (want[: s.R, 0]["match_blocks"] > 0).sum() >= s.R // 2
    ranked = s.gpu.pick_batch_ranked(tok, offs, h0, 4)
    _eq(ranked, s.ref.pick_batch_ranked(tok, offs, h0, 4), "pick_batch_ranked k=4 vs the oracle")
    # the pipelined submit, k = 0
    d_tok = torch.from_numpy(tok.copy()).cuda()
    d_off = torch.from_numpy(offs.view(np.int64).copy()).cuda()
    d_h0 = torch.full((R,), h0, dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    t = s.gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(offs[-1]), d_out.data_ptr(), k=0,
                             stream=st)
    s.gpu.pick_wait_batch(t, st)
    torch.cuda.synchronize()
    _eq(d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1), want, "pick_submit_ex k=0 vs the oracle")
    _membership(s.gpu, s.ref, s.ever, s.endpoints, "membership")
    s.close()


@pytest.mark.parametrize("mode", MODES, ids=["upstream", "lpm"])
def test_removal_through_runs(mode):
    s = _PickScene(40, mode, shuffled=False, seed=12, ref_cls=RemovalOracle)
    s.assert_layout()
    ref, gpu, m = s.ref, s.gpu, s.model
    # the endpoints holding the blocks that wrap or sit behind tombstones, and a filler endpoint
    victims = sorted({e for r, _ in s.wraps + s.tomb_blocks for e in s.held[r]})[:6]
    for drop in (victims[:3], victims[3:] + [s.fill_pairs[0][1]]):
        got = gpu.remove_endpoints(drop, count=True)
        assert got == ref.remove_endpoints(drop)
        m.remove_endpoints(drop)
        st = gpu.index_stats()
        assert st.used - st.tombstones == m.live_regular() and st.tombstones == m.tombstones
        _membership(gpu, ref, s.ever, s.endpoints, f"after removing {drop}")
        _eq(gpu.pick_batch(s.tok, s.offs, s.h0), ref.pick_batch(s.tok, s.offs, s.h0), f"picks after removing {drop}")
    # the removed endpoints take their chains again: the keys are re-claimed past the tombstones the removal left
    again = [(h, e) for h, e in s.chain_pairs if e in victims]
    s.apply(_ops(again, SET))
    assert any(m.probe(s.chains[r, j]).tombs >= 1 for r, j in s.tomb_blocks + s.wraps)
    st = gpu.index_stats()
    assert st.used - st.tombstones == m.live_regular() and (st.used, st.tombstones) == (m.used, m.tombstones)
    _membership(gpu, ref, s.ever, s.endpoints, "after the re-Add")
    _eq(gpu.pick_batch(s.tok, s.offs, s.h0), ref.pick_batch(s.tok, s.offs, s.h0), "picks after the re-Add")
    s.close()


# ---- d. the device LRU -------------------------------------------------------------------------------------------------
class _Lru:
    """a device-LRU handle (lru_table_slots pinned), the capacity oracle and one LruModel per endpoint"""

    C, MB, E = 64, 32, 4

    def __init__(self, ts_option):
        self.cfg = make_config(num_endpoints=self.E, max_blocks=self.MB, lru_capacity=self.C, max_batch=32,
                               index_slots=1 << 14)
        self.gpu = EndpointPicker(self.cfg)
        self.gpu.set_option("device_lru", 1)
        self.gpu.set_option("lru_table_slots", ts_option)
        self.ref = CapacityOracle(self.cfg)
        self.TS = X.dlru_table_slots(self.C, ts_option)
        self.models = [X.LruModel(self.TS, self.C) for _ in range(self.E)]
        self.caps = [self.C] * self.E
        self.rng = np.random.default_rng(ts_option)
        self.ever = set()
        self.tracked = True  # the models follow the device (false after a pass the models do not replay)
        self.maintained = 0
        self.rebuilds = [0] * self.E  # table rebuilds the models replayed

    def close(self):
        self.gpu.close()
        self.ref.close()

    def keys(self, slot, n):
        ks = X.dlru_keys(slot % self.TS, n, self.TS, self.rng, avoid=self.ever)
        self.ever.update(ks)
        return ks

    def add(self, reqs, what):
        """reqs: [(endpoint, chain)] in request order, one fi_epp_index_add_chains call"""
        eps = np.array([e for e, _ in reqs], dtype=np.uint32)
        chains = np.zeros((len(reqs), self.MB), dtype=np.uint64)
        nb = np.array([len(c) for _, c in reqs], dtype=np.uint32)
        for r, (_, c) in enumerate(reqs):
            chains[r, : len(c)] = np.asarray(c, dtype=np.uint64)
            self.ever.update(int(k) for k in c)
        before = [self.ref.lru(e) for e in range(self.E)]
        self.gpu.index_add_chains(eps, chains, nb)
        self.ref.index_add_chains(eps, chains, nb)
        if self.tracked:  # one sub-batch: maintain, inserts, appends, evictions
            ran = 0
            for e, mdl in enumerate(self.models):
                mine = [c for ep, c in reqs if ep == e]
                r, rb = mdl.maintain(sum(len(c) for c in mine), before[e])
                ran += r
                self.rebuilds[e] += rb
                touched = list(dict.fromkeys(int(k) for c in mine for k in c))
                mdl.insert([k for k in touched if k not in set(int(x) for x in before[e])])
                mdl.appended(min(len(touched), self.caps[e]))
                after = set(int(k) for k in self.ref.lru(e))
                mdl.retire([k for k in set(int(x) for x in before[e]) | set(touched) if k not in after])
            self.maintained += ran
        self.check(what)

    def check(self, what):
        for e in range(self.E):
            assert np.array_equal(self.gpu.lru_dump(e), self.ref.lru(e)), f"{what}: LRU of endpoint {e}"
        assert self.gpu.index_stats().lru_entries == sum(self.ref.lru_size(e) for e in range(self.E)), what
        if self.tracked:
            assert self.gpu.lru_counters()["maintained"] == self.maintained, f"{what}: maintenance passes"
        _membership(self.gpu, self.ref, self.ever, self.E, what)


@pytest.mark.parametrize("ts_option", [1, 512], ids=["TS256", "TS512"])
def test_device_lru_through_runs(ts_option):
    t = _Lru(ts_option)
    TS, mdl = t.TS, t.models
    assert TS == (256 if ts_option == 1 else 512)
    # runs homed at TS - 1 and TS - 2 (with the hashes 0 and ~0 in the chain); endpoint 1 gets the same 24 new keys
    # from four requests of one batch (the same-key CAS race)
    a = t.keys(TS - 1, 16)
    b = t.keys(TS - 2, 8)
    shared = t.keys(TS - 1, 24)
    perm = lambda ks: [ks[i] for i in t.rng.permutation(len(ks))]
    t.add([(0, a[:8] + [0] + b + [M64] + a[8:]), (1, perm(shared)), (1, perm(shared)), (1, perm(shared)),
           (1, perm(shared))], "first runs")
    p = [mdl[0].probe(k) for k in a + b]
    assert sorted(q.found for q in p) == sorted([(TS - 2 + i) % TS for i in range(24)])
    assert sum(q.wrapped for q in p) >= 14 and all(mdl[1].probe(k).found is not None for k in shared)
    # a later call: 16 keys homed at TS - 1 land behind the run, past the end of the table
    c = t.keys(TS - 1, 16)
    t.add([(0, c)], "keys behind a wrapped run")
    assert all(mdl[0].probe(k).distance >= 23 and mdl[0].probe(k).wrapped for k in c)
    # 32 more keys: the 10 oldest (the hash 0 and keys of the first run) are evicted into tombstones in front of the later keys
    d = t.keys(TS - 2, 32)
    t.add([(0, d)], "evictions inside the run")
    assert mdl[0].tombstones() == 9  # (the hash 0 among them has a slot of its own)
    assert all(mdl[0].probe(k).tombs >= 8 and mdl[0].probe(k).wrapped for k in c)
    # endpoint 1: more of its run's keys, evicting the oldest shared ones (tombstones inside its run)
    t.add([(1, t.keys(TS - 1, 32)), (1, t.keys(TS - 1, 24))], "evictions on endpoint 1")
    assert mdl[1].tombstones() >= 16
    # churn on both endpoints until maintenance rebuilds a table crowded with tombstones
    for i in range(40):
        t.add([(0, t.keys(TS - 1 - 2 * (i % 3), 16) + t.keys(int(t.rng.integers(0, TS)), 16)),
               (1, t.keys(TS - 2, 8) + [0, M64]),
               (3, t.keys(TS // 2, 4))], f"churn {i}")
        if t.rebuilds[0]:
            break
    assert t.rebuilds[0] == 1 and t.gpu.lru_counters()["maintained"] >= 1
    # a resize that evicts from inside the runs
    before = t.ref.lru(0)
    got = t.gpu.set_lru_capacities([0, 1], [t.MB, 40], want_evicted=True)
    gone = t.ref.set_lru_capacities([0, 1], [t.MB, 40])
    assert got == len(gone) >= 32
    for e, cap in ((0, t.MB), (1, 40)):
        t.caps[e] = cap
    mdl[0].retire([h for h, e in gone if e == 0])
    mdl[1].retire([h for h, e in gone if e == 1])
    assert len(before) == t.C and mdl[0].tombstones() >= 32
    t.check("resize")
    # one batch brings endpoint 2 more new keys than its table takes (0.85 TS): its touches are rolled back into
    # tombstones inside its runs and its requests deferred to sub-batches that fit
    t.add([(2, t.keys(TS - 1, 20))], "endpoint 2 before the overflow")
    limit = TS * 85 // 100
    n_req = limit // 30 + 2
    reqs = [(2, t.keys(TS - 1 - (r % 4) * 9, 30) + ([0] if r == 0 else [])) for r in range(n_req)]
    reqs[1] = (2, reqs[1][1][:28] + [int(x) for x in t.ref.lru(2)[:2]])  # two existing entries touched again
    t.tracked = False
    deferred = t.gpu.lru_counters()["deferred_requests"]
    t.add(reqs, "deferred endpoint")
    assert sum(len(set(c)) for _, c in reqs) > limit
    assert t.gpu.lru_counters()["deferred_requests"] > deferred
    # the endpoint keeps working afterwards
    t.add([(2, t.keys(TS - 1, 24)), (0, t.keys(TS - 2, 24))], "after the deferral")
    t.close()
