"""GPU (-m gpu): index snapshots (fi_epp_snapshot_save / fi_epp_snapshot_load, docs/SPEC.md S.2d).

A snapshot stores the pair set, the LRU lists and the capacities; tests/test_snapshot_cpu.py shows on the oracle that
these carry every later call.  Here the GPU's blobs are read with the independent reader of tests/snapshot_ref.py and
held to the extended oracle (tests/ext_oracle.py) after a churn history; loaded handles of other internal sizes are
compared bit for bit with the source and the oracle, also over further pick + Add steps; a save of a load gives the
same bytes (node order is kept); failing loads change nothing; loads are ordered against submitted batches and tickets;
and an aged cfg 3 handle round-trips.
"""
import ctypes as C

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, make_config, snapshot_info, synth
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import craft
from tests import helpers as H
from tests import resize_ref as RR
from tests import snapshot_ref as SR
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu
U64_MAX = 0xFFFFFFFFFFFFFFFF


def _handle(cfg, table_slots=0, host_lru=False):
    gpu = EndpointPicker(cfg)
    if table_slots:
        gpu.set_option("lru_table_slots", table_slots)
    if host_lru:
        gpu.set_option("device_lru", 0)
    return gpu


class Aged:
    """a GPU handle and the oracle after the same churn history: states, adapters, direct SETs and CLEARs (the markers
    0 and ~0 and crafted hashes included), Adds with evictions, capacities (one lowered below its LRU's size) and a
    removal.  `hist` keeps the state and adapter calls, which a loaded handle is sent again."""

    def __init__(self, E=40, seed=1, mode=abi.FI_MATCH_UPSTREAM, lru_capacity=48, n=16):
        self.cfg = RR.config(E, match_mode=mode, lru_capacity=lru_capacity)
        self.E = E
        self.cs = RR.CallStream(seed, RR.config(E, match_mode=mode))
        self.gpu = _handle(self.cfg)
        self.ora = ExtOracle(self.cfg, track_removal=True)
        self.hist = [("states", H.states_array(E, roles=abi.FI_ROLE_WORKER | RR.LABEL))]
        self.both(self.hist[0])
        calls = self.cs.calls(E, n=n)
        if not lru_capacity:
            calls = [c for c in calls if c[0] in ("states", "lora", "ops")]
        for i, entry in enumerate(calls):
            self.both(entry)
            if i == n // 2 and lru_capacity:
                self.remove([int(self.cs.rng.integers(0, E))])
        zero, ones = craft.MARKERS
        self.both(("ops", H.ops_array([(zero, 1, abi.FI_OP_SET), (ones, 2, abi.FI_OP_SET), (ones, 3, abi.FI_OP_SET),
                                       (zero, 4, abi.FI_OP_SET), (zero, 4, abi.FI_OP_CLEAR)])))
        if lru_capacity:  # chains whose second block hashes to a marker, Added to endpoints 6 and 7
            B = self.cfg.block_bytes
            blocks = [self.cs.rng.integers(0, 256, size=B, dtype=np.uint8).tobytes() for _ in range(4)]
            tok, offs = H.pack_prompts([b"".join(blocks)])
            for e, target in zip((6, 7), craft.MARKERS):
                chains, nb = self.ora.hash_batch(tok, offs, craft.h0_for(blocks, 1, target))
                assert int(chains[0, 1]) == target
                self.both(("chains", np.array([e], np.uint32), chains, nb.astype(np.uint32)))
        if lru_capacity:
            e = max(range(E), key=lambda x: self.ora.lru_size(x))
            self.both(("caps", np.array([e], np.uint32), np.array([self.cfg.max_blocks], np.uint32)))

    def both(self, entry):
        RR.apply(self.gpu, entry)
        RR.apply(self.ora, entry)
        if entry[0] in ("states", "lora"):
            self.hist.append(entry)

    def remove(self, eps):
        self.gpu.remove_endpoints(eps)
        self.ora.remove_endpoints(eps)

    def loaded(self, blob, index_slots=0, table_slots=0):
        cfg = abi.fi_epp_config.from_buffer_copy(self.cfg)
        cfg.index_slots = index_slots
        g = _handle(cfg, table_slots)
        for entry in self.hist:
            RR.apply(g, entry)
        g.load_snapshot(blob)
        return g

    def close(self):
        self.gpu.close()
        self.ora.close()


def _picks(a, b, cs, E, what):
    """single (with adapters), ranked k = 4 and subset picks of a and b (a GPU handle or the oracle) are bit-equal"""
    tok, offs, h0 = cs.tok, cs.offs, cs.h0
    ad = cs.adapters()
    got, want = a.pick_batch(tok, offs, h0, adapters=ad), b.pick_batch(tok, offs, h0, adapters=ad)
    assert H.picks_equal(got, want), what + " (single)\n" + H.describe_diff(got, want)
    got, want = a.pick_batch(tok, offs, h0), b.pick_batch(tok, offs, h0)
    assert H.picks_equal(got, want), what + " (plain)\n" + H.describe_diff(got, want)
    got, want = a.pick_batch_ranked(tok, offs, h0, 4, adapters=ad), b.pick_batch_ranked(tok, offs, h0, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (ranked)\n" + H.describe_diff(got, want)
    sub = cs.subsets(E)
    got, want = a.pick_batch_subset(tok, offs, h0, sub, 4, adapters=ad), b.pick_batch_subset(tok, offs, h0, sub, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (subset)\n" + H.describe_diff(got, want)


def _contains(gpu, hashes, E):
    q = np.zeros(len(hashes) * E, dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(hashes, E)
    q["endpoint"] = np.tile(np.arange(E, dtype=np.uint32), len(hashes))
    return gpu.index_contains(q)


def _same(gpu, ora, cs, E, what, lru=True):
    """gpu equals the oracle: picks, membership of every hash the calls used, every LRU"""
    _picks(gpu, ora, cs, E, what)
    got = _contains(gpu, cs.hashes, E)
    want = np.array([ora.index_contains(e, int(h)) for h in cs.hashes for e in range(E)], dtype=np.uint8)
    assert np.array_equal(got, want), f"{what}: {int((got != want).sum())} memberships differ"
    if lru:
        for e in range(E):
            assert np.array_equal(gpu.lru_dump(e), ora.lru(e)), (what, e)


@pytest.mark.parametrize("E", [40, 100])
def test_save_matches_the_oracle(E):
    a = Aged(E=E, seed=E)
    blob = a.gpu.save_snapshot()
    s = SR.read(blob)  # (the reader checks the magic, sizes and checksum)
    pairs, lrus, caps = a.ora.state()
    assert s.pairs() == pairs
    assert {(1, 0), (2, U64_MAX), (3, U64_MAX)} <= pairs and (4, 0) not in pairs
    assert s.caps.tolist() == caps and min(caps) == a.cfg.max_blocks
    for e in range(E):
        assert np.array_equal(s.lrus[e], lrus[e]), e
    assert (s.block_bytes, s.max_blocks, s.lru_capacity, s.num_endpoints) == \
        (a.cfg.block_bytes, a.cfg.max_blocks, a.cfg.lru_capacity, E)
    info = snapshot_info(blob)
    assert info.pairs == len(pairs) and info.n_nodes == len(s.node_keys) and info.bytes == len(blob)
    st = a.gpu.index_stats()
    assert info.n_lru == st.lru_entries
    a.close()


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_load_then_continue(mode):
    """Loaded into handles with another index_slots and lru_table_slots, the state picks, dumps and answers membership
    like the source and the oracle, and all three stay equal over further pick + Add steps with evictions and a lowered
    capacity."""
    E = 64
    a = Aged(E=E, seed=7 + mode, mode=mode)
    blob = a.gpu.save_snapshot()
    bs = [a.loaded(blob, index_slots=1 << 15, table_slots=1 << 10), a.loaded(blob, table_slots=1 << 13)]
    for b in bs:
        assert b.save_snapshot().tobytes() == blob.tobytes()
        _same(b, a.ora, a.cs, E, "loaded")
        _picks(b, a.gpu, a.cs, E, "loaded vs source")
        assert np.array_equal(_contains(b, a.cs.hashes, E), _contains(a.gpu, a.cs.hashes, E))
        st = b.index_stats()
        assert st.tombstones == 0 and st.used == len(SR.read(blob).node_keys) - 2  # (the two marker keys have no slot)
        assert st.lru_entries == a.gpu.index_stats().lru_entries
    cs = a.cs
    for step in range(4):
        got = a.gpu.pick_batch(cs.tok, cs.offs, cs.h0)
        eps = got[:, 1]["endpoint"].copy()
        eps[eps == abi.FI_NO_ENDPOINT] = 0
        eps = (eps + step) % E
        nb = got[:, 1]["n_blocks"].astype(np.uint32) if step % 2 else cs.nb.copy()
        calls = [("chains", eps.astype(np.uint32), cs.chains.copy(), nb)] + \
                [c for c in cs.calls(E, n=4) if c[0] not in ("states", "lora")]
        if step == 2:
            e = max(range(E), key=lambda x: a.ora.lru_size(x))
            calls.append(("caps", np.array([e], np.uint32), np.array([a.cfg.max_blocks + 1], np.uint32)))
        for entry in calls:
            a.both(entry)
            for b in bs:
                RR.apply(b, entry)
        for b in bs:
            _same(b, a.ora, cs, E, f"step {step}")
        _same(a.gpu, a.ora, cs, E, f"step {step} (source)")
    for b in bs:
        b.close()
    a.close()


def test_shuffled_reference_blob_loads():
    """A blob the reference writer made from the oracle's state, in shuffled node order, loads and picks like the oracle.
    Its save keeps the blob's order of the regular keys (the load numbered them so); the marker keys 0 and ~0 have fixed
    nodes and come last."""
    E = 50
    a = Aged(E=E, seed=21)
    blob = SR.from_oracle(a.ora, np.random.default_rng(3))
    b = a.loaded(np.frombuffer(blob, np.uint8))
    _same(b, a.ora, a.cs, E, "shuffled blob")
    s = SR.read(blob)
    keys = s.node_keys.tolist()
    order = [i for i, k in enumerate(keys) if k not in (0, U64_MAX)] + [keys.index(m) for m in (0, U64_MAX) if m in keys]
    assert len(order) == len(keys) > 2
    want = SR.write(SR.Snapshot(**{**s.__dict__, "node_keys": s.node_keys[order], "node_rows": s.node_rows[order]}))
    assert b.save_snapshot().tobytes() == want
    b.close()
    a.close()


def _expect(rc_status, fn):
    with pytest.raises(FiEppError) as ei:
        fn()
    assert ei.value.status == rc_status, ei.value


def test_errors_change_nothing():
    E = 40
    a = Aged(E=E, seed=33)
    blob = a.gpu.save_snapshot()
    s = SR.read(blob)
    b = a.loaded(blob, index_slots=1 << 14)
    tok, offs, h0 = a.cs.tok, a.cs.offs, a.cs.h0
    ref = b.pick_batch(tok, offs, h0)
    ref_lru = [b.lru_dump(e) for e in range(E)]

    def unchanged(what):
        got = b.pick_batch(tok, offs, h0)
        assert H.picks_equal(got, ref), what + "\n" + H.describe_diff(got, ref)
        for e in range(E):
            assert np.array_equal(b.lru_dump(e), ref_lru[e]), (what, e)

    def patched(off, fmt, value):
        bad = bytearray(blob.tobytes())
        import struct
        struct.pack_into(fmt, bad, off, value)
        return SR.resealed(bytes(bad))

    other = ExtOracle(RR.config(E + 1))
    cases = [
        ("block_bytes", abi.FI_ERR_INVALID, patched(16, "<I", 64)),
        ("max_blocks", abi.FI_ERR_INVALID, patched(20, "<I", a.cfg.max_blocks + 1)),
        ("lru_capacity", abi.FI_ERR_INVALID, patched(24, "<I", a.cfg.lru_capacity + 8)),
        ("num_endpoints", abi.FI_ERR_INVALID, SR.from_oracle(other)),
    ]
    bad = bytearray(blob.tobytes())
    bad[-3] ^= 1
    cases.append(("checksum", abi.FI_ERR_INVALID, bytes(bad)))
    regular = [i for i, k in enumerate(s.node_keys.tolist()) if k not in (0, U64_MAX)]
    keys = s.node_keys.copy()
    keys[regular[-1]] = keys[regular[0]]  # a repeated node key: found on the device
    cases.append(("duplicate node key", abi.FI_ERR_INVALID, SR.write(SR.Snapshot(**{**s.__dict__, "node_keys": keys}))))
    e = max(range(E), key=lambda x: len(s.lrus[x]))
    lrus = [x.copy() for x in s.lrus]
    lrus[e][-1] = lrus[e][0]  # a repeated LRU key: found on the device
    cases.append(("duplicate LRU key", abi.FI_ERR_INVALID, SR.write(SR.Snapshot(**{**s.__dict__, "lrus": lrus}))))
    many = np.arange(1, 10001, dtype=np.uint64) << np.uint64(20)  # 10 000 keys: above 60 % of 1 << 14 slots
    rows = np.zeros((len(many), SR.row_words(E)), np.uint32)
    rows[:, 0] = 1
    cases.append(("pinned index_slots", abi.FI_ERR_CAPACITY,
                  SR.write(SR.Snapshot(**{**s.__dict__, "node_keys": many, "node_rows": rows}))))
    for what, status, data in cases:
        _expect(status, lambda: b.load_snapshot(np.frombuffer(data, np.uint8)))
        unchanged(what)
    other.close()
    # the size query and a buffer too small
    lib, n = abi.load(), C.c_uint64(0)
    assert lib.fi_epp_snapshot_save(b._h, None, 0, C.byref(n)) == abi.FI_OK and n.value == len(blob)
    small = np.full(len(blob) - 1, 0xAB, np.uint8)
    n.value = 0
    assert lib.fi_epp_snapshot_save(b._h, small.ctypes.data_as(C.c_void_p), len(small), C.byref(n)) == abi.FI_ERR_CAPACITY
    assert n.value == len(blob) and (small == 0xAB).all()
    unchanged("too small a buffer")
    # a handle the host LRU serves: neither call
    h = _handle(a.cfg, host_lru=True)
    h.index_add_chains(np.array([0], np.uint32), a.cs.chains[:1].copy(), a.cs.nb[:1].copy())
    _expect(abi.FI_ERR_STATE, h.save_snapshot)
    _expect(abi.FI_ERR_STATE, lambda: h.load_snapshot(blob))
    h.close()
    b.close()
    a.close()


def _device(cs, R):
    import torch

    d_tok = torch.from_numpy(np.ascontiguousarray(cs.tok).view(np.uint8).copy()).cuda()
    d_off = torch.from_numpy(cs.offs[: R + 1].copy().view(np.int64)).cuda()
    d_h0 = torch.full((R,), cs.h0, dtype=torch.int64, device="cuda")
    return d_tok, d_off, d_h0


def test_load_is_ordered_against_submitted_batches_and_tickets():
    """Batch A submitted before the load picks on the old state, batch B after it on the loaded one;
    index_add_submitted of A's ticket then adds A's chains to the loaded state."""
    import torch

    E = 48
    old, new = Aged(E=E, seed=41), Aged(E=E, seed=42)
    blob = new.gpu.save_snapshot()
    cs = new.cs
    R, P = cs.R, old.cfg.n_profiles
    d_tok, d_off, d_h0 = _device(cs, R)
    s = torch.cuda.current_stream().cuda_stream
    out_a = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    out_b = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    want_a = old.ora.pick_batch(cs.tok, cs.offs, cs.h0)
    old.ora.load_state(*new.ora.state())  # the oracle's load: the handle keeps its own endpoint states and adapters
    want_b = old.ora.pick_batch(cs.tok, cs.offs, cs.h0)
    ta = old.gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out_a.data_ptr(), stream=s)
    old.gpu.load_snapshot(blob)
    tb = old.gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out_b.data_ptr(), stream=s)
    old.gpu.pick_wait_batch(tb, s)
    torch.cuda.synchronize()
    got_a = out_a.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
    got_b = out_b.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
    assert H.picks_equal(got_a, want_a), "A (before the load)\n" + H.describe_diff(got_a, want_a)
    assert H.picks_equal(got_b, want_b), "B (after the load)\n" + H.describe_diff(got_b, want_b)
    eps = cs.rng.integers(0, E, size=R).astype(np.uint32)
    nb = want_a[:, 0]["n_blocks"].astype(np.uint32)
    old.gpu.index_add_submitted(ta, eps, nb)
    old.ora.index_add_chains(eps, cs.chains, nb)
    _same(old.gpu, old.ora, cs, E, "after index_add_submitted of the earlier ticket")
    old.close()
    new.close()


def test_load_before_the_first_add():
    E = 40
    a = Aged(E=E, seed=51)
    blob = a.gpu.save_snapshot()
    b = EndpointPicker(a.cfg)  # no Add yet: the load allocates the device LRU
    for entry in a.hist:
        RR.apply(b, entry)
    b.load_snapshot(blob)
    _same(b, a.ora, a.cs, E, "loaded before any Add")
    entry = ("chains", a.cs.rng.integers(0, E, size=a.cs.R).astype(np.uint32), a.cs.chains.copy(), a.cs.nb.copy())
    a.both(entry)
    RR.apply(b, entry)
    _same(b, a.ora, a.cs, E, "then an Add")
    b.close()
    a.close()


def test_empty_and_lru_free_handles_round_trip():
    cfg = RR.config(9)
    e1, e2 = EndpointPicker(cfg), EndpointPicker(cfg)
    blob = e1.save_snapshot()
    info = snapshot_info(blob)
    assert (info.n_nodes, info.n_lru, info.pairs) == (0, 0, 0)
    assert SR.read(blob).caps.tolist() == [cfg.lru_capacity] * 9
    e2.load_snapshot(blob)
    assert e2.save_snapshot().tobytes() == blob.tobytes()
    e1.close()
    e2.close()
    E = 30
    a = Aged(E=E, seed=61, lru_capacity=0)
    blob = a.gpu.save_snapshot()
    s = SR.read(blob)
    assert s.lru_capacity == 0 and not s.caps.any() and not any(len(x) for x in s.lrus)
    assert s.pairs() == a.ora.index_pairs()
    b = a.loaded(blob)
    _same(b, a.ora, a.cs, E, "no LRU", lru=False)
    assert b.save_snapshot().tobytes() == blob.tobytes()
    b.close()
    a.close()


def test_full_size_cfg3_round_trip():
    """cfg 3 (1 024 endpoints, lruCapacityPerServer 31 250, device LRU), aged by pick + Add steps: save, load into a
    handle with a smaller LRU table, save again (the same bytes), and a 768-request sample picks bit-equal on both."""
    wl = synth.baseline_workload(3)
    profiles, pd = synth.baseline_profiles(3)
    R = wl.R
    cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=wl.lru_capacity,
                      max_batch=R, max_prompt_bytes=R * wl.T * 4, profiles=profiles, pd=pd)
    main_p = pd["decode"] if pd else 0
    a = EndpointPicker(cfg)
    a.set_option("device_lru", 1)
    states = wl.endpoint_states()
    a.update_endpoints(states)
    for k in range(4):
        tok, offs = wl.prompts(batch=300 + k)
        got, chains = a.pick_batch(tok, offs, wl.h0, want_chains=True)
        a.index_add_chains(got[:, main_p]["endpoint"].copy(), chains, got[:, main_p]["n_blocks"].astype(np.uint32))
    blob = a.save_snapshot()
    info = snapshot_info(blob)
    assert info.n_lru == a.index_stats().lru_entries and info.n_nodes > 100_000
    b = EndpointPicker(cfg)
    b.set_option("lru_table_slots", 1 << 17)
    b.update_endpoints(states)
    b.load_snapshot(blob)
    again = b.save_snapshot()
    assert again.tobytes() == blob.tobytes()
    del again
    tok, offs = wl.prompts(batch=300)
    n = 768
    offs = offs[: n + 1].copy()
    tok = tok.reshape(-1).view(np.uint8)[: int(offs[n])].copy()
    got_a = a.pick_batch(tok, offs, wl.h0)
    got_b = b.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got_a, got_b), H.describe_diff(got_a, got_b)
    assert (got_a[:, main_p]["match_blocks"] > 0).any()
    a.close()
    b.close()
