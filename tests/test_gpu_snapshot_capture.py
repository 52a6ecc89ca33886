"""GPU (-m gpu): snapshot captures (fi_epp_snapshot_capture / _read / _free, docs/SPEC.md S.2d).

A capture is the save taken on the device at a point of the handle's call order and copied out later without the
handle.  Its blob must be byte for byte the save's at that point, hold every call issued before it and none issued
after, not wait for picks in flight, survive every later call on the handle (destroy included), and load like a saved
blob.  The blobs are read with the independent reader of tests/snapshot_ref.py and held to the snapshot oracle.
"""
import ctypes as C
import queue
import threading

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, snapshot_info
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import craft
from tests import helpers as H
from tests import resize_ref as RR
from tests import snapshot_ref as SR
from tests.snapshot_oracle import SnapshotOracle
from tests.test_gpu_snapshot import Aged, _device, _handle, _same
from tests.test_gpu_stream_order import Rig, _device_call, _eq, _held, _want

pytestmark = pytest.mark.gpu
U64_MAX = 0xFFFFFFFFFFFFFFFF


def _state_of(blob, ora, what):
    """the blob passes snapshot_info and the independent reader, and holds the oracle's state"""
    s = SR.read(blob)
    info = snapshot_info(blob)
    assert info.bytes == len(blob) and info.n_nodes == len(s.node_keys), what
    pairs, lrus, caps = ora.state()
    assert s.pairs() == pairs, what
    assert s.caps.tolist() == caps, what
    for e in range(len(caps)):
        assert np.array_equal(s.lrus[e], lrus[e]), (what, e)


def _captured(gpu):
    with gpu.capture_snapshot() as c:
        blob = c.read()
        assert c.nbytes == len(blob)
        return blob


class Small:
    """a handle and the oracle after a random call history on E endpoints (any E >= 1), the marker keys 0 and ~0 SET
    for endpoint 0 in the index and Added to endpoint 0's LRU"""

    def __init__(self, E, seed, lru_capacity=48, index_slots=0, n=12, add=True):
        self.E = E
        self.cfg = RR.config(E, lru_capacity=lru_capacity, index_slots=index_slots)
        self.cs = RR.CallStream(seed, RR.config(E))
        self.gpu, self.ora = EndpointPicker(self.cfg), SnapshotOracle(self.cfg, track_removal=True)
        self.both(("states", H.states_array(E, roles=abi.FI_ROLE_WORKER | RR.LABEL)))
        calls = self.cs.calls(E, n=n)
        if not (lru_capacity and add):
            calls = [c for c in calls if c[0] in ("states", "lora", "ops")]
        for entry in calls:
            self.both(entry)
        zero, ones = craft.MARKERS
        self.both(("ops", H.ops_array([(zero, 0, abi.FI_OP_SET), (ones, 0, abi.FI_OP_SET)])))
        if lru_capacity and add:
            B = self.cfg.block_bytes
            blocks = [self.cs.rng.integers(0, 256, size=B, dtype=np.uint8).tobytes() for _ in range(3)]
            tok, offs = H.pack_prompts([b"".join(blocks)])
            for target in craft.MARKERS:
                chains, nb = self.ora.hash_batch(tok, offs, craft.h0_for(blocks, 1, target))
                self.both(("chains", np.array([0], np.uint32), chains, nb.astype(np.uint32)))

    def both(self, entry):
        RR.apply(self.gpu, entry)
        RR.apply(self.ora, entry)

    def close(self):
        self.gpu.close()
        self.ora.close()


def _same_bytes(gpu, ora, what):
    saved = gpu.save_snapshot()
    blob = _captured(gpu)
    assert blob.tobytes() == saved.tobytes(), what
    _state_of(blob, ora, what)
    return blob


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("E", [31, 32, 33, 40])
def test_capture_equals_save(E, mode):
    """aged handles (markers in the index and the LRUs, a lowered capacity, a removal) in both match modes"""
    a = Aged(E=E, seed=E + 100 * mode, mode=mode)
    assert {(1, 0), (2, U64_MAX)} <= a.ora.index_pairs()
    _same_bytes(a.gpu, a.ora, f"E={E} mode={mode}")
    a.close()


@pytest.mark.parametrize("E", [1, 31, 32, 33])
def test_capture_equals_save_small_pools(E):
    a = Small(E, seed=E)
    assert (0, 0) in a.ora.index_pairs() and len(a.ora.lru(0)) > 0
    _same_bytes(a.gpu, a.ora, f"E={E}")
    a.close()


def test_capture_without_lru_before_add_and_empty():
    a = Aged(E=30, seed=61, lru_capacity=0)
    _same_bytes(a.gpu, a.ora, "lru_capacity 0")
    a.close()
    b = Small(20, seed=5, add=False)  # SETs but no Add: no device LRU yet
    _same_bytes(b.gpu, b.ora, "before the first Add")
    b.close()
    cfg = RR.config(9)
    e, ora = EndpointPicker(cfg), SnapshotOracle(cfg)
    blob = _same_bytes(e, ora, "empty handle")
    info = snapshot_info(blob)
    assert (info.n_nodes, info.n_lru, info.pairs) == (0, 0, 0)
    e.close()
    ora.close()


def test_later_calls_are_not_in_the_capture():
    """after the capture: direct SET / CLEAR ops, a stream-ordered Add, add_submitted of an earlier ticket, a removal, a
    capacity shrink, index rebuilds, a resize, a load and destroy; the read still gives the save taken before it"""
    import torch

    E = 40
    a = Small(E, seed=71, index_slots=1 << 13)
    cs, g = a.cs, a.gpu
    R, P = cs.R, a.cfg.n_profiles
    d_tok, d_off, d_h0 = _device(cs, R)
    out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    ticket = g.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out.data_ptr(), stream=s)
    g.pick_wait_batch(ticket, s)
    torch.cuda.synchronize()
    want = g.save_snapshot()
    c = g.capture_snapshot()
    rebuilds = g.index_stats().rebuilds
    g.index_apply(H.ops_array([(int(h), 3, abi.FI_OP_SET) for h in cs.hashes[:20]] +
                              [(int(h), 5, abi.FI_OP_CLEAR) for h in cs.hashes[:20]]))
    d_chains = torch.from_numpy(cs.chains.view(np.int64).copy()).cuda()
    eps = (np.arange(R) % E).astype(np.uint32)
    g.index_add_chains_device(eps, d_chains.data_ptr(), cs.chains.shape[1], cs.nb.copy(), s)
    g.index_add_submitted(ticket, (eps + 1) % E, cs.nb.copy())
    g.remove_endpoints([4, 9])
    e = max(range(E), key=lambda x: len(g.lru_dump(x)))
    g.set_lru_capacities([e], [a.cfg.max_blocks])
    rng = np.random.default_rng(3)
    for _ in range(6):  # churn of fresh keys SET then CLEARed: tombstones until the index rebuilds
        keys = rng.integers(1, 2**63, size=1500, dtype=np.uint64)
        g.index_apply(H.ops_array([(int(k), 1, abi.FI_OP_SET) for k in keys]))
        g.index_apply(H.ops_array([(int(k), 1, abi.FI_OP_CLEAR) for k in keys]))
        g.index_sync()
    assert g.index_stats().rebuilds > rebuilds
    g.resize_pool(E + 8)
    other = EndpointPicker(RR.config(E + 8, index_slots=1 << 13))
    g.load_snapshot(other.save_snapshot())
    other.close()
    assert c.read().tobytes() == want.tobytes()
    g.close()
    assert c.read().tobytes() == want.tobytes()
    c.close()
    a.ora.close()


def test_calls_before_the_capture_are_in_it():
    """staged ops not yet flushed, a removal, a raised capacity and add_submitted of a ticket still in flight, all
    issued before the capture"""
    import torch

    E = 40
    a = Small(E, seed=81)
    cs, g, ora = a.cs, a.gpu, a.ora
    R, P = cs.R, a.cfg.n_profiles
    d_tok, d_off, d_h0 = _device(cs, R)
    out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    want_picks = ora.pick_batch(cs.tok, cs.offs, cs.h0)
    low = [2, 3]
    for x in (g, ora):
        x.set_lru_capacities(low, [a.cfg.max_blocks] * 2)  # (lowering blocks; the raise below does not)
    ticket = g.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out.data_ptr(), stream=s)
    eps = cs.rng.integers(0, E, size=R).astype(np.uint32)
    nb = want_picks[:, 0]["n_blocks"].astype(np.uint32)
    g.index_add_submitted(ticket, eps, nb)
    ora.index_add_chains(eps, cs.chains, nb)
    ops = H.ops_array([(int(h), 11, abi.FI_OP_SET) for h in cs.hashes[:30]] + [(int(cs.hashes[40]), 12, abi.FI_OP_SET)])
    for entry in [("ops", ops), ("caps", np.array(low, np.uint32), np.array([a.cfg.lru_capacity] * 2, np.uint32))]:
        a.both(entry)
    for x in (g, ora):
        x.remove_endpoints([7])
    c = g.capture_snapshot()
    blob = c.read()
    c.close()
    g.pick_wait_batch(ticket, s)
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
    assert H.picks_equal(got, want_picks), H.describe_diff(got, want_picks)
    _state_of(blob, ora, "calls before the capture")
    assert blob.tobytes() == g.save_snapshot().tobytes()
    a.close()


def test_capture_does_not_wait_for_picks():
    """a device pick and a pick_submit_ex batch held behind a spin on the caller's stream: the capture returns while
    their inputs are still in flight, the picks match the oracle, the blob equals a later save"""
    import torch

    rig = Rig(64)
    g, s = rig.gpu, torch.cuda.Stream()
    rig.decoy()
    _device_call(rig, "device", s)  # warm-up (flushes the staged ops of the rig's history)
    s.synchronize()
    _captured(g)
    for case in ("device", "submit_ex"):
        rig.decoy()
        e_in = rig.late(s)
        if case == "device":
            _device_call(rig, "device", s)
        else:
            p = rig.ptrs()
            t = g.pick_submit_ex(p[0], p[1], p[2], len(rig.h0), rig.tok.nbytes, rig.out.data_ptr(), stream=s.cuda_stream)
        c = g.capture_snapshot()
        _held(e_in, f"the capture ({case})")
        if case != "device":
            g.pick_wait_batch(t, s.cuda_stream)
        got, _ = rig.snapshot(s)
        _eq(got, _want(rig, "device"), f"{case} pick held across a capture")
        assert c.read().tobytes() == g.save_snapshot().tobytes(), case
        c.close()
    rig.close()


def test_reads_on_another_thread():
    """one thread runs pick + Add steps (bit-exact against the oracle) and takes captures at known steps; another
    reads and frees them, each blob holding the oracle's state of its step"""
    E = 48
    a = Aged(E=E, seed=91)
    cs = a.cs
    todo, errors, done = queue.Queue(), [], []

    def reader():
        while True:
            item = todo.get()
            if item is None:
                return
            step, c, state = item
            try:
                blob = c.read()
                c.close()
                s = SR.read(blob)
                pairs, lrus, caps = state
                assert s.pairs() == pairs and s.caps.tolist() == caps, step
                for e in range(E):
                    assert np.array_equal(s.lrus[e], lrus[e]), (step, e)
                done.append(step)
            except Exception as ex:  # pragma: no cover
                errors.append((step, repr(ex)))

    th = threading.Thread(target=reader)
    th.start()
    for step in range(8):
        got = a.gpu.pick_batch(cs.tok, cs.offs, cs.h0)
        want = a.ora.pick_batch(cs.tok, cs.offs, cs.h0)
        assert H.picks_equal(got, want), f"step {step}\n" + H.describe_diff(got, want)
        eps = got[:, 0]["endpoint"].copy()
        eps[eps == abi.FI_NO_ENDPOINT] = 0
        eps = ((eps + step) % E).astype(np.uint32)
        a.both(("chains", eps, cs.chains.copy(), got[:, 0]["n_blocks"].astype(np.uint32)))
        if step % 2:
            todo.put((step, a.gpu.capture_snapshot(), a.ora.state()))
    todo.put(None)
    th.join(timeout=600)
    assert not errors, errors
    assert done == [1, 3, 5, 7]
    a.close()


def test_capture_lifetimes():
    E = 40
    a = Aged(E=E, seed=101)
    g = a.gpu
    a.gpu.capture_snapshot().close()  # freed at once, its export still running
    g.capture_snapshot().close()      # and never read
    blobs, caps = [], []
    for k in range(3):  # three outstanding captures, each of its own point
        blobs.append(g.save_snapshot())
        caps.append(g.capture_snapshot())
        fresh = np.random.default_rng(k).integers(1, 2**63, size=(2, a.cfg.max_blocks), dtype=np.uint64)
        a.both(("chains", np.array([k, k + 1], np.uint32), fresh, np.array([4, 4], np.uint32)))
    assert len({b.tobytes() for b in blobs}) == 3
    first = caps[0].read()
    assert first.tobytes() == caps[0].read().tobytes() == blobs[0].tobytes()
    g.close()
    for c, b in zip(caps, blobs):
        assert c.read().tobytes() == b.tobytes()  # after destroy
        c.close()
    lib = abi.load()
    lib.fi_epp_snapshot_free(None)
    a.ora.close()


def test_captured_blob_loads_and_continues():
    E = 64
    a = Aged(E=E, seed=111)
    blob = _captured(a.gpu)
    b = a.loaded(blob, table_slots=1 << 10)
    assert b.save_snapshot().tobytes() == blob.tobytes()
    _same(b, a.ora, a.cs, E, "loaded from a capture")
    cs = a.cs
    for step in range(3):
        got = a.gpu.pick_batch(cs.tok, cs.offs, cs.h0)
        eps = got[:, 0]["endpoint"].copy()
        eps[eps == abi.FI_NO_ENDPOINT] = 0
        entry = ("chains", ((eps + step) % E).astype(np.uint32), cs.chains.copy(), got[:, 0]["n_blocks"].astype(np.uint32))
        a.both(entry)
        RR.apply(b, entry)
        _same(b, a.ora, cs, E, f"step {step}")
    b.close()
    a.close()


def _expect(status, fn):
    with pytest.raises(FiEppError) as ei:
        fn()
    assert ei.value.status == status, ei.value


def test_capture_errors():
    E = 40
    a = Aged(E=E, seed=121)
    g, lib = a.gpu, abi.load()
    out, n = C.c_void_p(), C.c_uint64(0)
    assert lib.fi_epp_snapshot_capture(None, C.byref(out), C.byref(n)) == abi.FI_ERR_INVALID
    assert lib.fi_epp_snapshot_capture(g._h, None, C.byref(n)) == abi.FI_ERR_INVALID
    assert lib.fi_epp_snapshot_capture(g._h, C.byref(out), None) == abi.FI_ERR_INVALID
    assert not out.value
    assert lib.fi_epp_snapshot_read(None, None, 0) == abi.FI_ERR_INVALID
    with g.capture_snapshot() as c:
        assert lib.fi_epp_snapshot_read(c._c, None, c.nbytes) == abi.FI_ERR_INVALID
        small = np.full(c.nbytes - 1, 0xAB, np.uint8)
        assert lib.fi_epp_snapshot_read(c._c, small.ctypes.data_as(C.c_void_p), len(small)) == abi.FI_ERR_CAPACITY
        assert (small == 0xAB).all()
        assert c.read().tobytes() == g.save_snapshot().tobytes()
    tok, offs, h0 = a.cs.tok, a.cs.offs, a.cs.h0
    for what, cfg, host in [("part of the pool", None, False), ("host LRU", a.cfg, True)]:
        if cfg is None:
            cfg = abi.fi_epp_config.from_buffer_copy(a.cfg)
            cfg.endpoint_begin, cfg.endpoint_count = 8, E - 8
        h = _handle(cfg, host_lru=host)
        h.update_endpoints(H.states_array(E, roles=abi.FI_ROLE_WORKER | RR.LABEL))
        h.index_add_chains(np.array([10], np.uint32), a.cs.chains[:1].copy(), a.cs.nb[:1].copy())
        before = h.pick_batch(tok, offs, h0)
        out.value = None
        assert lib.fi_epp_snapshot_capture(h._h, C.byref(out), C.byref(n)) == abi.FI_ERR_STATE, what
        assert not out.value, what
        _expect(abi.FI_ERR_STATE, h.capture_snapshot)
        got = h.pick_batch(tok, offs, h0)
        assert H.picks_equal(got, before), what
        h.close()
    a.close()


def test_capture_statistics():
    a = Aged(E=40, seed=131)
    g = a.gpu
    g.index_sync()
    st0, ix0 = g.stats(), g.index_stats()
    c = g.capture_snapshot()
    st1, ix1 = g.stats(), g.index_stats()
    assert st1.kernel_launches - st0.kernel_launches == 3  # the tile count, the LRU dump, the node export
    for f, _ in abi.fi_index_stats._fields_:
        assert getattr(ix1, f) == getattr(ix0, f), f
    c.read()
    assert g.stats().kernel_launches == st1.kernel_launches
    c.close()
    a.close()
