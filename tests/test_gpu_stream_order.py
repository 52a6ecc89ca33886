"""GPU (-m gpu): the device entry points against work still running on the caller's stream.

Every other device-path test writes its inputs, synchronises the device and only then calls.  Here the inputs first
hold a decoy batch (all-zero offsets: every request has n_blocks = 0, so every row of its picks differs from the real
batch's), the outputs hold 0xFF bytes, and then, on the caller's stream: a spin of SLEEP_CYCLES, device-to-device
copies of the real inputs, the call, and copies of the outputs into snapshots.  A call that did not order its work
after the caller's stream reads the decoy; one that did not make the stream wait for its result leaves 0xFF or the
decoy's picks in the snapshot.  Each case checks that the real inputs were still in flight when the call returned
(else it fails with "sleep too short"), and compares with the CPU oracle on the real batch.

Also: index updates issued while an earlier device pick is held behind the spin are not seen by it and are seen by
the next pick (docs/SPEC.md S.2a, S.2b, S.9), and an index_apply issued before a pick whose stream is still spinning
is seen by the early-exit hashing of that pick.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.ext_oracle import ExtOracle
from tests.test_gpu_ranked import _lora, _states

pytestmark = pytest.mark.gpu
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
PROFILES = [{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5), (Q, 5)]}]
# ~57 ms at the H100 SXM's 1755 MHz boost clock: far longer than the host needs to enqueue the copies and make the
# call, so the real inputs are still in flight when a non-blocking call returns
SLEEP_CYCLES = 100_000_000
E, R, MB, CAP, KR = 48, 64, 32, 64, 4


def _torch():
    import torch

    return torch


def _dev(a, dtype=np.int64):
    return _torch().from_numpy(np.ascontiguousarray(a).view(dtype).ravel().copy()).cuda()


def _picks(t, k=0):
    return t.cpu().numpy().view(H.PICK_DTYPE).reshape((R, 1, k) if k else (R, 1))


def _eq(got, want, what):
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)


def _held(e_in, what):
    assert not e_in.query(), f"sleep too short: the inputs of {what} had landed when it returned"


class Rig:
    """One handle and its oracle in the same state, the real batch on the device, and input buffers holding the decoy."""

    def __init__(self, block_bytes, lru_capacity=CAP, seed=0):
        torch = _torch()
        rng = np.random.default_rng(block_bytes + seed)
        self.wl = wl = H.small_workload(E=E, R=R, T=600, max_blocks=MB, block_tokens=block_bytes // 4, holes=True,
                                        lru_capacity=CAP)
        cfg = H.config_for(wl, profiles=PROFILES, lru_capacity=lru_capacity, max_prompt_bytes=R * wl.T * 4)
        self.gpu, self.cpu = EndpointPicker(cfg), ExtOracle(cfg, track_removal=True)
        st, lo = _states(wl, rng, roles=False), _lora(E, rng)
        for g in (self.gpu, self.cpu):
            g.update_endpoints(st)
            g.update_endpoints_lora(lo)
            for ops in wl.index_ops():
                g.index_apply(ops)
        self.tok, self.offs = wl.prompts(batch=1)
        self.h0 = np.full(R, wl.h0, dtype=np.uint64)
        self.ad = (rng.integers(0, 14, R) + 1000).astype(np.uint64)
        self.sub = subset_bitsets([rng.choice(E, [1, 8, E // 2, E][r % 4], replace=False).tolist() for r in range(R)], E)
        self.chains, self.nb = self.cpu.hash_batch(self.tok, self.offs, self.h0)
        assert (self.nb > 0).all()  # the decoy's n_blocks = 0 differs in every row
        # the real inputs, and the buffers the calls read (filled with the decoy by decoy())
        self.src = [_dev(self.tok, np.int32), _dev(self.offs), _dev(self.h0), _dev(self.ad), _dev(self.sub, np.int32)]
        self.buf = [torch.empty_like(t) for t in self.src]
        self.out = torch.empty(R * KR * 16, dtype=torch.uint8, device="cuda")
        self.ch = torch.empty(R * MB, dtype=torch.int64, device="cuda")
        self.rng = rng

    def ptrs(self):
        return [b.data_ptr() for b in self.buf]

    def decoy(self):
        """decoy inputs (no blocks, other seeds, no adapters, empty subsets), 0xFF outputs, one device-wide sync"""
        torch = _torch()
        for b in self.buf:
            b.zero_()
        self.out.fill_(0xFF)
        self.ch.fill_(-1)
        torch.cuda.synchronize()

    def late(self, s, extra=()):
        """on stream s: spin, then copy the real inputs in; -> the event recorded after the copies"""
        torch = _torch()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            for d, src in list(zip(self.buf, self.src)) + list(extra):
                d.copy_(src)
            e = torch.cuda.Event()
            e.record(s)
        return e

    def snapshot(self, s, k=0):
        """copy the outputs on s and wait for s only"""
        torch = _torch()
        with torch.cuda.stream(s):
            out, ch = self.out.clone(), self.ch.clone()
        s.synchronize()
        n = R * max(k, 1) * 16
        return _picks(out[:n], k), ch.cpu().numpy().view(np.uint64).reshape(R, MB)

    def check_chains(self, got, what):
        for r in range(R):
            assert np.array_equal(got[r, : self.nb[r]], self.chains[r, : self.nb[r]]), f"{what}: chain of request {r}"

    def close(self):
        self.gpu.close()
        self.cpu.close()


def _stream(kind):
    torch = _torch()
    return torch.cuda.default_stream() if kind == "legacy" else torch.cuda.Stream()


def _device_call(rig, kind, s):
    """one stream-ordered device pick of the given kind on stream s; -> k"""
    g, p, ss = rig.gpu, rig.ptrs(), s.cuda_stream
    nbytes = rig.tok.nbytes
    if kind == "device":
        g.pick_batch_device(p[0], p[1], p[2], R, nbytes, rig.out.data_ptr(), rig.ch.data_ptr(), ss)
        return 0
    if kind == "lora":
        rc = abi.load().fi_epp_pick_batch_device_lora(g._h, p[0], p[1], p[2], p[3], R, nbytes, rig.out.data_ptr(),
                                                       rig.ch.data_ptr(), ss or None)
        g._check(rc, "fi_epp_pick_batch_device_lora")
        return 0
    if kind == "ranked":
        g.pick_batch_device_ranked(p[0], p[1], p[2], R, nbytes, KR, rig.out.data_ptr(), rig.ch.data_ptr(), ss, p[3])
        return KR
    g.pick_batch_device_subset(p[0], p[1], p[2], R, nbytes, KR, rig.out.data_ptr(), p[4], rig.ch.data_ptr(), ss, p[3])
    return KR


def _want(rig, kind):
    c, a = rig.cpu, (rig.tok, rig.offs, rig.h0)
    if kind == "device":
        return c.pick_batch(*a)
    if kind == "lora":
        return c.pick_batch(*a, adapters=rig.ad)
    if kind == "ranked":
        return c.pick_batch_ranked(*a, KR, adapters=rig.ad)
    return c.pick_batch_subset(*a, rig.sub, KR, adapters=rig.ad)


KINDS = ["device", "lora", "ranked", "subset"]
BLOCK_BYTES = [64, 40]  # 40: pick_submit(_ex) takes its stream-ordered fallback


@pytest.mark.parametrize("stream", ["side", "legacy"])
@pytest.mark.parametrize("block_bytes", BLOCK_BYTES)
def test_device_picks_wait_for_late_inputs(block_bytes, stream):
    """pick_batch_device, _lora, _ranked and _subset with prompts, offsets, seeds, adapters and subsets written on the
    caller's stream behind a spin; picks and chains_out read back on that stream"""
    rig = Rig(block_bytes)
    s = _stream(stream)
    for kind in KINDS:  # warm-up: lazy buffers and the endpoint / adapter uploads stay out of the calls below
        rig.decoy()
        _device_call(rig, kind, s)
        s.synchronize()
    for kind in KINDS:
        rig.decoy()
        e_in = rig.late(s)
        k = _device_call(rig, kind, s)
        _held(e_in, kind)
        got, ch = rig.snapshot(s, k)
        _eq(got, _want(rig, kind), f"{kind} pick on the {stream} stream")
        rig.check_chains(ch, kind)
    rig.close()


@pytest.mark.parametrize("block_bytes", BLOCK_BYTES)
def test_submits_wait_for_late_inputs(block_bytes):
    """pick_submit and pick_submit_ex (k = 0 with adapters, k = 4 with subsets) whose inputs land on the caller's stream
    behind a spin; pick_wait / pick_wait_batch on a second stream, which then reads d_out"""
    torch = _torch()
    rig = Rig(block_bytes)
    g, s, s2 = rig.gpu, torch.cuda.Stream(), torch.cuda.Stream()
    nbytes = rig.tok.nbytes

    def submit(case):
        p = rig.ptrs()
        if case == "submit":
            g.pick_submit(p[0], p[1], p[2], R, nbytes, rig.out.data_ptr(), s.cuda_stream)
            return None, 0
        k = 0 if case == "ex0" else KR
        t = g.pick_submit_ex(p[0], p[1], p[2], R, nbytes, rig.out.data_ptr(), k=k, d_adapters=p[3],
                             d_subsets=p[4] if k else 0, d_chains=rig.ch.data_ptr(), stream=s.cuda_stream)
        return t, k

    def wait(t):
        if t is None:
            g.pick_wait(s2.cuda_stream)
        else:
            g.pick_wait_batch(t, s2.cuda_stream)

    cases = {"submit": rig.cpu.pick_batch(rig.tok, rig.offs, rig.h0),
             "ex0": _want(rig, "lora"), "ex4": _want(rig, "subset")}
    for case in cases:  # warm-up
        rig.decoy()
        wait(submit(case)[0])
        torch.cuda.synchronize()
    for case, want in cases.items():
        rig.decoy()
        e_in = rig.late(s)
        t, k = submit(case)
        _held(e_in, case)
        wait(t)
        got, ch = rig.snapshot(s2, k)
        _eq(got, want, f"{case}, read on the waiting stream")
        if case != "submit":
            rig.check_chains(ch, case)
        torch.cuda.synchronize()
    rig.close()


@pytest.mark.parametrize("block_bytes", BLOCK_BYTES)
def test_add_chains_device_waits_for_late_chains(block_bytes):
    """index_add_chains_device with explicit chains written on the caller's stream behind a spin, over decoy chains of
    other keys: the index and the LRUs hold the real chains, none of the decoy's"""
    torch = _torch()
    rig = Rig(block_bytes)
    g, c, s = rig.gpu, rig.cpu, torch.cuda.Stream()
    eps = (np.arange(R) % 6 * 7).astype(np.uint32)  # 6 endpoints, ~11 requests each: evictions at capacity 64
    decoy = rig.rng.integers(1, 2**63, (R, MB), dtype=np.int64)
    d_chains = _dev(decoy)
    real = _dev(rig.chains)
    warm = _dev(decoy[:1])
    g.index_add_chains_device(eps[:1], warm.data_ptr(), MB, rig.nb[:1], s.cuda_stream)  # warm-up
    c.index_add_chains(eps[:1], decoy[:1].view(np.uint64), rig.nb[:1])
    torch.cuda.synchronize()
    rig.decoy()
    e_in = rig.late(s, [(d_chains, real)])
    _held(e_in, "the call to index_add_chains_device")  # (it may block for its overflow readback)
    g.index_add_chains_device(eps, d_chains.data_ptr(), MB, rig.nb, s.cuda_stream)
    c.index_add_chains(eps, rig.chains, rig.nb)
    torch.cuda.synchronize()
    q = H.ops_array([(int(ch[r, j]), int(eps[r]), abi.FI_OP_SET) for ch in (rig.chains, decoy.view(np.uint64))
                     for r in range(R) for j in range(int(rig.nb[r]))])
    want = np.array([c.index_contains(int(o["endpoint"]), int(o["hash"])) for o in q], dtype=np.uint8)
    assert np.array_equal(g.index_contains(q), want)
    assert want[: len(q) // 2].any()
    for e in sorted(set(eps.tolist())):
        assert np.array_equal(g.lru_dump(e), c.lru(e)), f"LRU of endpoint {e}"
    rig.close()


@pytest.mark.parametrize("block_bytes", BLOCK_BYTES)
def test_updates_do_not_reach_a_held_pick(block_bytes):
    """index_apply, remove_endpoints, a raising set_lru_capacities, index_add_chains, update_endpoints(_lora) and a
    resize_pool, all issued while a device pick is held behind the spin: the held pick returns the oracle's picks from
    before the updates, a pick issued after them sees them"""
    torch = _torch()
    rig = Rig(block_bytes)
    g, c, s = rig.gpu, rig.cpu, torch.cuda.Stream()
    low = [5, 11, 17]
    for x in (g, c):  # lowered before the hold (a lowering call blocks), raised during it
        x.set_lru_capacities(low, [MB] * len(low))
    want_before = _want(rig, "subset")
    plain_before = c.pick_batch(rig.tok, rig.offs, rig.h0, adapters=rig.ad)
    for kind in KINDS:
        rig.decoy()
        _device_call(rig, kind, s)
    rig.decoy()
    e_in = rig.late(s)
    _device_call(rig, "subset", s)
    _held(e_in, "the held pick")
    # the updates: each one changes the real batch's picks
    rows = range(0, R, 2)
    ops = H.ops_array([(int(rig.chains[r, j]), (r * 5) % E, abi.FI_OP_SET) for r in rows for j in range(int(rig.nb[r]))]
                      + [(int(rig.chains[r, 0]), e, abi.FI_OP_CLEAR) for r in range(1, R, 4) for e in range(0, E, 3)])
    st = _states(rig.wl, rig.rng, roles=False)
    lo = _lora(E, rig.rng)
    eps = np.array([low[r % 3] for r in range(R)], dtype=np.uint32)
    updates = [lambda x: x.index_apply(ops), lambda x: x.remove_endpoints([2, 30, 47]),
               lambda x: x.set_lru_capacities(low, [CAP] * len(low)),
               lambda x: x.index_add_chains(eps, rig.chains, rig.nb),
               lambda x: x.update_endpoints(st), lambda x: x.update_endpoints_lora(lo)]
    for u in updates:
        u(g)
    g.resize_pool(E + 8)  # blocks until the held pick is done
    got, _ = rig.snapshot(s, KR)
    _eq(got, want_before, "the held pick")
    for u in updates:
        u(c)
    c.resize(E + 8)
    sub = subset_bitsets([rig.rng.choice(E + 8, 8, replace=False).tolist() for _ in range(R)], E + 8)
    after = g.pick_batch_subset(rig.tok, rig.offs, rig.h0, sub, KR, adapters=rig.ad)
    want_after = c.pick_batch_subset(rig.tok, rig.offs, rig.h0, sub, KR, adapters=rig.ad)
    _eq(after, want_after, "a pick after the updates")
    assert not H.picks_equal(c.pick_batch(rig.tok, rig.offs, rig.h0, adapters=rig.ad), plain_before)
    for e in low:
        assert np.array_equal(g.lru_dump(e), c.lru(e)), f"LRU of endpoint {e}"
    rig.close()


@pytest.mark.parametrize("block_bytes", BLOCK_BYTES)
def test_ops_before_a_held_early_exit_pick(block_bytes):
    """lru_capacity = 0 and no chains_out: hash_chain stops each request at its first block no endpoint holds, reading
    the index while it hashes.  An index_apply issued after the caller's stream started spinning and before the pick
    extends the cached prefixes; the pick sees all of it."""
    torch = _torch()
    rig = Rig(block_bytes, lru_capacity=0, seed=1)
    g, c, s = rig.gpu, rig.cpu, torch.cuda.Stream()
    nbytes = rig.tok.nbytes
    rig.decoy()
    g.pick_batch_device(*rig.ptrs()[:3], R, nbytes, rig.out.data_ptr(), 0, s.cuda_stream)  # warm-up
    rig.decoy()
    e_in = rig.late(s)
    ops = H.ops_array([(int(rig.chains[r, j]), (r * 3) % E, abi.FI_OP_SET) for r in range(R)
                       for j in range(int(rig.nb[r]) * (r % 4) // 3)])
    g.index_apply(ops)
    g.pick_batch_device(*rig.ptrs()[:3], R, nbytes, rig.out.data_ptr(), 0, s.cuda_stream)
    _held(e_in, "the early-exit pick")
    got, _ = rig.snapshot(s)
    want_before = c.pick_batch(rig.tok, rig.offs, rig.h0)
    c.index_apply(ops)
    want = c.pick_batch(rig.tok, rig.offs, rig.h0)
    assert not H.picks_equal(want, want_before)
    _eq(got, want, "early-exit pick after index_apply")
    rig.close()
