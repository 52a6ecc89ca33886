"""GPU (-m gpu): per-endpoint LRU capacities (fi_epp_set_lru_capacities, SPEC S.2b) against the CPU reference.

The reference is tests/ext_oracle.cpp: the CPU oracle with an LRU capacity per endpoint.  Every check is
bit-exact: the device LRU's recency order (fi_epp_lru_dump) against the reference's, index
membership (fi_epp_index_contains) and picks against the oracle's.  Where a test takes `device_lru`, it runs on the
device LRU and on the host LRU (device_lru = 0), whose recency order is not observable (membership and picks are).
"""
import threading

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.dist import shard_range
from fusioninfer_b200.picker import FiEppError
from tests import helpers as H
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q
WEIGHTED = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]


class _Run:
    """a handle and its reference fed the same calls; `ever` = every key added so far"""

    def __init__(self, device_lru=1, E=40, R=256, T=512, max_blocks=32, cap=120, seed=0, track_removal=False, **cfg_kw):
        self.wl = H.small_workload(E=E, R=R, T=T, max_blocks=max_blocks, lru_capacity=0)
        self.cfg = H.config_for(self.wl, profiles=WEIGHTED, lru_capacity=cap, index_slots=1 << 17, **cfg_kw)
        self.gpu = EndpointPicker(self.cfg)
        self.gpu.set_option("device_lru", device_lru)
        self.device_lru = device_lru
        self.ref = ExtOracle(self.cfg, track_removal=track_removal)
        st = self.wl.endpoint_states()
        self.gpu.update_endpoints(st)
        self.ref.update_endpoints(st)
        self.rng = np.random.default_rng(seed)
        self.ever = set()
        self.E, self.R, self.C, self.mb = E, R, cap, max_blocks

    def close(self):
        self.gpu.close()
        self.ref.close()

    def picks(self, batch, what=""):
        tok, offs = self.wl.prompts(batch=batch)
        got, ch = self.gpu.pick_batch(tok, offs, self.wl.h0, want_chains=True)
        want = self.ref.pick_batch(tok, offs, self.wl.h0)
        assert H.picks_equal(got, want), f"batch {batch} {what}\n" + H.describe_diff(got, want)
        return got, ch

    def step(self, batch, hot=(), hot_share=0.5):
        """pick batch `batch`, then Add every chain to its picked endpoint, or (hot_share of them) to a hot one"""
        got, ch = self.picks(batch)
        eps = got[:, 0]["endpoint"].copy()
        nb = got[:, 0]["n_blocks"].copy()
        if len(hot):
            sel = self.rng.random(self.R) < hot_share
            eps[sel] = self.rng.choice(np.asarray(hot, dtype=np.uint32), size=int(sel.sum()))
        self.add(eps, ch, nb)
        return eps, ch, nb

    def add(self, eps, ch, nb):
        self.gpu.index_add_chains(eps, ch, nb)
        self.ref.index_add_chains(eps, ch, nb)
        for r in range(len(eps)):
            self.ever.update(int(k) for k in ch[r, : nb[r]])

    def set_caps(self, eps, caps):
        got = self.gpu.set_lru_capacities(eps, caps, want_evicted=True)
        gone = self.ref.set_lru_capacities(eps, caps)
        assert got == len(gone), f"entries evicted: {got} vs the reference's {len(gone)}"
        return gone

    def membership(self, keys=None, endpoints=None):
        keys = sorted(self.ever) if keys is None else list(keys)
        keys = keys[:: max(1, len(keys) // 400)]
        endpoints = np.arange(self.E) if endpoints is None else np.asarray(endpoints)
        q = np.zeros(len(keys) * len(endpoints), dtype=H.OP_DTYPE)
        q["hash"] = np.repeat(np.asarray(keys, dtype=np.uint64), len(endpoints))
        q["endpoint"] = np.tile(endpoints.astype(np.uint32), len(keys))
        got = self.gpu.index_contains(q)
        want = np.array([self.ref.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
        assert np.array_equal(got, want), f"{int((got != want).sum())} of {len(q)} memberships differ"
        return got

    def check(self, batch=None):
        self.membership()
        assert self.gpu.index_stats().lru_entries == sum(self.ref.lru_size(e) for e in range(self.E))
        if self.device_lru:
            for e in range(self.E):
                assert np.array_equal(self.gpu.lru_dump(e), self.ref.lru(e)), f"LRU of endpoint {e}"
        if batch is not None:
            self.picks(batch, "(check)")


@pytest.mark.parametrize("device_lru", [1, 0])
def test_random_capacities(device_lru):
    """Random capacities in [max_blocks, lru_capacity], hot endpoints receiving many times their capacity in one
    batch, capacities redrawn between batches."""
    run = _Run(device_lru, seed=1)
    caps = run.rng.integers(run.mb, run.C + 1, size=run.E)
    caps[:3] = [run.mb, run.C, 0]
    run.set_caps(np.arange(run.E), caps)
    for b in range(8):
        hot = run.rng.choice(run.E, size=2, replace=False)
        run.step(b, hot=hot, hot_share=0.6)
        run.check(batch=b + 1)
        if b % 3 == 2:
            eps = run.rng.choice(run.E, size=10, replace=False)
            run.set_caps(eps, run.rng.integers(run.mb, run.C + 1, size=len(eps)))
            run.check()
    run.close()


@pytest.mark.parametrize("device_lru", [1, 0])
def test_shrink_then_grow(device_lru):
    """Shrink several endpoints mid-stream, grow some back, Add more: the evicted pairs leave the index, including one
    first SET directly through fi_epp_index_apply, and later Adds fill the grown LRUs up to their new capacity."""
    run = _Run(device_lru, seed=2)
    hot = [3, 7, 11]
    run.step(0, hot=hot)
    run.step(1, hot=hot)
    # a pair SET directly, then taken into endpoint 3's LRU by an Add, then 40 newer keys on top of it
    fresh = run.rng.integers(1, 2**63, size=41, dtype=np.uint64)
    direct, newer = int(fresh[0]), fresh[1:]
    ops = H.ops_array([(direct, 3, abi.FI_OP_SET)])
    run.gpu.index_apply(ops)
    run.ref.index_apply(ops)
    for chain in (np.array([direct], dtype=np.uint64), newer):
        run.gpu.index_add_chain(3, chain)
        run.ref.index_add_chain(3, chain)
        run.ever.update(int(k) for k in chain)
    run.check(batch=2)
    gone = run.set_caps(hot + [20], [run.mb, run.mb, 50, 0])
    assert (direct, 3) in gone, "the directly SET pair should have been evicted"
    assert len(gone) > 0
    q = np.zeros(len(gone), dtype=H.OP_DTYPE)
    q["hash"] = [h for h, _ in gone]
    q["endpoint"] = [e for _, e in gone]
    assert not run.gpu.index_contains(q).any(), "an evicted pair is still in the index"
    run.check(batch=2)
    run.step(2, hot=hot)
    run.check()
    assert run.set_caps([3, 11], [run.C, 90]) == []  # growing evicts nothing
    for b in range(3, 6):
        run.step(b, hot=hot, hot_share=0.7)
        run.check(batch=b + 1)
    assert run.ref.lru_size(3) > 90 and run.ref.lru_size(11) <= 90 and run.ref.lru_size(7) <= run.mb
    run.close()


@pytest.mark.parametrize("case", ["many_endpoints", "one_endpoint"])
def test_rounds_exceed_the_clear_buffer(case):
    """A shrink with more evictions than one CLEAR buffer (2 * max(max_batch * max_blocks, 65 536) ops) runs in
    rounds: many endpoints filled and cut to max_blocks, and one endpoint whose capacity alone exceeds the buffer."""
    mb, pitch = 32, 1024
    # many: 64 endpoints x 4 064 evictions; one: 200 672 evictions of endpoint 0 alone (a round is 131 072 here)
    E, cap, filled = (64, 4096, list(range(64))) if case == "many_endpoints" else (2, 196 * pitch, [0])
    wl = H.small_workload(E=E, R=8, max_blocks=mb, lru_capacity=0)
    cfg = H.config_for(wl, profiles=WEIGHTED, lru_capacity=cap, max_batch=8, index_slots=1 << 20)
    gpu, ref = EndpointPicker(cfg), ExtOracle(cfg)
    rng = np.random.default_rng(3)
    keys = rng.integers(1, 2**63, size=len(filled) * cap, dtype=np.uint64)
    rows = keys.reshape(-1, pitch)
    eps = np.repeat(np.asarray(filled, dtype=np.uint32), cap // pitch)
    nb = np.full(len(rows), pitch, dtype=np.uint32)
    gpu.index_add_chains(eps, rows, nb)
    ref.index_add_chains(eps, rows, nb)
    before = gpu.lru_counters()["clears"]
    got = gpu.set_lru_capacities(filled, [mb] * len(filled), want_evicted=True)
    gone = ref.set_lru_capacities(filled, [mb] * len(filled))
    assert got == len(gone) > 2 * 65536, (got, len(gone))
    assert gpu.lru_counters()["clears"] - before == got
    for e in range(E):
        assert np.array_equal(gpu.lru_dump(e), ref.lru(e)), e
    assert gpu.index_stats().lru_entries == len(filled) * mb
    sample = np.concatenate([keys[:: max(1, len(keys) // 3000)], ref.lru(0)])
    q = np.zeros(len(sample) * 2, dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(sample, 2)
    q["endpoint"] = np.tile(np.array([0, E - 1], dtype=np.uint32), len(sample))
    have = gpu.index_contains(q)
    want = np.array([ref.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
    assert np.array_equal(have, want)
    gpu.close()
    ref.close()


@pytest.mark.parametrize("device_lru", [1, 0])
@pytest.mark.parametrize("value", ["lru_capacity", "zero"])
def test_uniform_capacities_change_nothing(device_lru, value):
    """Every capacity set to lru_capacity (or 0): LRU contents, index membership and picks are identical to those of a
    handle that never called fi_epp_set_lru_capacities."""
    a, b = _Run(device_lru, seed=4), _Run(device_lru, seed=4)
    E = a.E
    assert b.gpu.set_lru_capacities(np.arange(E), [a.C if value == "lru_capacity" else 0] * E, want_evicted=True) == 0
    for batch in range(5):
        tok, offs = a.wl.prompts(batch=batch)
        pa, ca = a.gpu.pick_batch(tok, offs, a.wl.h0, want_chains=True)
        pb = b.gpu.pick_batch(tok, offs, b.wl.h0)
        assert pa.tobytes() == pb.tobytes(), batch
        eps = pa[:, 0]["endpoint"].copy()
        eps[a.rng.random(a.R) < 0.5] = 5
        a.gpu.index_add_chains(eps, ca, pa[:, 0]["n_blocks"])
        b.gpu.index_add_chains(eps, ca, pa[:, 0]["n_blocks"])
        a.ever.update(int(k) for k in ca[ca != 0])
        if batch == 2:
            b.gpu.set_lru_capacities(np.arange(E), [a.C if value == "lru_capacity" else 0] * E)
    keys = sorted(a.ever)[::5]
    q = np.zeros(len(keys) * E, dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(np.asarray(keys, dtype=np.uint64), E)
    q["endpoint"] = np.tile(np.arange(E, dtype=np.uint32), len(keys))
    assert np.array_equal(a.gpu.index_contains(q), b.gpu.index_contains(q))
    assert a.gpu.index_stats().lru_entries == b.gpu.index_stats().lru_entries
    if device_lru:
        for e in range(E):
            assert np.array_equal(a.gpu.lru_dump(e), b.gpu.lru_dump(e)), e
        assert a.gpu.lru_counters() == b.gpu.lru_counters()
    a.close()
    b.close()


def _device_batch(tok, offs, h0, R, mb):
    import torch

    d_tok = torch.from_numpy(np.ascontiguousarray(tok).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs[: R + 1].copy().view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(R * mb, dtype=torch.int64, device="cuda")
    return d_tok, d_off, d_h0, d_out, d_ch


def test_ordering_against_the_pipelined_api():
    """Submit A, set capacities, submit B: A's picks are the reference's before the shrink, B's after it, and
    fi_epp_index_add_submitted(A), issued after the call, evicts against the new capacities."""
    import torch

    run = _Run(1, seed=5)
    for b in range(3):
        run.step(b, hot=[1, 2])
    s = torch.cuda.current_stream().cuda_stream
    (tokA, offsA), (tokB, offsB) = run.wl.prompts(batch=3), run.wl.prompts(batch=4)
    dA = _device_batch(tokA, offsA, run.wl.h0, run.R, run.mb)
    dB = _device_batch(tokB, offsB, run.wl.h0, run.R, run.mb)
    torch.cuda.synchronize()
    wantA, chA = run.ref.pick_batch(tokA, offsA, run.wl.h0, want_chains=True)
    tA = run.gpu.pick_submit_ex(dA[0].data_ptr(), dA[1].data_ptr(), dA[2].data_ptr(), run.R, tokA.nbytes, dA[3].data_ptr(),
                                d_chains=dA[4].data_ptr(), stream=s)
    # the endpoints A's picks hit most lose most of their LRU
    popular = np.argsort(-np.bincount(wantA[:, 0]["endpoint"], minlength=run.E))[:6]
    run.gpu.set_lru_capacities(popular, [run.mb] * 6)  # asynchronous
    gone = run.ref.set_lru_capacities(popular, [run.mb] * 6)
    assert gone
    wantB = run.ref.pick_batch(tokB, offsB, run.wl.h0)
    tB = run.gpu.pick_submit_ex(dB[0].data_ptr(), dB[1].data_ptr(), dB[2].data_ptr(), run.R, tokB.nbytes, dB[3].data_ptr(),
                                d_chains=dB[4].data_ptr(), stream=s)
    run.gpu.pick_wait_batch(tB, s)
    torch.cuda.synchronize()
    gotA = dA[3].cpu().numpy().view(H.PICK_DTYPE).reshape(run.R, 1)
    gotB = dB[3].cpu().numpy().view(H.PICK_DTYPE).reshape(run.R, 1)
    assert H.picks_equal(gotA, wantA), "batch A (submitted before the call)\n" + H.describe_diff(gotA, wantA)
    assert H.picks_equal(gotB, wantB), "batch B (submitted after the call)\n" + H.describe_diff(gotB, wantB)
    epsA, nbA = gotA[:, 0]["endpoint"].copy(), gotA[:, 0]["n_blocks"].copy()
    epsA[: run.R // 2] = popular[0]  # many chains onto one shrunken endpoint
    run.gpu.index_add_submitted(tA, epsA, nbA)
    run.ref.index_add_chains(epsA, chA, nbA)
    run.ever.update(int(k) for k in chA[chA != 0])
    assert len(run.gpu.lru_dump(int(popular[0]))) == run.mb
    run.check(batch=5)
    run.close()


@pytest.mark.parametrize("device_lru", [1, 0])
def test_capacities_set_before_the_first_add(device_lru):
    """Set while the LRU mode is undecided and the device LRU not allocated: they apply to the LRU built later."""
    run = _Run(device_lru, seed=6)
    caps = run.rng.integers(run.mb, run.C + 1, size=run.E)
    assert run.set_caps(np.arange(run.E), caps) == []
    for b in range(4):
        run.step(b, hot=[0, 9], hot_share=0.6)
        run.check(batch=b + 1)
    assert run.ref.lru_size(0) == caps[0] and run.ref.lru_size(9) == caps[9]
    run.close()


@pytest.mark.parametrize("device_lru", [1, 0])
def test_removal_keeps_the_capacity(device_lru):
    """After fi_epp_index_remove_endpoints the emptied LRUs refill only up to their own capacity."""
    run = _Run(device_lru, seed=7, track_removal=True)
    run.set_caps([4, 5, 6], [run.mb, 60, 0])
    for b in range(2):
        run.step(b, hot=[4, 5, 6])
    run.gpu.remove_endpoints([4, 5])
    run.ref.remove_endpoints([4, 5])
    run.check(batch=2)
    for b in range(2, 5):
        run.step(b, hot=[4, 5, 6], hot_share=0.7)
        run.check(batch=b + 1)
    assert run.ref.lru_size(4) == run.mb and run.ref.lru_size(5) == 60 and run.ref.lru_size(6) == run.C
    run.close()


def test_errors_change_nothing():
    """Every rejected call leaves the LRUs, the index and the picks as they were."""
    run = _Run(1, seed=8)
    for b in range(2):
        run.step(b, hot=[2])
    run.check(batch=2)
    dumps = [run.gpu.lru_dump(e) for e in range(run.E)]
    member = run.membership()
    bad = [([run.E], [run.mb], abi.FI_ERR_INVALID),                    # endpoint out of range
           ([1, 2], [run.mb, run.C + 1], abi.FI_ERR_INVALID),          # above lru_capacity
           ([2, 1], [run.mb - 1, run.mb], abi.FI_ERR_INVALID),         # in (0, max_blocks)
           ([2], [1], abi.FI_ERR_INVALID)]
    for eps, caps, status in bad:
        with pytest.raises(FiEppError) as ei:
            run.gpu.set_lru_capacities(eps, caps, want_evicted=True)
        assert ei.value.status == status, (eps, caps)
    lib = abi.load()
    assert lib.fi_epp_set_lru_capacities(run.gpu._h, None, None, 3, None) == abi.FI_ERR_INVALID
    assert run.gpu.set_lru_capacities([], [], want_evicted=True) == 0
    for e in range(run.E):
        assert np.array_equal(run.gpu.lru_dump(e), dumps[e]), e
    assert np.array_equal(run.membership(), member)
    run.check(batch=2)
    run.close()
    wl = H.small_workload(E=8, R=16)
    g = EndpointPicker(H.config_for(wl, lru_capacity=0))
    with pytest.raises(FiEppError) as ei:
        g.set_lru_capacities([1], [0])
    assert ei.value.status == abi.FI_ERR_STATE
    g.close()


def test_sharded_pool_is_refused(gpu_count):
    if gpu_count < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    wl = H.small_workload(E=64, R=32)
    uid = EndpointPicker.comm_unique_id()
    status = [None] * world
    errors = []

    def worker(rank):
        try:
            begin, count = shard_range(wl.E, rank, world)
            p = EndpointPicker(H.config_for(wl, device=rank, endpoint_begin=begin, endpoint_count=count, lru_capacity=400))
            p.comm_init(uid, rank, world)
            try:
                p.set_lru_capacities([0], [64])
            except FiEppError as e:
                status[rank] = e.status
            p.close()
        except Exception as e:  # pragma: no cover
            errors.append((rank, repr(e)))

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=300)
    assert not errors, errors
    assert status == [abi.FI_ERR_STATE] * world
