"""GPU (-m gpu): fi_epp_resize_pool (docs/SPEC.md S.2c) against the extended CPU oracle.

The oracle resizes with ExtOracle.resize, which tests/test_resize_cpu.py holds to S.2c's definition (a fresh pool fed
the history without the dropped endpoints).  Here the GPU is compared with it bit for bit after every resize and after
further calls: single, ranked and subset picks (PD config, by-label filter, LoRA), index membership of every hash the
calls ever aimed anywhere, the device LRU's content, the LRU entry total and the pairs a shrink removed.  The sharded
pool's FI_ERR_STATE needs several GPUs and is not exercised here.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import helpers as H
from tests import resize_ref as RR
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu


def _pair(cfg):
    return EndpointPicker(cfg), ExtOracle(cfg, track_removal=True)


def _both(gpu, ora, entries):
    for entry in entries:
        RR.apply(gpu, entry)
        RR.apply(ora, entry)


def _probe_endpoints(E, rng):
    if E <= 160:
        return np.arange(E)
    return np.unique(np.concatenate([np.arange(64), rng.choice(E, size=96, replace=False), [E - 1]]))


def _picks(gpu, ora, cs, E, what):
    """single, ranked and subset picks of the stream's prompts, with adapters"""
    tok, offs, h0 = cs.tok, cs.offs, cs.h0
    ad = cs.adapters()
    got, want = gpu.pick_batch(tok, offs, h0, adapters=ad), ora.pick_batch(tok, offs, h0, adapters=ad)
    assert H.picks_equal(got, want), what + " (single)\n" + H.describe_diff(got, want)
    got, want = gpu.pick_batch_ranked(tok, offs, h0, 4, adapters=ad), ora.pick_batch_ranked(tok, offs, h0, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (ranked)\n" + H.describe_diff(got, want)
    sub = cs.subsets(E)
    got, want = gpu.pick_batch_subset(tok, offs, h0, sub, 4, adapters=ad), ora.pick_batch_subset(tok, offs, h0, sub, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (subset)\n" + H.describe_diff(got, want)
    return got


def _check(gpu, ora, cs, E, what, lru=True):
    _picks(gpu, ora, cs, E, what)
    eps = _probe_endpoints(E, cs.rng)
    q = np.zeros(len(cs.hashes) * len(eps), dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(cs.hashes, len(eps))
    q["endpoint"] = np.tile(eps.astype(np.uint32), len(cs.hashes))
    got = gpu.index_contains(q)
    want = np.array([ora.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
    assert np.array_equal(got, want), f"{what}: {int((got != want).sum())} of {len(q)} memberships differ"
    if lru:
        for e in range(E):
            assert np.array_equal(gpu.lru_dump(e), ora.lru(e)), (what, e)
        assert gpu.index_stats().lru_entries == sum(ora.lru_size(e) for e in range(E)), what


def _resize(gpu, ora, En):
    got = gpu.resize_pool(En, count=True)
    want = ora.resize(En)
    assert got == want, f"pairs removed: {got} vs the oracle's {want}"
    assert gpu.cfg.num_endpoints == gpu.cfg.endpoint_count == En


@pytest.mark.parametrize("E,En", [(33, 60), (60, 200), (1, 4096), (1024, 100), (4096, 1), (100, 97), (50, 50)])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("holes", [False, True])
def test_size_transitions(E, En, mode, holes):
    """Direct SETs, device-LRU Adds, capacities, adapters and states; resize; check; then Adds to kept and new
    endpoints, capacities on new ones, a removal and a resize back, where the dropped endpoints return empty."""
    cfg = RR.config(E, match_mode=mode)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(E * 7 + En + holes, cfg)
    if not holes:  # every endpoint listed and alive
        _both(gpu, ora, [("states", H.states_array(E, roles=abi.FI_ROLE_WORKER | RR.LABEL))])
    _both(gpu, ora, cs.calls(E, n=12))
    _check(gpu, ora, cs, E, "before")
    _resize(gpu, ora, En)
    _check(gpu, ora, cs, En, f"after {E} -> {En}")
    if not holes and En > E:
        _both(gpu, ora, [("states", H.states_array(En, roles=abi.FI_ROLE_WORKER | RR.LABEL))])
    new = np.arange(E, En, dtype=np.uint32) if En > E else np.array([En - 1], dtype=np.uint32)
    caps = np.full(min(len(new), 3), cfg.max_blocks + 3, dtype=np.uint32)
    _both(gpu, ora, cs.calls(En, n=8) + [("caps", new[: len(caps)], caps),
                                         ("chains", new[cs.rng.integers(0, len(new), size=24)], cs.chains[:24].copy(),
                                          cs.nb[:24].copy())])
    victims = sorted(set(int(x) for x in cs.rng.integers(0, En, size=2)))
    assert gpu.remove_endpoints(victims, count=True) == _removed(ora, cs, victims)
    ora.remove_endpoints(victims)
    _check(gpu, ora, cs, En, f"after more calls at {En}")
    _resize(gpu, ora, E)
    _check(gpu, ora, cs, E, f"after {En} -> {E}")
    for e in range(min(E, En), E):
        assert len(gpu.lru_dump(e)) == 0
    _both(gpu, ora, cs.calls(E, n=6))
    _check(gpu, ora, cs, E, f"after more calls at {E}")
    gpu.close()
    ora.close()


def _removed(ora, cs, eps):
    return sum(ora.index_contains(e, int(h)) for e in eps for h in cs.hashes)


def _device(cs, R):
    import torch

    d_tok = torch.from_numpy(np.ascontiguousarray(cs.tok).view(np.uint8).copy()).cuda()
    d_off = torch.from_numpy(cs.offs[: R + 1].copy().view(np.int64)).cuda()
    d_h0 = torch.full((R,), cs.h0, dtype=torch.int64, device="cuda")
    return d_tok, d_off, d_h0


def test_pipeline_across_a_resize():
    """Submit A keeping its chains, resize, submit B: A is the old pool's pick, B the new pool's.  index_add_submitted(A)
    with endpoints of the new pool then evicts like the oracle; one endpoint past the new pool is refused, and nothing
    changes."""
    import torch

    E, En = 80, 40
    cfg = RR.config(E)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(11, cfg)
    _both(gpu, ora, [("states", H.states_array(E, roles=abi.FI_ROLE_WORKER | RR.LABEL))] + cs.calls(E, n=10))
    R, P = cs.R, cfg.n_profiles
    d_tok, d_off, d_h0 = _device(cs, R)
    s = torch.cuda.current_stream().cuda_stream
    out_a = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    out_b = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    want_a = ora.pick_batch(cs.tok, cs.offs, cs.h0)
    ta = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out_a.data_ptr(), stream=s)
    _resize(gpu, ora, En)
    want_b = ora.pick_batch(cs.tok, cs.offs, cs.h0)
    tb = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out_b.data_ptr(), stream=s)
    gpu.pick_wait_batch(tb, s)
    torch.cuda.synchronize()
    got_a = out_a.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
    got_b = out_b.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
    assert H.picks_equal(got_a, want_a), "A (old pool)\n" + H.describe_diff(got_a, want_a)
    assert H.picks_equal(got_b, want_b), "B (new pool)\n" + H.describe_diff(got_b, want_b)
    nb = want_a[:, 0]["n_blocks"].astype(np.uint32)
    eps = cs.rng.integers(0, En, size=R).astype(np.uint32)
    bad = eps.copy()
    bad[5] = En
    # (no pick in between: a stream-ordered pick would take the ticket's chains)
    entries = gpu.index_stats().lru_entries
    with pytest.raises(FiEppError) as ei:
        gpu.index_add_submitted(ta, bad, nb)
    assert ei.value.status == abi.FI_ERR_INVALID
    assert gpu.index_stats().lru_entries == entries
    for e in range(En):
        assert np.array_equal(gpu.lru_dump(e), ora.lru(e)), e
    gpu.index_add_submitted(ta, eps, nb)
    ora.index_add_chains(eps, cs.chains, nb)
    _check(gpu, ora, cs, En, "after index_add_submitted of the earlier ticket")
    gpu.close()
    ora.close()


def test_index_shape_follows_the_pool():
    """index_slots = 0: a resize across a power of two of the default takes the new default; a pinned index_slots is
    kept; a shrink whose direct-SET keys exceed the new default keeps room for them.  Picks stay exact throughout."""
    # default slots for lru_capacity 48: 4 096 at 40 endpoints, 32 768 at 200
    for pinned, sizes in ((0, (40, 200, 40)), (1 << 14, (40, 200, 40))):
        cfg = RR.config(sizes[0], index_slots=pinned)
        gpu, ora = _pair(cfg)
        cs = RR.CallStream(3, cfg)
        _both(gpu, ora, cs.calls(sizes[0], n=8))
        for En in sizes[1:]:
            _resize(gpu, ora, En)
            want = pinned or (32768 if En == 200 else 4096)
            assert gpu.index_stats().slots == want, (pinned, En)
            _both(gpu, ora, cs.calls(En, n=4))
            _check(gpu, ora, cs, En, f"index_slots={pinned}, {En} endpoints", lru=False)
        gpu.close()
        ora.close()
    cfg = RR.config(200)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(4, cfg)
    keys = np.arange(1, 9001, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    ops = np.zeros(len(keys), dtype=H.OP_DTYPE)
    ops["hash"], ops["endpoint"], ops["op"] = keys, np.arange(len(keys)) % 5, abi.FI_OP_SET
    _both(gpu, ora, [("ops", ops)] + cs.calls(200, n=6))
    _resize(gpu, ora, 10)
    assert gpu.index_stats().slots * 6 >= len(keys) * 10 and gpu.index_stats().slots > 4096
    q = np.zeros(len(keys), dtype=H.OP_DTYPE)
    q["hash"], q["endpoint"] = keys, np.arange(len(keys)) % 5
    assert gpu.index_contains(q).all()
    _check(gpu, ora, cs, 10, "after a shrink below the direct SETs' keys")
    gpu.close()
    ora.close()


def test_errors_change_nothing():
    cfg = RR.config(20)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(5, cfg)
    _both(gpu, ora, cs.calls(20, n=8))
    before = gpu.pick_batch(cs.tok, cs.offs, cs.h0)
    for En, status in ((0, abi.FI_ERR_INVALID), (4097, abi.FI_ERR_INVALID)):
        with pytest.raises(FiEppError) as ei:
            gpu.resize_pool(En)
        assert ei.value.status == status
        assert H.picks_equal(gpu.pick_batch(cs.tok, cs.offs, cs.h0), before)
    assert gpu.cfg.num_endpoints == 20
    _check(gpu, ora, cs, 20, "after the refused resizes")
    gpu.close()
    ora.close()
    # a handle over part of the pool
    sub = RR.config(64)
    sub.endpoint_count = 32
    gpu = EndpointPicker(sub)
    gpu.update_endpoints(H.states_array(32))
    before = gpu.pick_batch(cs.tok, cs.offs, cs.h0)
    with pytest.raises(FiEppError) as ei:
        gpu.resize_pool(48)
    assert ei.value.status == abi.FI_ERR_STATE
    assert H.picks_equal(gpu.pick_batch(cs.tok, cs.offs, cs.h0), before)
    gpu.close()
    # a handle the host LRU already serves
    gpu, ora = _pair(cfg)
    gpu.set_option("device_lru", 0)
    _both(gpu, ora, [("chains", np.arange(8, dtype=np.uint32), cs.chains[:8].copy(), cs.nb[:8].copy())])
    before = gpu.pick_batch(cs.tok, cs.offs, cs.h0)
    with pytest.raises(FiEppError) as ei:
        gpu.resize_pool(30)
    assert ei.value.status == abi.FI_ERR_STATE
    assert H.picks_equal(gpu.pick_batch(cs.tok, cs.offs, cs.h0), before)
    _check(gpu, ora, cs, 20, "host LRU, after the refused resize", lru=False)
    gpu.close()
    ora.close()


@pytest.mark.parametrize("device_lru", [1, 0])
def test_resize_before_the_first_add(device_lru):
    """Both LRUs are ready for the new pool until one is chosen: Adds through the device LRU, or through the host LRU
    selected after the resize, match the oracle (capacities set before the resize carry over)."""
    cfg = RR.config(30)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(6 + device_lru, cfg)
    _both(gpu, ora, [("states", H.states_array(30)), ("caps", np.array([3, 29], dtype=np.uint32),
                                                      np.array([20, 20], dtype=np.uint32))])
    _resize(gpu, ora, 70)
    gpu.set_option("device_lru", device_lru)
    _both(gpu, ora, [c for c in cs.calls(70, n=16)] + [("chains", np.arange(64, dtype=np.uint32) % 70, cs.chains.copy(),
                                                        cs.nb.copy())])
    _check(gpu, ora, cs, 70, f"device_lru={device_lru}", lru=bool(device_lru))
    assert gpu.index_stats().lru_entries == sum(ora.lru_size(e) for e in range(70))
    gpu.close()
    ora.close()


def test_lazy_buffers_are_reallocated():
    """Every lazily allocated buffer group used once (removal, subset staging, ranked staging, device-LRU plans and
    capacity rounds, index_add_submitted's plans), then a resize, then each used again."""
    import torch

    cfg = RR.config(50)
    gpu, ora = _pair(cfg)
    cs = RR.CallStream(8, cfg)
    R, P = cs.R, cfg.n_profiles
    d_tok, d_off, d_h0 = _device(cs, R)
    s = torch.cuda.current_stream().cuda_stream
    out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")

    def use_all(E, what):
        _both(gpu, ora, cs.calls(E, n=8))
        gpu.remove_endpoints([E - 1])
        ora.remove_endpoints([E - 1])
        _both(gpu, ora, [("caps", np.array([0, E // 2], dtype=np.uint32), np.array([cfg.max_blocks] * 2, dtype=np.uint32))])
        t = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(cs.offs[R]), out.data_ptr(), stream=s)
        want = ora.pick_batch(cs.tok, cs.offs, cs.h0)
        eps = cs.rng.integers(0, E, size=R).astype(np.uint32)
        nb = want[:, 0]["n_blocks"].astype(np.uint32)
        gpu.index_add_submitted(t, eps, nb)
        ora.index_add_chains(eps, cs.chains, nb)
        gpu.pick_wait_batch(t, s)
        torch.cuda.synchronize()
        got = out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P)
        assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)
        _check(gpu, ora, cs, E, what)

    use_all(50, "before the resize")
    for En in (150, 20, 33):
        _resize(gpu, ora, En)
        use_all(En, f"after the resize to {En}")
    gpu.close()
    ora.close()
