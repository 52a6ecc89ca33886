"""GPU (-m gpu): fi_epp_index_remove_endpoints (upstream indexer.RemovePod) against the CPU oracle.

The oracle side of a removal is tests/remove_ref.py (the oracle's calls replayed without the removed endpoints).
After every removal the picks are bit-equal to the oracle's after the same calls, the count of removed pairs is the
oracle's, and index membership is false for every removed pair and unchanged for every other one.
"""
import threading

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, make_config
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.dist import shard_range
from fusioninfer_b200.picker import FiEppError
from tests import helpers as H
from tests.remove_ref import RemovalOracle

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q
WEIGHTED = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]
U64_MAX = 0xFFFFFFFFFFFFFFFF


def _pair(cfg):
    return EndpointPicker(cfg), RemovalOracle(cfg)


def _load(wl, gpu, cpu):
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for ops in wl.index_ops():
        gpu.index_apply(ops)
        cpu.index_apply(ops)


def _membership_queries(hashes, endpoints):
    q = np.zeros(len(hashes) * len(endpoints), dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(np.asarray(hashes, dtype=np.uint64), len(endpoints))
    q["endpoint"] = np.tile(np.asarray(endpoints, dtype=np.uint32), len(hashes))
    return q


def _check_membership(gpu, cpu, q):
    got = gpu.index_contains(q)
    want = np.array([cpu.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {len(q)} memberships differ"
    return got


def _remove_both(gpu, cpu, eps):
    got = gpu.remove_endpoints(eps, count=True)
    want = cpu.remove_endpoints(eps)
    assert got == want, f"pairs removed: {got} vs the oracle's {want}"
    return got


def _picks_equal(gpu, cpu, tok, offs, h0, what):
    got = gpu.pick_batch(tok, offs, h0)
    want = cpu.pick_batch(tok, offs, h0)
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)
    return got


@pytest.mark.parametrize("E", [1, 33, 100, 1024, 2048])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("holes", [False, True])
def test_remove_parity_over_pool_sizes(E, mode, holes):
    """One endpoint; endpoints spanning several row words (E = 33: a partial last word); duplicates; the empty list;
    every endpoint — one after the other on the same handle, checked after each."""
    wl = H.small_workload(E=E, R=160, holes=holes, lru_capacity=300)
    cfg = H.config_for(wl, profiles=WEIGHTED, match_mode=mode)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    rng = np.random.default_rng(E)
    first = _picks_equal(gpu, cpu, tok, offs, wl.h0, "before any removal")
    hashes = np.unique(np.concatenate([ops["hash"] for ops in wl.index_ops()]))
    hashes = rng.choice(hashes, size=min(len(hashes), 150), replace=False)
    # the most popular pick goes first: its removal changes many picks
    popular = int(np.bincount(first[:, 0]["endpoint"], minlength=E).argmax())
    sets = [[popular],
            sorted(set(int(x) for x in rng.integers(0, E, size=min(E, 7))) | {E - 1}),  # several words, last (partial) one
            [int(x) for x in rng.integers(0, E, size=3)] * 3,                          # duplicates
            [],
            list(range(E))]
    removed = set()
    for eps in sets:
        before = gpu.index_contains(_membership_queries(hashes, np.arange(E)))
        n = _remove_both(gpu, cpu, eps)
        removed |= set(eps)
        probe = sorted(set(eps) | set(int(x) for x in rng.integers(0, E, size=min(E, 48))))
        q = _membership_queries(hashes, probe)
        have = _check_membership(gpu, cpu, q)
        gone = np.isin(q["endpoint"], list(removed))
        assert not have[gone].any()
        after = gpu.index_contains(_membership_queries(hashes, np.arange(E))).reshape(len(hashes), E)
        keep = np.ones(E, dtype=bool)
        keep[list(set(eps))] = False
        assert np.array_equal(after[:, keep], before.reshape(len(hashes), E)[:, keep]), "other endpoints' pairs changed"
        if eps == []:
            assert n == 0
        _picks_equal(gpu, cpu, tok, offs, wl.h0, f"after removing {eps[:8]}")
    assert gpu.remove_endpoints(list(range(E)), count=True) == 0  # every endpoint already holds nothing
    gpu.close()


def test_upstream_stop_moves_when_the_only_holder_leaves():
    """Upstream mode stops at the first block NO pod holds.  B holds h1..h3 and h5..h8, only A holds h4: B matches 7
    blocks; once A is removed, h4 is held by nobody and B matches 3."""
    cfg = make_config(num_endpoints=2, block_bytes=64, max_blocks=8, max_batch=4, index_slots=4096,
                      profiles=[{"name": "default", "scorers": [(P, 100)]}])
    gpu, cpu = _pair(cfg)
    st = H.states_array(2)
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    data, offs = H.pack_prompts([bytes(range(256)) * 2])  # 8 blocks of 64 bytes
    h0 = 12345
    chains, nb = gpu.hash_batch(data, offs, h0)
    assert nb[0] == 8
    h = [int(x) for x in chains[0, :8]]
    A, B = 0, 1
    ops = H.ops_array([(h[i], B, abi.FI_OP_SET) for i in (0, 1, 2, 4, 5, 6, 7)] + [(h[3], A, abi.FI_OP_SET)])
    gpu.index_apply(ops)
    cpu.index_apply(ops)
    pk = _picks_equal(gpu, cpu, data, offs, h0, "before")
    assert (pk[0, 0]["endpoint"], pk[0, 0]["match_blocks"]) == (B, 7)
    assert _remove_both(gpu, cpu, [A]) == 1
    pk = _picks_equal(gpu, cpu, data, offs, h0, "after")
    assert (pk[0, 0]["endpoint"], pk[0, 0]["match_blocks"]) == (B, 3)
    gpu.close()


def test_direct_sets_and_special_hashes_are_removed():
    """Pairs SET through fi_epp_index_apply (no LRU involved), including the hashes 0 and ~0 that the table uses as
    markers, leave the index; the same keys stay for the endpoints that were not removed."""
    E = 70
    cfg = make_config(num_endpoints=E, max_batch=8, index_slots=8192, lru_capacity=64)
    gpu, cpu = _pair(cfg)
    rng = np.random.default_rng(5)
    universe = np.concatenate([rng.integers(1, 2**63, size=200, dtype=np.uint64), np.array([0, U64_MAX], dtype=np.uint64)])
    ops = np.zeros(3000, dtype=H.OP_DTYPE)
    ops["hash"] = universe[rng.integers(0, len(universe) - 2, size=len(ops))]  # 0 and ~0 only in `special`
    ops["endpoint"] = rng.integers(0, E, size=len(ops))
    ops["op"] = abi.FI_OP_SET
    special = H.ops_array([(0, e, abi.FI_OP_SET) for e in (3, 40, 69)] + [(U64_MAX, e, abi.FI_OP_SET) for e in (3, 41)])
    for o in (ops, special):
        gpu.index_apply(o)
        cpu.index_apply(o)
    q = _membership_queries(universe, np.arange(E))
    _check_membership(gpu, cpu, q)
    n = _remove_both(gpu, cpu, [3, 40, 41, 64])
    assert n > 0
    have = _check_membership(gpu, cpu, q).reshape(len(universe), E)
    assert not have[:, [3, 40, 41, 64]].any()
    assert have[-2, 69] and not have[-1].any()  # 0 still held by 69; ~0 held by nobody
    gpu.close()


@pytest.mark.parametrize("device_lru", [0, 1])
def test_remove_resets_the_lru(device_lru):
    """The removed endpoints' LRUs are empty (lru_dump, lru_entries); re-adding the same chains SETs them again; churn
    past capacity afterwards keeps picks, membership and (device LRU) recency order equal to the oracle."""
    wl = H.small_workload(E=40, R=256, T=512, max_blocks=32, lru_capacity=0)
    cap = 120
    cfg = H.config_for(wl, profiles=WEIGHTED, lru_capacity=cap, index_slots=1 << 17)
    gpu, cpu = _pair(cfg)
    gpu.set_option("device_lru", device_lru)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    ref = H.OrderedLrus(wl.E, cap)
    ever = set()

    def step(batch):
        tok, offs = wl.prompts(batch=batch)
        got, ch = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        want = cpu.pick_batch(tok, offs, wl.h0)
        assert H.picks_equal(got, want), f"batch {batch}\n" + H.describe_diff(got, want)
        eps, nb = got[:, 0]["endpoint"], got[:, 0]["n_blocks"]
        gpu.index_add_chains(eps, ch, nb)
        cpu.index_add_chains(eps, ch, nb)
        for r in range(wl.R):
            ref.add_chain(eps[r], ch[r, : nb[r]])
            ever.update(int(k) for k in ch[r, : nb[r]])
        return eps, ch, nb

    def check():
        keys = sorted(ever)
        _check_membership(gpu, cpu, _membership_queries(keys[:: max(1, len(keys) // 300)], np.arange(wl.E)))
        assert gpu.index_stats().lru_entries == sum(len(l) for l in ref.lru)
        if device_lru:
            for e in range(wl.E):
                assert np.array_equal(gpu.lru_dump(e), np.array(list(ref.lru[e]), dtype=np.uint64)), e

    for b in range(3):
        step(b)
    check()
    eps, ch, nb = step(3)
    victims = sorted(set(int(e) for e in eps[:6]))
    sizes = sum(len(ref.lru[e]) for e in victims)
    assert sizes > 0
    entries = gpu.index_stats().lru_entries
    _remove_both(gpu, cpu, victims)
    ref.remove(victims)
    assert gpu.index_stats().lru_entries == entries - sizes
    if device_lru:
        for e in victims:
            assert len(gpu.lru_dump(e)) == 0
    check()
    # the same chains again: new to the emptied LRUs, so SET again
    gpu.index_add_chains(eps, ch, nb)
    cpu.index_add_chains(eps, ch, nb)
    for r in range(wl.R):
        ref.add_chain(eps[r], ch[r, : nb[r]])
    q = _membership_queries([int(ch[r, 0]) for r in range(wl.R) if eps[r] in victims and nb[r]], victims)
    assert _check_membership(gpu, cpu, q).any()
    check()
    for b in range(4, 12):  # churn past capacity
        step(b)
    check()
    gpu.close()


def _device_batch(tok, offs, h0, R):
    import torch

    d_tok = torch.from_numpy(np.ascontiguousarray(tok[:R]).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs[: R + 1].copy().view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    return d_tok, d_off, d_h0, d_out


@pytest.mark.parametrize("path", ["submit", "stream_ordered", "host_lru_staged"])
def test_removal_is_ordered_between_picks(path):
    """A pick called before the removal does not see it (also while it is still in flight), a pick called after it
    does.  host_lru_staged: host-LRU deltas still staged (not yet launched) at the call are applied before it."""
    import torch

    wl = H.small_workload(E=64, R=256, T=512, max_blocks=32, lru_capacity=200)
    cfg = H.config_for(wl, profiles=WEIGHTED, lru_capacity=200 if path == "host_lru_staged" else 0)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    s = torch.cuda.current_stream().cuda_stream
    tok0, offs0 = wl.prompts(batch=0)
    tok1, offs1 = wl.prompts(batch=1)
    R = wl.R
    b0 = _device_batch(tok0, offs0, wl.h0, R)
    b1 = _device_batch(tok1, offs1, wl.h0, R)
    torch.cuda.synchronize()
    if path == "host_lru_staged":
        gpu.set_option("device_lru", 0)
        want0, ch = cpu.pick_batch(tok0, offs0, wl.h0, want_chains=True)
        eps, nb = want0[:, 0]["endpoint"], want0[:, 0]["n_blocks"]
        gpu.index_add_chains(eps, ch, nb)  # the deltas stay staged until the next flush
        cpu.index_add_chains(eps, ch, nb)
    else:
        want0 = cpu.pick_batch(tok0, offs0, wl.h0)
    victims = sorted(set(int(e) for e in want0[:40, 0]["endpoint"]))
    if path == "submit":
        gpu.pick_submit(b0[0].data_ptr(), b0[1].data_ptr(), b0[2].data_ptr(), R, tok0.nbytes, b0[3].data_ptr(), s)
    elif path == "stream_ordered":
        gpu.pick_batch_device(b0[0].data_ptr(), b0[1].data_ptr(), b0[2].data_ptr(), R, tok0.nbytes, b0[3].data_ptr(), 0, s)
    gpu.remove_endpoints(victims)  # asynchronous
    cpu.remove_endpoints(victims)
    want1 = cpu.pick_batch(tok1, offs1, wl.h0)
    if path == "submit":
        gpu.pick_submit(b1[0].data_ptr(), b1[1].data_ptr(), b1[2].data_ptr(), R, tok1.nbytes, b1[3].data_ptr(), s)
        gpu.pick_wait(s)
    else:
        gpu.pick_batch_device(b1[0].data_ptr(), b1[1].data_ptr(), b1[2].data_ptr(), R, tok1.nbytes, b1[3].data_ptr(), 0, s)
    torch.cuda.synchronize()
    if path != "host_lru_staged":
        got0 = b0[3].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        assert H.picks_equal(got0, want0), "the pick called before the removal\n" + H.describe_diff(got0, want0)
    got1 = b1[3].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
    assert H.picks_equal(got1, want1), "the pick called after the removal\n" + H.describe_diff(got1, want1)
    assert not np.isin(got1[:, 0]["endpoint"][got1[:, 0]["match_blocks"] > 0], victims).any()
    gpu.close()


def test_removal_tombstones_trigger_a_rebuild():
    """Removing every endpoint retires every key; the tombstones let a small table take new keys by rebuilding (with
    the keys still live it would be full), and everything stays exact after the rebuild."""
    wl = H.small_workload(E=16, R=64, T=64, max_blocks=4, lru_capacity=40)
    cfg = H.config_for(wl, profiles=WEIGHTED, index_slots=2048)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    _picks_equal(gpu, cpu, tok, offs, wl.h0, "loaded")
    used0 = gpu.index_stats().used
    assert _remove_both(gpu, cpu, list(range(wl.E))) > 0
    st = gpu.index_stats()
    assert st.tombstones == used0 and st.rebuilds == 0
    rng = np.random.default_rng(9)
    fresh = []
    for _ in range(30):
        ks = rng.integers(1, 2**63, size=100, dtype=np.uint64)
        fresh.extend(int(k) for k in ks)
        ops = H.ops_array([(int(k), int(e), abi.FI_OP_SET) for k, e in zip(ks, rng.integers(0, wl.E, size=100))])
        gpu.index_apply(ops)
        cpu.index_apply(ops)
        gpu.index_sync()
        if gpu.index_stats().rebuilds:
            break
    assert gpu.index_stats().rebuilds >= 1
    for ops in wl.index_ops(0, 4):  # a quarter of the pool back: still below 60 % live keys
        gpu.index_apply(ops)
        cpu.index_apply(ops)
    _picks_equal(gpu, cpu, tok, offs, wl.h0, "after the rebuild")
    _check_membership(gpu, cpu, _membership_queries(fresh[::7], np.arange(wl.E)))
    gpu.close()


def test_out_of_range_endpoint_is_rejected_and_nothing_changes():
    wl = H.small_workload(E=40, R=128)
    cfg = H.config_for(wl, profiles=WEIGHTED)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    before = _picks_equal(gpu, cpu, tok, offs, wl.h0, "loaded")
    with pytest.raises(FiEppError) as ei:
        gpu.remove_endpoints([1, 2, wl.E], count=True)
    assert ei.value.status == abi.FI_ERR_INVALID
    assert H.picks_equal(gpu.pick_batch(tok, offs, wl.h0), before)
    hashes = np.concatenate([ops["hash"] for ops in wl.index_ops()])[::50]
    _check_membership(gpu, cpu, _membership_queries(hashes, np.arange(wl.E)))
    gpu.close()


def test_sharded_pool_is_refused(gpu_count):
    """Sharded pools return FI_ERR_STATE: their removal would have to gossip its VANISH transitions in rounds."""
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
            p = EndpointPicker(H.config_for(wl, device=rank, endpoint_begin=begin, endpoint_count=count))
            p.comm_init(uid, rank, world)
            try:
                p.remove_endpoints([0])
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
