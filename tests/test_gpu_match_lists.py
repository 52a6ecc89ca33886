"""GPU (-m gpu): fi_epp_match_lists / _device (docs/SPEC.md S.3b), bit-exact against the sparsified match counts of the
same handle (fi_epp_match_counts) and of the oracle (tests/match_lists_ref.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from fusioninfer_b200 import EndpointPicker, make_config, synth
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import craft
from tests import helpers as H
from tests import match_counts_cases as MC
from tests import match_lists_ref as ML
from tests.ext_oracle import ExtOracle
from tests.test_gpu_match_counts import PROFILES, Inputs

pytestmark = pytest.mark.gpu
MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
SENTINEL = 0xA5


def _cfg(E, B, M, R, mode, lru, **kw):
    kw.setdefault("index_slots", 1 << 16)
    return H.make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=lru, max_batch=R, match_mode=mode,
                         profiles=PROFILES, **kw)


def device_lists(p, x: Inputs, cap: int, stream=None, chains=False, room=None):
    """fi_epp_match_lists_device into sentinel-filled buffers -> (offsets, entries [room] as left by the call, nblocks[,
    chains]); the entry buffer holds room >= cap entries (default cap) and the call is given cap"""
    room = cap if room is None else room
    assert room >= cap
    off = torch.full((x.R + 1,), -1, dtype=torch.int64, device="cuda")
    ent = torch.full((max(room, 1) * 8,), SENTINEL, dtype=torch.uint8, device="cuda")
    nb = torch.zeros(max(x.R, 1), dtype=torch.int32, device="cuda")
    ch = torch.zeros((max(x.R, 1), p.max_blocks), dtype=torch.int64, device="cuda") if chains else None
    s = stream or torch.cuda.current_stream()
    p.match_lists_device(x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), x.R, int(x.offs[-1]),
                         off.data_ptr(), ent.data_ptr() if cap else 0, cap, nb.data_ptr(),
                         ch.data_ptr() if chains else 0, s.cuda_stream)
    s.synchronize()
    out = (off.cpu().numpy().view(np.uint64).copy(), ent.cpu().numpy()[: room * 8].copy().view(ML.ENTRY),
           nb.cpu().numpy().view(np.uint32)[: x.R].copy())
    return out + (ch.cpu().numpy().view(np.uint64)[: x.R].copy(),) if chains else out


def check(p, o, x: Inputs, begin=0):
    """host and device lists equal the sparsified counts of the handle and of the oracle; -> (offsets, entries)"""
    want_off, want, wnb = ML.oracle_lists(o, x.tok, x.offs, x.h0)
    counts, _ = p.match_counts(x.tok, x.offs, x.h0)
    s_off, s_ent = ML.sparsify(counts, begin)
    assert np.array_equal(s_off, want_off) and s_ent.tobytes() == want.tobytes()
    off, ent, nb = p.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(off, want_off) and ent.tobytes() == want.tobytes() and np.array_equal(nb, wnb)
    total = int(want_off[-1])
    doff, dent, dnb = device_lists(p, x, total + 3, room=total + 5)
    assert np.array_equal(doff, want_off) and np.array_equal(dnb, wnb)
    assert dent[:total].tobytes() == want.tobytes() and (dent[total:].view(np.uint8) == SENTINEL).all()
    return want_off, want


def _world(E, B, M, R, mode, lru, seed, shard=None, **kw):
    rng = np.random.default_rng(seed)
    tok, offs = MC.prompts(R, B, M, rng)
    if shard is not None:
        kw.update(endpoint_begin=shard[0], endpoint_count=shard[1])
    p = EndpointPicker(_cfg(E, B, M, R, mode, lru, **kw))
    o = ExtOracle(_cfg(E, B, M, R, mode, lru), shard=shard, track_removal=lru > 0)
    return rng, p, o, Inputs(tok, offs, 0x5EED + seed)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [64, 96, 5])
@pytest.mark.parametrize("E", [8, 40, 1024, 4096])
def test_lists_equal_the_sparsified_counts(mode, B, E):
    """SET / CLEAR with holes, then Adds through the device LRU after a lists call (its chains), then removals"""
    M, R = 48, 160
    rng, p, o, x = _world(E, B, M, R, mode, lru=2 * M, seed=E + B)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2):
        p.index_apply(ops)
        o.index_apply(ops)
    off, _ = check(p, o, x)
    assert off[-1] > R and (np.diff(off) == 0).any()
    for dest, _, _ in MC.add_batches(chains, nb, E, rng, batches=2):
        _, _, gnb, gch = p.match_lists(x.tok, x.offs, x.h0, want_chains=True)
        assert np.array_equal(gch, chains)
        p.index_add_chains_device(dest, 0, 0, gnb)  # the chains of the lists call just made
        o.index_add_chains(dest, chains, nb)
        check(p, o, x)
    gone = rng.choice(E, size=min(3, E), replace=False)
    p.remove_endpoints(gone)
    o.remove_endpoints(gone)
    check(p, o, x)
    p.close()
    o.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M", [1023, 2047, 4095])
def test_early_exit_and_long_prompts(mode, M):
    """lru_capacity 0 without chains (hashing stops early), and max_blocks above 1 023 (the windowed kernel)"""
    E, B, R = 40, 64, 24
    rng, p, o, x = _world(E, B, M, R, mode, lru=0, seed=M)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    top = int(np.argmax(nb))
    full = H.ops_array([(int(h), E - 1, abi.FI_OP_SET) for h in chains[top, : nb[top]]])
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2, holes=0.02) + [full]:
        p.index_apply(ops)
        o.index_apply(ops)
    _, ent = check(p, o, x)
    assert int(ent["match_blocks"].max()) == int(nb.max())
    off, ent2, gnb, gch = p.match_lists(x.tok, x.offs, x.h0, want_chains=True)
    hch, hnb = p.hash_batch(x.tok, x.offs, x.h0)
    assert ent2.tobytes() == ent.tobytes() and np.array_equal(gnb, hnb) and np.array_equal(gch, hch)
    p.close()


def test_every_endpoint_no_match_and_marker_hashes():
    """requests whose every block every endpoint holds (nnz = E), requests with no match, and block hashes 0 / ~0"""
    for E in (40, 1024):
        for mode in MODES:
            B, M, R = 64, 16, 64
            rng = np.random.default_rng(E)
            tok, offs = MC.prompts(R, B, M, rng)
            raw = np.ascontiguousarray(tok).view(np.uint8).ravel()
            h0 = np.full(R, 77, dtype=np.uint64)
            for r in range(3, R, 4):
                n = min((int(offs[r + 1]) - int(offs[r])) // B, M)
                if n >= 3:
                    blocks = [bytes(raw[int(offs[r]) + i * B: int(offs[r]) + (i + 1) * B]) for i in range(3)]
                    h0[r] = craft.h0_for(blocks, 1 + (r // 4) % 2, craft.MARKERS[(r // 8) % 2])
            cfg = _cfg(E, B, M, R, mode, 0, index_slots=1 << 14)
            p, o = EndpointPicker(cfg), ExtOracle(cfg)
            x = Inputs(tok, offs, h0)
            chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
            every = [(int(chains[r, i]), e, abi.FI_OP_SET) for r in range(4, 12) for i in range(nb[r]) for e in range(E)]
            for a in [H.ops_array(every)] + MC.family_ops(chains, nb, E, rng, per_endpoint=1)[:1]:
                p.index_apply(a)
                o.index_apply(a)
            off, _ = check(p, o, x)
            lens = np.diff(off)
            assert (lens == E).any() and (lens == 0).any()
            p.close()


def test_capacity():
    """cap 0, total - 1 and total: the host call writes the offsets and exactly the first cap entries and returns
    FI_ERR_CAPACITY; the device call returns FI_OK and leaves entries at cap and beyond untouched"""
    E, B, M, R = 300, 64, 32, 128
    rng, p, o, x = _world(E, B, M, R, abi.FI_MATCH_LPM, lru=0, seed=4)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=3):
        p.index_apply(ops)
        o.index_apply(ops)
    want_off, want, _ = ML.oracle_lists(o, x.tok, x.offs, x.h0)
    total = int(want_off[-1])
    lib, h = p._lib, p._h
    for cap in (0, total - 1, total):
        off = np.zeros(R + 1, dtype=np.uint64)
        ent = np.full(total + 2, 0, dtype=ML.ENTRY)
        ent.view(np.uint8)[:] = SENTINEL
        nbo = np.zeros(R, dtype=np.uint32)
        rc = lib.fi_epp_match_lists(h, x.tok.ctypes.data, x.offs.ctypes.data, x.h0.ctypes.data, R, off.ctypes.data,
                                    ent.ctypes.data if cap else None, cap, nbo.ctypes.data, None)
        assert rc == (abi.FI_OK if cap == total else abi.FI_ERR_CAPACITY)
        assert np.array_equal(off, want_off) and np.array_equal(nbo, nb)
        assert ent[:cap].tobytes() == want[:cap].tobytes() and (ent[cap:].view(np.uint8) == SENTINEL).all()
        # the device buffer has room for every entry and two more; only the first cap may be written
        doff, dent, _ = device_lists(p, x, cap, room=total + 2)
        assert len(dent) == total + 2
        assert np.array_equal(doff, want_off) and dent[:cap].tobytes() == want[:cap].tobytes()
        assert (dent[cap:].view(np.uint8) == SENTINEL).all()
    with pytest.raises(FiEppError) as ei:
        p.match_lists(x.tok, x.offs, x.h0, cap=total - 1)
    assert ei.value.status == abi.FI_ERR_CAPACITY
    p.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shard", [(0, 1), (3, 33), (34, 990), (1000, 24)])
def test_partial_pool_handles_list_global_endpoints(mode, shard):
    E, B, M, R = 1024, 64, 48, 128
    rng, p, o, x = _world(E, B, M, R, mode, lru=2 * M, seed=shard[0], shard=shard)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2):
        p.index_apply(ops)
        o.index_apply(ops)
    _, ent = check(p, o, x, begin=shard[0])
    assert ((ent["endpoint"] >= shard[0]) & (ent["endpoint"] < shard[0] + shard[1])).all()
    p.close()


def test_ordering_resize_snapshot_and_stats():
    """after work on the caller's stream, index updates, a capacity change, resize and snapshot load; statistics"""
    E, B, M, R = 300, 64, 32, 128
    rng, p, o, x = _world(E, B, M, R, abi.FI_MATCH_UPSTREAM, lru=3 * M, seed=11)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for dest, _, _ in MC.add_batches(chains, nb, E, rng, batches=2):
        p.index_add_chains(dest, chains, nb)
        o.index_add_chains(dest, chains, nb)
    check(p, o, x)
    eps = rng.choice(E, size=60, replace=False)
    caps = np.full(60, M, dtype=np.uint32)
    p.set_lru_capacities(eps, caps)
    o.set_lru_capacities(eps, caps)
    off, ent = check(p, o, x)
    q = EndpointPicker(_cfg(E, B, M, R, abi.FI_MATCH_UPSTREAM, 3 * M))
    q.load_snapshot(p.save_snapshot())
    qo, qe, _ = q.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(qo, off) and qe.tobytes() == ent.tobytes()
    q.close()
    p.resize_pool(E + 100)
    go, ge, _ = p.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(go, off) and ge.tobytes() == ent.tobytes()
    p.resize_pool(E - 77)
    o.remove_endpoints(np.arange(E - 77, E))
    want = ML.sparsify(o.match_counts(x.tok, x.offs, x.h0)[0][:, : E - 77])
    go, ge, _ = p.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(go, want[0]) and ge.tobytes() == want[1].tobytes()
    dgo, dge, _ = device_lists(p, x, int(want[0][-1]))
    assert np.array_equal(dgo, want[0]) and dge.tobytes() == want[1].tobytes()
    # behind work still queued on the caller's stream, and after an op issued just before
    ops = MC.family_ops(chains, nb, E - 77, rng, per_endpoint=2)[0]
    p.index_apply(ops)
    o.index_apply(ops)
    want = ML.sparsify(o.match_counts(x.tok, x.offs, x.h0)[0][:, : E - 77])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        late = Inputs(x.tok, x.offs, x.h0)
        late.d_tok = torch.zeros_like(x.d_tok)
        torch.cuda._sleep(50_000_000)
        late.d_tok.copy_(x.d_tok)
        p.reset_stats()
        p.set_profiling(True)
        dgo, dge, _ = device_lists(p, late, int(want[0][-1]), stream=s)
    assert np.array_equal(dgo, want[0]) and dge.tobytes() == want[1].tobytes()
    st = p.stats()
    assert st.pick_calls == 1 and st.requests == R and st.ms_match_pick > 0 and st.ms_other > 0
    p.set_profiling(False)
    p.close()
    o.close()


def test_errors_write_nothing():
    E, B, M, R = 40, 64, 16, 32
    rng, p, o, x = _world(E, B, M, R, abi.FI_MATCH_LPM, lru=0, seed=1, max_prompt_bytes=1 << 16)
    lib, h = p._lib, p._h
    off = np.full(R + 2, 9, dtype=np.uint64)
    ent = np.zeros(R * E, dtype=ML.ENTRY)
    ent.view(np.uint8)[:] = SENTINEL
    nb = np.full(R, 7, dtype=np.uint32)
    args = (x.tok.ctypes.data, x.offs.ctypes.data, x.h0.ctypes.data)
    assert lib.fi_epp_match_lists(None, *args, R, off.ctypes.data, ent.ctypes.data, R * E, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_lists(h, *args, R, None, ent.ctypes.data, R * E, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_lists(h, *args, R, off.ctypes.data, None, 5, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_lists(h, x.tok.ctypes.data, None, x.h0.ctypes.data, R, off.ctypes.data, ent.ctypes.data,
                                  R * E, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_lists_device(h, x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), R, 0, None,
                                         None, 0, None, None, None) == abi.FI_ERR_INVALID
    big = Inputs(np.zeros(70000, np.uint8), np.array([0, 70000], np.uint64), 1)
    assert lib.fi_epp_match_lists(h, big.tok.ctypes.data, big.offs.ctypes.data, big.h0.ctypes.data, 1, off.ctypes.data,
                                  ent.ctypes.data, R * E, nb.ctypes.data, None) == abi.FI_ERR_CAPACITY
    offs33 = np.zeros(R + 2, dtype=np.uint64)
    h033 = np.zeros(R + 1, dtype=np.uint64)
    assert lib.fi_epp_match_lists(h, x.tok.ctypes.data, offs33.ctypes.data, h033.ctypes.data, R + 1, off.ctypes.data,
                                  ent.ctypes.data, R * E, nb.ctypes.data, None) == abi.FI_ERR_CAPACITY
    assert lib.fi_epp_match_lists_device(h, x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), R + 1, 0,
                                         C.c_void_p(8), C.c_void_p(8), 4, None, None, None) == abi.FI_ERR_CAPACITY
    assert (off == 9).all() and (ent.view(np.uint8) == SENTINEL).all() and (nb == 7).all()
    assert lib.fi_epp_match_lists(h, *args, 0, off.ctypes.data, None, 0, None, None) == abi.FI_OK
    assert off[0] == 0 and (off[1:] == 9).all()
    d_off = torch.full((1,), 5, dtype=torch.int64, device="cuda")
    assert lib.fi_epp_match_lists_device(h, None, x.d_offs.data_ptr(), None, 0, 0, d_off.data_ptr(), None, 0, None, None,
                                         None) == abi.FI_OK
    torch.cuda.synchronize()
    assert int(d_off.item()) == 0
    assert p.stats().pick_calls == 0
    p.close()


def test_deterministic_and_sliced_feed():
    """two calls give identical bytes; a host call of >= 8 MiB of prompts (the sliced feed) equals the device call"""
    wl = synth.Workload(R=4096, E=256, T=2304, lru_capacity=160, groups_per_endpoint=4, max_blocks=64, holes=True)
    cfg = H.config_for(wl, profiles=PROFILES, max_prompt_bytes=wl.R * wl.T * 4)
    p, o = EndpointPicker(cfg), ExtOracle(cfg)
    for ops in wl.index_ops():
        p.index_apply(ops)
        o.index_apply(ops)
    tok, offs = wl.prompts()
    x = Inputs(tok, offs, wl.h0)
    assert int(x.offs[-1]) >= 8 << 20
    a = p.match_lists(x.tok, x.offs, x.h0)
    b = p.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes()
    total = int(a[0][-1])
    d1, d2 = device_lists(p, x, total), device_lists(p, x, total)
    assert np.array_equal(d1[0], a[0]) and d1[1].tobytes() == a[1].tobytes() and d2[1].tobytes() == d1[1].tobytes()
    want_off, want, _ = ML.oracle_lists(o, x.tok, x.offs, x.h0)
    assert np.array_equal(a[0], want_off) and a[1].tobytes() == want.tobytes()
    p.close()
    o.close()


def test_full_size_batch_equals_the_dense_call():
    """bench.py's cfg 3: its workload, profiles, index and first batch (16 384 requests over 1 024 endpoints)"""
    wl = synth.baseline_workload(3)
    profiles, pd = synth.baseline_profiles(3)
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=wl.R,
                      max_prompt_bytes=wl.R * wl.T * 4, index_slots=slots, profiles=profiles, pd=pd)
    p = EndpointPicker(cfg)
    p.update_endpoints(wl.endpoint_states())
    for ops in wl.index_ops():
        p.index_apply(ops)
    tok, offs = wl.prompts(batch=0)
    x = Inputs(tok, offs, wl.h0)
    counts, nb = p.match_counts(x.tok, x.offs, x.h0)
    want_off, want = ML.sparsify(counts)
    off, ent, gnb = p.match_lists(x.tok, x.offs, x.h0)
    assert np.array_equal(off, want_off) and ent.tobytes() == want.tobytes() and np.array_equal(gnb, nb)
    doff, dent, _ = device_lists(p, x, int(want_off[-1]))
    assert np.array_equal(doff, want_off) and dent.tobytes() == want.tobytes()
    assert int(want_off[-1]) > wl.R
    p.close()


def test_sharded_pool_is_refused(gpu_count):
    """a sharded pool gets FI_ERR_STATE on every rank and nothing is written (needs >= 2 GPUs)"""
    if gpu_count < 2:
        pytest.skip("needs >= 2 GPUs")
    import threading

    from fusioninfer_b200.dist import shard_range

    world = 2
    wl = H.small_workload(E=64, R=16)
    uid = EndpointPicker.comm_unique_id()
    tok, offs = wl.prompts()
    h0 = np.full(wl.R, wl.h0, dtype=np.uint64)
    results, errors = [None] * world, []

    def worker(rank):
        try:
            begin, count = shard_range(wl.E, rank, world)
            p = EndpointPicker(H.config_for(wl, device=rank, endpoint_begin=begin, endpoint_count=count))
            p.comm_init(uid, rank, world)
            off = np.full(wl.R + 1, 7, dtype=np.uint64)
            ent = np.zeros(wl.R * count, dtype=ML.ENTRY)
            ent.view(np.uint8)[:] = SENTINEL
            raw = np.ascontiguousarray(tok).view(np.uint8)
            rc = p._lib.fi_epp_match_lists(p._h, raw.ctypes.data, offs.ctypes.data, h0.ctypes.data, wl.R, off.ctypes.data,
                                           ent.ctypes.data, len(ent), None, None)
            results[rank] = (rc, bool((off == 7).all() and (ent.view(np.uint8) == SENTINEL).all()))
            p.close()
        except Exception as e:  # pragma: no cover
            errors.append((rank, repr(e)))

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=600)
    assert not errors, errors
    assert results == [(abi.FI_ERR_STATE, True)] * world
