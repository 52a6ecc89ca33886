"""GPU (-m gpu): fi_epp_match_counts / _device (docs/SPEC.md S.3a), bit-exact against the oracle's match_counts
(tests/counts_oracle.cpp) on every row shape of the match kernel, and consistent with the picks of the same handle.

Rows are checked where they are least aligned: the device call writes at an odd 2-byte offset of a guarded buffer,
so rows start anywhere inside a 32-byte sector, and the guards must come back untouched."""
import ctypes as C

import numpy as np
import pytest
import torch

from fusioninfer_b200 import EndpointPicker, synth
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import collide, craft
from tests import helpers as H
from tests import match_counts_cases as MC
from tests import shard_view as SV
from tests.counts_oracle import CountsOracle
from tests.test_match_counts_cpu import check_picks_against_matrix

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q
MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
PROFILES = [{"name": "a", "scorers": [(P, 100), (K, 10), (Q, 10)]},
            {"name": "b", "role_mask": 3, "more_filters": [6], "scorers": [(P, 20), (Q, 7)]}]
GUARD = 0x5A5A


def _cfg(E, B, M, R, mode, lru, **kw):
    kw.setdefault("index_slots", 1 << 16)
    return H.make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=lru, max_batch=R, match_mode=mode,
                         profiles=PROFILES, **kw)


class Inputs:
    """a batch's prompts, offsets and seeds on the host and on the device"""

    def __init__(self, tok, offs, h0):
        self.tok = np.ascontiguousarray(tok).view(np.uint8).ravel()
        self.offs = np.ascontiguousarray(offs, dtype=np.uint64)
        self.R = len(self.offs) - 1
        self.h0 = np.ascontiguousarray(np.broadcast_to(np.asarray(h0, dtype=np.uint64), (self.R,)))
        self.d_tok = torch.from_numpy(np.concatenate([self.tok, np.zeros(16, np.uint8)])).cuda()
        self.d_offs = torch.from_numpy(self.offs.view(np.int64).copy()).cuda()
        self.d_h0 = torch.from_numpy(self.h0.view(np.int64).copy()).cuda()


def device_counts(p, x: Inputs, cols: int, shift: int = 1, stream=None, chains=False):
    """fi_epp_match_counts_device into a guarded buffer at a 2-byte offset `shift` -> (counts, nblocks[, chains])"""
    n = x.R * cols
    buf = torch.full((n + shift + 40,), GUARD, dtype=torch.int16, device="cuda")
    nb = torch.zeros(max(x.R, 1), dtype=torch.int32, device="cuda")
    ch = torch.zeros((max(x.R, 1), p.max_blocks), dtype=torch.int64, device="cuda") if chains else None
    s = stream or torch.cuda.current_stream()
    p.match_counts_device(x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), x.R, int(x.offs[-1]),
                          buf.data_ptr() + 2 * shift, nb.data_ptr(), ch.data_ptr() if chains else 0, s.cuda_stream)
    s.synchronize()
    raw = buf.cpu().numpy().view(np.uint16)
    assert (raw[:shift] == GUARD).all() and (raw[shift + n:] == GUARD).all(), "a store left the rows"
    out = (raw[shift:shift + n].reshape(x.R, cols).copy(), nb.cpu().numpy().view(np.uint32)[: x.R].copy())
    return out + (ch.cpu().numpy().view(np.uint64)[: x.R].copy(),) if chains else out


def check(p, o, x: Inputs, cols: int, shift: int = 1):
    """host and device calls equal the oracle (and each other) byte for byte; -> the matrix"""
    want, wnb = o.match_counts(x.tok, x.offs, x.h0)
    got, nb = p.match_counts(x.tok, x.offs, x.h0)
    assert got.shape == want.shape and np.array_equal(got, want), np.argwhere(got != want)[:5]
    assert np.array_equal(nb, wnb)
    dgot, dnb = device_counts(p, x, cols, shift)
    assert np.array_equal(dgot, want) and np.array_equal(dnb, wnb)
    return want


def _world(E, B, M, R, mode, lru, seed, shard=None, **kw):
    rng = np.random.default_rng(seed)
    tok, offs = MC.prompts(R, B, M, rng)
    if shard is not None:
        kw.update(endpoint_begin=shard[0], endpoint_count=shard[1])
    cfg = _cfg(E, B, M, R, mode, lru, **kw)
    p = EndpointPicker(cfg)
    o = CountsOracle(_cfg(E, B, M, R, mode, lru), shard=shard, track_removal=lru > 0)
    st = SV.tie_states(E, rng)
    p.update_endpoints(st)
    o.update_endpoints(st)
    x = Inputs(tok, offs, 0x5EED + seed)
    return rng, p, o, x


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [32, 64, 128, 96, 5])
@pytest.mark.parametrize("E", [37, 1000, 1024, 4096])
def test_counts_equal_the_oracle(mode, B, E):
    """SET / CLEAR with holes, then Adds through the device LRU that evict chain fronts (the PreRequest after a counts
    call), then removals; picks and ranked lists of the same handle agree with the matrix"""
    M, R = 48, 160
    rng, p, o, x = _world(E, B, M, R, mode, lru=2 * M, seed=E + B)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2):
        p.index_apply(ops)
        o.index_apply(ops)
    m = check(p, o, x, E, shift=1 + (E % 7))
    assert MC.unique_counts(m) > 3
    check_picks_against_matrix(p.pick_batch(x.tok, x.offs, x.h0), m)
    check_picks_against_matrix(p.pick_batch_ranked(x.tok, x.offs, x.h0, 16), m)
    for dest, _, _ in MC.add_batches(chains, nb, E, rng, batches=3):
        got, gnb, gch = p.match_counts(x.tok, x.offs, x.h0, want_chains=True)
        assert np.array_equal(got, o.match_counts(x.tok, x.offs, x.h0)[0]) and np.array_equal(gch, chains)
        p.index_add_chains_device(dest, 0, 0, gnb)  # the chains of the counts call just made
        o.index_add_chains(dest, chains, nb)
        check(p, o, x, E, shift=3)
    gone = rng.choice(E, size=min(5, E), replace=False)
    p.remove_endpoints(gone)
    o.remove_endpoints(gone)
    m = check(p, o, x, E, shift=0)
    check_picks_against_matrix(p.pick_batch_ranked(x.tok, x.offs, x.h0, 4), m)
    p.close()
    o.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [64, 96])
@pytest.mark.parametrize("E", [37, 1024])
def test_early_exit_and_long_prompts(mode, B, E):
    """lru_capacity 0 (hashing stops at each request's first uncached block) and prompts of up to 1 023 blocks; the
    host call with chains hashes whole chains, which equal fi_epp_hash_batch's"""
    M, R = 1023, 48
    rng, p, o, x = _world(E, B, M, R, mode, lru=0, seed=7)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    assert nb.max() == M
    top = int(np.argmax(nb))
    full = H.ops_array([(int(h), E - 1, abi.FI_OP_SET) for h in chains[top, :M]])  # one endpoint holds a whole chain
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2, holes=0.02) + [full]:
        p.index_apply(ops)
        o.index_apply(ops)
    m = check(p, o, x, E)
    assert m.max() == M
    got, gnb, gch = p.match_counts(x.tok, x.offs, x.h0, want_chains=True)
    hch, hnb = p.hash_batch(x.tok, x.offs, x.h0)
    assert np.array_equal(got, m) and np.array_equal(gnb, hnb) and np.array_equal(gch, hch)
    dm, dnb, dch = device_counts(p, x, E, chains=True)
    assert np.array_equal(dm, m) and np.array_equal(dnb, hnb) and np.array_equal(dch, hch)
    p.close()


@pytest.mark.parametrize("mode", MODES)
def test_capacity_change_resize_and_snapshot(mode):
    E, B, M, R = 300, 64, 32, 128
    rng, p, o, x = _world(E, B, M, R, mode, lru=3 * M, seed=11)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for dest, _, _ in MC.add_batches(chains, nb, E, rng, batches=2):
        p.index_add_chains(dest, chains, nb)
        o.index_add_chains(dest, chains, nb)
    check(p, o, x, E)
    eps = rng.choice(E, size=60, replace=False)
    caps = np.full(60, M, dtype=np.uint32)
    p.set_lru_capacities(eps, caps)
    o.set_lru_capacities(eps, caps)
    m = check(p, o, x, E)
    q = EndpointPicker(_cfg(E, B, M, R, mode, 3 * M))  # a snapshot load into another handle
    q.load_snapshot(p.save_snapshot())
    assert np.array_equal(q.match_counts(x.tok, x.offs, x.h0)[0], m)
    q.close()
    p.resize_pool(E + 100)  # grow: the rows widen, the new endpoints hold nothing
    got, _ = p.match_counts(x.tok, x.offs, x.h0)
    assert got.shape == (R, E + 100) and np.array_equal(got[:, :E], m) and not got[:, E:].any()
    dgot, _ = device_counts(p, x, E + 100, shift=5)
    assert np.array_equal(dgot, got)
    p.resize_pool(E - 77)  # shrink: the dropped endpoints' pairs leave, as a removal takes them
    o.remove_endpoints(np.arange(E - 77, E))
    want = o.match_counts(x.tok, x.offs, x.h0)[0][:, : E - 77]
    assert np.array_equal(p.match_counts(x.tok, x.offs, x.h0)[0], want)
    assert np.array_equal(device_counts(p, x, E - 77, shift=2)[0], want)
    p.close()
    o.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shard", [(0, 1), (3, 33), (34, 990), (1000, 24)])
def test_partial_pool_handles_match_the_shard_view(mode, shard):
    E, B, M, R = 1024, 64, 48, 128
    rng, p, o, x = _world(E, B, M, R, mode, lru=2 * M, seed=shard[0], shard=shard)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    for ops in MC.family_ops(chains, nb, E, rng, per_endpoint=2):
        p.index_apply(ops)
        o.index_apply(ops)
    for dest, _, _ in MC.add_batches(chains, nb, E, rng, batches=1):
        p.index_add_chains(dest, chains, nb)
        o.index_add_chains(dest, chains, nb)
    m = check(p, o, x, shard[1], shift=1)
    check_picks_against_matrix(p.pick_batch_ranked(x.tok, x.offs, x.h0, 8), m, shard[0])
    p.close()


def test_crafted_marker_hashes_and_collisions():
    """block hashes 0 and ~0 (the table's EMPTY / TOMB markers, which own fixed nodes) and chain keys whose home
    buckets are full of other keys"""
    E, B, M, R, slots = 64, 64, 16, 64, 1 << 12
    for mode in MODES:
        rng = np.random.default_rng(5)
        tok, offs = MC.prompts(R, B, M, rng)
        raw = np.ascontiguousarray(tok).view(np.uint8).ravel()
        h0 = np.full(R, 77, dtype=np.uint64)
        for r in range(3, R, 4):  # put a marker at block 1 or 2 of every fourth prompt
            n = min((int(offs[r + 1]) - int(offs[r])) // B, M)
            if n >= 3:
                blocks = [bytes(raw[int(offs[r]) + i * B: int(offs[r]) + (i + 1) * B]) for i in range(3)]
                h0[r] = craft.h0_for(blocks, 1 + (r // 4) % 2, craft.MARKERS[(r // 8) % 2])
        cfg = _cfg(E, B, M, R, mode, 0, index_slots=slots)
        p, o = EndpointPicker(cfg), CountsOracle(cfg)
        x = Inputs(tok, offs, h0)
        chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
        valid = np.arange(M)[None, :] < nb[:, None]
        assert (chains[valid] == 0).any() and (chains[valid] == np.uint64(2**64 - 1)).any()
        fill = []
        for h in chains[5:40:5, 0]:
            fill += [(k, int(rng.integers(0, E)), abi.FI_OP_SET) for k in collide.index_fillers_for(int(h), 6, slots, rng)]
        ops = [H.ops_array(fill)] + MC.family_ops(chains, nb, E, rng, per_endpoint=3)
        for a in ops:
            p.index_apply(a)
            o.index_apply(a)
        check(p, o, x, E, shift=7)
        p.close()


def test_stream_order_tickets_and_stats():
    """the device call runs behind work still queued on the caller's stream and behind pipelined batches in flight; it
    sees every op issued before it; afterwards a ticket submitted before it has lost its chains (S.9), and it counts
    as a pick call"""
    E, B, M, R = 256, 64, 64, 512
    rng, p, o, x = _world(E, B, M, R, abi.FI_MATCH_UPSTREAM, lru=2 * M, seed=9)
    chains, nb = o.hash_batch(x.tok, x.offs, x.h0)
    ops = MC.family_ops(chains, nb, E, rng, per_endpoint=3)
    p.index_apply(ops[0])
    o.index_apply(ops[0])
    d_out = torch.zeros((R, 2 * 16), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        t = p.pick_submit_ex(x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), R, int(x.offs[-1]),
                             d_out.data_ptr(), stream=s.cuda_stream)
        p.index_apply(ops[1])  # issued after the submit, before the counts call
        o.index_apply(ops[1])
        late = Inputs(x.tok, x.offs, x.h0)
        late.d_tok = torch.zeros_like(x.d_tok)
        torch.cuda._sleep(50_000_000)  # the prompts reach the buffer only after this
        late.d_tok.copy_(x.d_tok)
        p.reset_stats()
        p.set_profiling(True)
        got, gnb = device_counts(p, late, E, shift=1, stream=s)
    want, _ = o.match_counts(x.tok, x.offs, x.h0)
    assert np.array_equal(got, want)
    st = p.stats()
    assert st.pick_calls == 1 and st.requests == R and st.ms_match_pick > 0 and st.probed_blocks > 0
    p.set_profiling(False)
    with pytest.raises(FiEppError) as ei:
        p.index_add_submitted(t, np.zeros(R, np.uint32), gnb)
    assert ei.value.status == abi.FI_ERR_STATE
    p.close()


def test_errors_write_nothing():
    E, B, M, R = 40, 64, 16, 32
    rng, p, o, x = _world(E, B, M, R, abi.FI_MATCH_LPM, lru=0, seed=1, max_prompt_bytes=1 << 16)
    lib, h = p._lib, p._h
    counts = np.full((R, E), GUARD, dtype=np.uint16)
    nb = np.full(R, 7, dtype=np.uint32)
    args = (x.tok.ctypes.data, x.offs.ctypes.data, x.h0.ctypes.data)
    assert lib.fi_epp_match_counts(None, *args, R, counts.ctypes.data, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_counts(h, *args, R, None, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_counts(h, x.tok.ctypes.data, None, x.h0.ctypes.data, R, counts.ctypes.data, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_counts(h, x.tok.ctypes.data, x.offs.ctypes.data, None, R, counts.ctypes.data, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_match_counts_device(h, x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), R, 0, None, None,
                                          None, None) == abi.FI_ERR_INVALID
    big = Inputs(np.zeros(70000, np.uint8), np.array([0, 70000], np.uint64), 1)
    assert lib.fi_epp_match_counts(h, big.tok.ctypes.data, big.offs.ctypes.data, big.h0.ctypes.data, 1,
                                   counts.ctypes.data, nb.ctypes.data, None) == abi.FI_ERR_CAPACITY
    offs33 = np.zeros(R + 2, dtype=np.uint64)
    h033 = np.zeros(R + 1, dtype=np.uint64)
    assert lib.fi_epp_match_counts(h, x.tok.ctypes.data, offs33.ctypes.data, h033.ctypes.data, R + 1,
                                   counts.ctypes.data, nb.ctypes.data, None) == abi.FI_ERR_CAPACITY
    assert lib.fi_epp_match_counts_device(h, x.d_tok.data_ptr(), x.d_offs.data_ptr(), x.d_h0.data_ptr(), R + 1, 0,
                                          C.c_void_p(8), None, None, None) == abi.FI_ERR_CAPACITY
    assert (counts == GUARD).all() and (nb == 7).all()
    assert lib.fi_epp_match_counts(h, *args, 0, None, None, None) == abi.FI_OK
    assert lib.fi_epp_match_counts_device(h, None, x.d_offs.data_ptr(), None, 0, 0, None, None, None, None) == abi.FI_OK
    assert p.stats().pick_calls == 0
    p.close()


def test_full_size_batch():
    """max_batch 16 384 requests over 1 024 endpoints (32 MiB of counts), bit-exact"""
    wl = synth.Workload(R=16384, E=1024, T=1024, lru_capacity=160, groups_per_endpoint=4, max_blocks=64, holes=True)
    cfg = H.config_for(wl, profiles=PROFILES)
    p, o = EndpointPicker(cfg), CountsOracle(cfg)
    for ops in wl.index_ops():
        p.index_apply(ops)
        o.index_apply(ops)
    tok, offs = wl.prompts()
    x = Inputs(tok, offs, wl.h0)
    m = check(p, o, x, wl.E, shift=3)
    assert (m > 0).sum() > wl.R
    p.close()
    o.close()
