"""GPU (-m gpu): chains of more than 1023 blocks (max_blocks up to FI_EPP_MAX_BLOCKS = 4095), bit-exact against the
CPU oracle.

A handle with max_blocks > 1023 runs match_window_kernel (DESIGN.md §4.9): a request's chain is staged, resolved to
index nodes and counted 1024 blocks (one window) at a time into 12 bit-planes.  The cases put the events the window
loop carries across a boundary at W - 1, W and W + 1 for W = 1024, 2048 and 3072:
- the first block no endpoint holds (the UPSTREAM walk ends there; later windows are not read);
- an endpoint's LPM break, and the block at which every endpoint has dropped out while the index still holds the
  chain (the window staged for the walk goes unread);
- cached runs inserted in chain order (block 0 of a window continues the previous window's run of nodes) and in
  shuffled order (it is looked up in the table).
One endpoint holds request 0's whole chain: its count is M, 4095 sets all 12 planes.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, make_config, subset_bitsets
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from oracle import epp_oracle as eo
from tests import helpers as H
from tests.counts_oracle import CountsOracle
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
UP, LPM = abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM
WEIGHTED = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]
WITH_LORA = [{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5), (Q, 5)]}]
W = 1024
BOUNDARIES = [W - 1, W, W + 1, 2 * W - 1, 2 * W, 2 * W + 1, 3 * W - 1, 3 * W, 3 * W + 1]


def _prompts(M, R, B=64, seed=0):
    """R prompts of M + 1 whole blocks and a partial one (n is capped at M); odd requests share their first M / 2
    blocks with the request before them"""
    rng = np.random.default_rng(seed)
    T = (M + 1) * B + B // 2
    tok = rng.integers(0, 256, size=(R, T), dtype=np.uint8)
    for r in range(1, R, 2):
        tok[r, : (M // 2) * B] = tok[r - 1, : (M // 2) * B]
    offs = np.arange(R + 1, dtype=np.uint64) * T
    h0 = rng.integers(0, 2**63, size=R, dtype=np.uint64)
    return tok.reshape(-1), offs, h0


def _sets(trip_ranges):
    """SET ops of (endpoint, hashes) pairs, each in chain order"""
    ops = [H.ops_array([(int(h), e, abi.FI_OP_SET) for h in hs]) for e, hs in trip_ranges if len(hs)]
    return np.concatenate(ops)


def _index(chains, M, E, seed=1):
    """Request 0: its whole chain on endpoint E // 2.  Request r > 0, with cut c = a boundary (or M for some):
    endpoint a_r holds blocks [0, c); endpoint b_r holds [0, M) but block c (its LPM break at c, the UPSTREAM walk
    goes on where a_r holds c or past it); for every fourth request endpoint d_r holds only [c, M), so that in LPM
    every endpoint has dropped out at c while the index still holds the rest of the chain."""
    rng = np.random.default_rng(seed)
    R = chains.shape[0]
    cuts = [c for c in BOUNDARIES if c < M] + [M - 1, M]
    parts = [(E // 2, chains[0, :M])]
    for r in range(1, R):
        c = cuts[r % len(cuts)]
        a, b, d = (int(x) for x in rng.choice(E, size=3, replace=E < 3))
        if r % 3 == 0:
            parts.append((a, chains[r, :c]))
        if r % 3 != 2:
            parts.append((b, np.concatenate([chains[r, :c], chains[r, c + 1:M]])))
        if r % 4 == 1:
            parts.append((d, chains[r, c:M]))
    return _sets(parts), cuts


def _slots(ops):
    keys = len(np.unique(ops["hash"]))
    s = 1 << 14
    while s < 2 * keys:
        s *= 2
    return s


def _cfg(E, M, R, offs, mode, B=64, **kw):
    kw.setdefault("profiles", WEIGHTED)
    return make_config(num_endpoints=E, block_bytes=B, max_blocks=M, max_batch=R, max_prompt_bytes=int(offs[-1]),
                       match_mode=mode, **kw)


def _states(E, seed=3):
    rng = np.random.default_rng(seed)
    return H.states_array(E, kv=rng.random(E), queue=rng.integers(0, 9, size=E))


def _same(got, want, tag):
    assert H.picks_equal(got, want), tag + "\n" + H.describe_diff(got, want)


def _pair(cfg, st, ops_list, oracle=eo.Oracle):
    g, o = EndpointPicker(cfg), oracle(cfg)
    for x in (g, o):
        x.update_endpoints(st)
        for ops in ops_list:
            x.index_apply(ops)
    return g, o


def _case(M, E, R=48, B=64, seed=0):
    tok, offs, h0 = _prompts(M, R, B=B, seed=seed)
    probe = eo.Oracle(make_config(num_endpoints=1, block_bytes=B, max_blocks=M, max_batch=R,
                                  max_prompt_bytes=int(offs[-1])))
    chains, nb = probe.hash_batch(tok, offs, h0)
    probe.close()
    assert (nb == M).all()
    ops, cuts = _index(chains, M, E)
    return tok, offs, h0, chains, ops


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1024, 1031, 2048, 4095])
@pytest.mark.parametrize("E", [8, 100, 1024])
def test_window_pick_parity(E, M):
    """single picks and chains in both match modes; the whole-chain request counts M on its endpoint"""
    tok, offs, h0, chains, ops = _case(M, E)
    st = _states(E)
    for mode in (UP, LPM):
        g, o = _pair(_cfg(E, M, len(h0), offs, mode, index_slots=_slots(ops)), st, [ops])
        got, gch = g.pick_batch(tok, offs, h0, want_chains=True)
        want, wch = o.pick_batch(tok, offs, h0, want_chains=True)
        g.close()
        o.close()
        tag = f"E={E} M={M} mode={mode}"
        assert np.array_equal(gch, wch), tag
        _same(got, want, tag)
        mb = want[:, 0]["match_blocks"]
        assert (want[:, 0]["n_blocks"] == M).all()
        assert mb[0] == M and want[0, 0]["endpoint"] == E // 2, tag
        assert (mb >= W - 1).sum() >= 3, tag  # counts at and past the first window boundary


@pytest.mark.parametrize("mode", [UP, LPM])
def test_window_counts_at_every_boundary(mode):
    """fi_epp_match_counts (u16) of every endpoint against the oracle: counts of 4095, and every cut of BOUNDARIES on
    either side of each window boundary, with the index in chain order and shuffled"""
    M, E = 4095, 100
    tok, offs, h0, chains, ops = _case(M, E, R=64)
    st = _states(E)
    for shuffled in (False, True):
        o_ops = ops[np.random.default_rng(9).permutation(len(ops))] if shuffled else ops
        cfg = _cfg(E, M, len(h0), offs, mode, index_slots=_slots(ops))
        g, o = _pair(cfg, st, [o_ops], oracle=CountsOracle)
        got, _ = g.match_counts(tok, offs, h0)
        want, _ = o.match_counts(tok, offs, h0)
        pg, po = g.pick_batch(tok, offs, h0), eo.Oracle.pick_batch(o, tok, offs, h0)
        g.close()
        o.close()
        tag = f"mode={mode} shuffled={shuffled}"
        assert got.dtype == np.uint16 and np.array_equal(got, want), tag
        _same(pg, po, tag)
        assert want[0, E // 2] == 4095
        vals = set(int(v) for v in np.unique(want))
        assert {W - 1, W, W + 1, 2 * W, 3 * W + 1} <= vals, (tag, sorted(vals)[-20:])


def test_window_lora_ranked_subset():
    """the LoRA variant, ranked k = 16 and per-request subsets over 4095-block chains"""
    M, E = 4095, 100
    tok, offs, h0, chains, ops = _case(M, E, R=32)
    rng = np.random.default_rng(11)
    st = _states(E)
    lo = np.zeros(E, dtype=abi.lora_dtype())
    lo["endpoint"] = np.arange(E)
    for e in range(E):
        na = int(rng.integers(0, 3))
        lo[e]["n_active"], lo[e]["max_active"] = na, int(rng.integers(0, 4))
        lo[e]["active"][:na] = rng.permutation(6)[:na] + 1000
    adapters = (rng.integers(0, 7, size=len(h0)) + 1000).astype(np.uint64)
    subsets = [np.flatnonzero(rng.random(E) < 0.3) for _ in range(len(h0))]
    subsets[0] = np.array([E // 2, 3])
    for mode in (UP, LPM):
        cfg = _cfg(E, M, len(h0), offs, mode, index_slots=_slots(ops), profiles=WITH_LORA)
        g, o = _pair(cfg, st, [ops], oracle=ExtOracle)
        g.update_endpoints_lora(lo)
        o.update_endpoints_lora(lo)
        _same(g.pick_batch(tok, offs, h0, adapters=adapters), o.pick_batch(tok, offs, h0, adapters=adapters), "lora")
        _same(g.pick_batch_ranked(tok, offs, h0, 16, adapters=adapters),
              o.pick_batch_ranked(tok, offs, h0, 16, adapters=adapters), "ranked")
        sb = subset_bitsets(subsets, E)
        got = g.pick_batch_subset(tok, offs, h0, sb, k=4, adapters=adapters)
        want = o.pick_batch_subset(tok, offs, h0, sb, k=4, adapters=adapters)
        _same(got, want, "subset")
        assert want[0, 0, 0]["match_blocks"] == M
        g.close()
        o.close()


def test_window_pd_threshold():
    """PD at n = 4095: the prefill profile stands iff (1 - hit) * len >= threshold; thresholds split the batch"""
    M, E = 4095, 64
    tok, offs, h0, chains, ops = _case(M, E, R=32)
    st = H.states_array(E, kv=np.linspace(0, 0.9, E), queue=np.arange(E) % 4,
                        roles=np.where(np.arange(E) % 2 == 0, abi.FI_ROLE_PREFILLER, abi.FI_ROLE_DECODER))
    profiles = [{"name": "prefill", "role_mask": abi.FI_ROLE_PREFILLER, "scorers": [(P, 100), (Q, 5)]},
                {"name": "decode", "role_mask": abi.FI_ROLE_DECODER, "scorers": [(P, 100), (K, 5)]}]
    seen = set()
    length = float(offs[1] - offs[0])
    for thr in (0.0, 0.3 * length, 0.7 * length, 1e12):
        cfg = _cfg(E, M, len(h0), offs, UP, index_slots=_slots(ops), profiles=profiles,
                   pd={"decode": 1, "prefill": 0, "threshold": thr})
        g, o = _pair(cfg, st, [ops])
        got, want = g.pick_batch(tok, offs, h0), o.pick_batch(tok, offs, h0)
        g.close()
        o.close()
        _same(got, want, f"threshold {thr}")
        seen.add(float((want[:, 0]["endpoint"] == abi.FI_NO_ENDPOINT).mean()))
    assert 0.0 in seen and 1.0 in seen and any(0.0 < s < 1.0 for s in seen)


def _device_pick(g, tok, offs, h0):
    """the stream-ordered device pick (host-buffer picks of large batches are fed in slices, each a smaller batch)"""
    import torch

    R = len(h0)
    d_tok = torch.from_numpy(np.ascontiguousarray(tok)).cuda()
    d_off = torch.from_numpy(offs.view(np.int64).copy()).cuda()
    d_h0 = torch.from_numpy(h0.view(np.int64).copy()).cuda()
    d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    g.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_out.data_ptr(), 0,
                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)


@pytest.mark.parametrize("B", [64, 40])
def test_window_early_exit_and_block_sizes(B):
    """lru_capacity = 0 and no chains_out: hashing stops each long request after its first uncached block, so fewer
    blocks are hashed than the prompts hold, and the picks are those of the whole chains.  Early exit runs in half-SM
    hashing tiles, so the device pick gets 48 prompts of 4095 blocks and 8 500 one-block prompts.  B = 40 is not a multiple of
    32 (hash_generic: no early exit)."""
    M, E, short = 4095, 100, 8500
    tok, offs, h0, chains, ops = _case(M, E, R=48, B=B)
    rng = np.random.default_rng(21)
    tok = np.concatenate([tok, rng.integers(0, 256, size=short * B, dtype=np.uint8)])
    offs = np.concatenate([offs, offs[-1] + B * np.arange(1, short + 1, dtype=np.uint64)])
    h0 = np.concatenate([h0, rng.integers(0, 2**63, size=short, dtype=np.uint64)])
    for mode in (UP, LPM):
        g, o = _pair(_cfg(E, M, len(h0), offs, mode, B=B, index_slots=_slots(ops)), _states(E), [ops])
        g.set_profiling(True)
        g.reset_stats()
        got = _device_pick(g, tok, offs, h0)
        hashed = g.stats().hashed_blocks
        want = o.pick_batch(tok, offs, h0)
        g.close()
        o.close()
        _same(got, want, f"B={B} mode={mode}")
        total = int(want[:, 0]["n_blocks"].sum())
        assert total == 48 * M + short
        if B % 32 == 0:
            assert 0 < hashed < total, (hashed, total)


def test_window_submit_and_add_submitted_evict():
    """fi_epp_pick_submit_ex + fi_epp_index_add_submitted on the device LRU with 4095-key Adds whose LRUs evict
    (capacity 6000 per endpoint), against the oracle's picks + index_add_chains, step by step"""
    import torch

    M, E, R = 4095, 16, 24
    cap = 6000
    tok, offs, h0, chains, ops = _case(M, E, R=R)
    cfg = _cfg(E, M, R, offs, UP, index_slots=1 << 18, lru_capacity=cap)
    g, o = EndpointPicker(cfg), eo.Oracle(cfg)
    st = _states(E)
    g.update_endpoints(st)
    o.update_endpoints(st)
    rng = np.random.default_rng(4)
    s = torch.cuda.current_stream().cuda_stream
    for step in range(4):
        sel = rng.permutation(R)
        tk = np.ascontiguousarray(tok.reshape(R, -1)[sel]).reshape(-1)
        hh = np.ascontiguousarray(h0[sel])
        d_tok = torch.from_numpy(tk).cuda()
        d_off = torch.from_numpy(offs.view(np.int64).copy()).cuda()
        d_h0 = torch.from_numpy(hh.view(np.int64)).cuda()
        d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
        t = g.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tk.nbytes, d_out.data_ptr(), stream=s)
        g.pick_wait_batch(t, s)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        want, wch = o.pick_batch(tk, offs, hh, want_chains=True)
        _same(got, want, f"step {step}")
        eps = want[:, 0]["endpoint"].copy()
        swap = rng.random(R) < 0.5  # spread the Adds over the pool
        eps[swap] = rng.integers(0, E, size=int(swap.sum()))
        nb = want[:, 0]["n_blocks"].astype(np.uint32)
        g.index_add_submitted(t, eps, nb)
        o.index_add_chains(eps, wch, nb)
    g.index_sync()
    for e in range(E):
        assert len(g.lru_dump(e)) <= cap
    assert any(len(g.lru_dump(e)) == cap for e in range(E))  # some LRU evicted
    final = g.pick_batch(tok, offs, h0)
    _same(final, o.pick_batch(tok, offs, h0), "after the Adds")
    g.close()
    o.close()


@pytest.mark.parametrize("R", [2000, 40000, 70000])
def test_window_sliced_host_feed_every_tile_shape(R):
    """Host-buffer picks feed the batch in 8 slices once it holds 8 MiB of prompts, and hash_chain chooses its tile
    from each slice's size (on a 132-SM H100): 32 requests per SM for R = 2 000, 64 per SM for R = 40 000 and
    half-SM tiles for R = 70 000.  48 prompts of 4095 blocks (12 MiB) are spread over the batch, the rest are one
    block each.  Picks of every request against the oracle, with early-exit hashing (no chains_out), and at
    R = 2 000 the chains too."""
    M, E, L = 4095, 100, 48
    ltok, loffs, lh0, chains, ops = _case(M, E, R=L)
    lsz = int(loffs[1] - loffs[0])
    rng = np.random.default_rng(R)
    where = np.linspace(0, R - 1, L).astype(np.int64)
    lens = np.full(R, 64 + 10, dtype=np.uint64)
    lens[where] = lsz
    offs = np.zeros(R + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    tok = rng.integers(0, 256, size=int(offs[-1]), dtype=np.uint8)
    for i, r in enumerate(where):
        tok[int(offs[r]):int(offs[r + 1])] = ltok[i * lsz:(i + 1) * lsz]
    h0 = rng.integers(0, 2**63, size=R, dtype=np.uint64)
    h0[where] = lh0
    assert offs[-1] >= 8 << 20
    g, o = _pair(_cfg(E, M, R, offs, UP, index_slots=_slots(ops)), _states(E), [ops])
    got = g.pick_batch(tok, offs, h0)
    want = o.pick_batch(tok, offs, h0)
    _same(got, want, f"R={R}")
    assert (want[where, 0]["n_blocks"] == M).all() and (want[where, 0]["match_blocks"] >= W - 1).sum() >= 3
    if R == 2000:
        got, gch = g.pick_batch(tok, offs, h0, want_chains=True)
        _same(got, want, "with chains")
        assert np.array_equal(gch[where], chains)
        assert not gch[np.arange(M)[None, :] >= got[:, 0]["n_blocks"][:, None]].any()
    g.close()
    o.close()


def test_window_snapshot_round_trip():
    """save a long handle's index and LRUs, load them into a fresh handle: the same blob and the same picks"""
    M, E, R = 4095, 32, 24
    tok, offs, h0, chains, ops = _case(M, E, R=R)
    cfg = _cfg(E, M, R, offs, LPM, index_slots=1 << 18, lru_capacity=2 * M)
    a = EndpointPicker(cfg)
    a.update_endpoints(_states(E))
    picks = a.pick_batch(tok, offs, h0, want_chains=True)
    a.index_add_chains(np.arange(R) % E, picks[1], picks[0][:, 0]["n_blocks"])  # one chain per endpoint
    blob = a.save_snapshot()
    b = EndpointPicker(cfg)
    b.update_endpoints(_states(E))
    b.load_snapshot(blob)
    assert b.save_snapshot().tobytes() == blob.tobytes()
    pa, pb = a.pick_batch(tok, offs, h0), b.pick_batch(tok, offs, h0)
    _same(pb, pa, "loaded")
    assert (pa[:, 0]["match_blocks"] == M).all()
    a.close()
    b.close()


@pytest.mark.parametrize("b,c", [(0, 40), (33, 60), (64, 36)])
def test_window_sub_range_handle(b, c):
    """a handle over endpoints [b, b + c) of a 100-endpoint pool against the oracle's shard view"""
    M, E = 4095, 100
    tok, offs, h0, chains, ops = _case(M, E, R=32)
    for mode in (UP, LPM):
        cfg = _cfg(E, M, len(h0), offs, mode, index_slots=_slots(ops))
        cfg.endpoint_begin, cfg.endpoint_count = b, c
        g, o = EndpointPicker(cfg), ExtOracle(cfg, shard=(b, c))
        for x in (g, o):
            x.update_endpoints(_states(E))
            x.index_apply(ops)
        _same(g.pick_batch(tok, offs, h0), o.pick_batch(tok, offs, h0), f"[{b}, {b + c}) mode={mode}")
        _same(g.pick_batch_ranked(tok, offs, h0, 5), o.pick_batch_ranked(tok, offs, h0, 5), "ranked")
        g.close()
        o.close()


def test_comm_init_refused_on_long_handles():
    cfg = make_config(num_endpoints=8, block_bytes=64, max_blocks=1024, max_batch=4)
    g = EndpointPicker(cfg)
    with pytest.raises(FiEppError) as ei:
        g.comm_init(bytes(abi.FI_EPP_UNIQUE_ID_BYTES), 0, 1)
    assert ei.value.status == abi.FI_ERR_STATE
    g.close()
    cfg = make_config(num_endpoints=8, block_bytes=64, max_blocks=1023, max_batch=4)
    g = EndpointPicker(cfg)
    g.comm_init(bytes(abi.FI_EPP_UNIQUE_ID_BYTES), 0, 1)  # one rank: no communicator is needed
    g.close()


def test_create_bounds():
    for m, ok in ((4095, True), (4096, False), (0, False)):
        cfg = make_config(num_endpoints=4, block_bytes=64, max_blocks=m, max_batch=2)
        if ok:
            EndpointPicker(cfg).close()
        else:
            with pytest.raises(FiEppError) as ei:
                EndpointPicker(cfg)
            assert ei.value.status == abi.FI_ERR_INVALID
