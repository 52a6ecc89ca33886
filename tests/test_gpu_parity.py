"""GPU (-m gpu): parity of the sm_90a path against the CPU oracle, through the C ABI.

Bit-exact for every integer/byte/index output (block hashes, index membership,
endpoint, match length) and for the fp64 score (compared as raw 64-bit patterns —
tolerance 0: both sides do the same IEEE-754 round-to-nearest mul/add/div sequence).
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, FiEppError, make_config, synth
from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import helpers as H

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q


def _pair(cfg):
    return EndpointPicker(cfg), eo.Oracle(cfg)


def _load(wl, gpu, cpu, states=None):
    st = wl.endpoint_states() if states is None else states
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for ops in wl.index_ops():
        gpu.index_apply(ops)
        cpu.index_apply(ops)


# ---------------------------------------------------------------------------------------
# block hashing
# ---------------------------------------------------------------------------------------
def test_hash_golden_vectors():
    g = H.golden()
    h0 = int(g["h0"], 16)
    for case in g["chains"]:
        cfg = make_config(num_endpoints=1, block_bytes=case["block_bytes"], max_blocks=case["max_blocks"], max_batch=4,
                          max_prompt_bytes=1 << 16)
        with EndpointPicker(cfg) as gpu:
            data, offs = H.pack_prompts([bytes.fromhex(case["hex"])])
            chains, nb = gpu.hash_batch(data, offs, h0)
            want = [int(x, 16) for x in case["chain"]]
            assert nb[0] == len(want)
            assert list(chains[0, : nb[0]]) == want, case["block_bytes"]
            assert not chains[0, nb[0]:].any()


@pytest.mark.parametrize("B", [64, 32, 128, 96, 5, 16, 7, 40])
def test_hash_parity_ragged_unaligned(B):
    rng = np.random.default_rng(B)
    M = 24
    lens = [0, 1, B - 1, B, B + 1, 2 * B, M * B, M * B + 3, (M + 5) * B, 3 * B + B // 2]
    lens += [int(x) for x in rng.integers(0, (M + 3) * B, size=54)]
    blobs = [rng.integers(0, 256, size=n, dtype=np.uint8).tobytes() for n in lens]  # offsets end up at every alignment
    data, offs = H.pack_prompts(blobs)
    cfg = make_config(num_endpoints=1, block_bytes=B, max_blocks=M, max_batch=len(blobs), max_prompt_bytes=len(data))
    gpu, cpu = _pair(cfg)
    h0 = rng.integers(0, 2**63, size=len(blobs), dtype=np.uint64)
    gc, gn = gpu.hash_batch(data, offs, h0)
    wc, wn = cpu.hash_batch(data, offs, h0)
    assert np.array_equal(gn, wn)
    assert np.array_equal(gc, wc)
    gpu.close()


def test_hash_token_prompts_aligned_fast_path():
    wl = H.small_workload(R=300, T=2048, max_blocks=128)
    cfg = H.config_for(wl)
    gpu, cpu = _pair(cfg)
    tok, offs = wl.prompts()
    gc, gn = gpu.hash_batch(tok, offs, wl.h0)
    wc, wn = cpu.hash_batch(tok, offs, wl.h0)
    assert np.array_equal(gn, wn) and np.array_equal(gc, wc)
    # prefix property: requests of the same group share the chain up to their shared length
    groups, shared = wl.request_params()
    i, j = 0, None
    for j in range(1, wl.R):
        if groups[j] == groups[0] and shared[j] and shared[0]:
            k = min(shared[0], shared[j]) // wl.block_tokens
            assert np.array_equal(gc[0, :k], gc[j, :k])
            break
    gpu.close()


# ---------------------------------------------------------------------------------------
# index
# ---------------------------------------------------------------------------------------
def test_index_set_clear_sequences_match_oracle():
    rng = np.random.default_rng(11)
    E = 70
    cfg = make_config(num_endpoints=E, max_batch=8, index_slots=4096)
    gpu, cpu = _pair(cfg)
    universe = np.concatenate([rng.integers(1, 2**63, size=298, dtype=np.uint64),
                               np.array([0, 0xFFFFFFFFFFFFFFFF], dtype=np.uint64)])  # incl. the sentinel values
    for step in range(12):
        n = 700
        ops = np.zeros(n, dtype=H.OP_DTYPE)
        ops["hash"] = universe[rng.integers(0, len(universe), size=n)]
        ops["endpoint"] = rng.integers(0, E, size=n)
        ops["op"] = rng.choice([abi.FI_OP_SET, abi.FI_OP_SET, abi.FI_OP_CLEAR], size=n)  # conflicts within a call
        gpu.index_apply(ops)
        cpu.index_apply(ops)
        q = np.zeros(len(universe) * E, dtype=H.OP_DTYPE)
        q["hash"] = np.repeat(universe, E)
        q["endpoint"] = np.tile(np.arange(E, dtype=np.uint32), len(universe))
        got = gpu.index_contains(q)
        want = np.array([cpu.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
        assert np.array_equal(got, want), f"step {step}: {int((got != want).sum())} memberships differ"
    gpu.close()


def test_index_tombstones_trigger_rebuild_and_stay_exact():
    E = 16
    cfg = make_config(num_endpoints=E, max_batch=8, index_slots=256)
    gpu, cpu = _pair(cfg)
    live = []
    nxt = 1
    for round_ in range(40):
        # retire the oldest 20 hashes, add 20 new ones: keys only ever become tombstones
        ops = []
        for h in live[:20]:
            ops.append((h, 3, abi.FI_OP_CLEAR))
        live = live[20:]
        for _ in range(20):
            ops.append((nxt, 3, abi.FI_OP_SET))
            live.append(nxt)
            nxt += 1
        arr = H.ops_array(ops)
        gpu.index_apply(arr)
        cpu.index_apply(arr)
    st = gpu.index_stats()
    assert st.rebuilds >= 1, "800 retired keys in a 256-slot table must have forced a rebuild"
    assert st.used - st.tombstones == len(live)
    q = H.ops_array([(h, 3, 0) for h in range(1, nxt)])
    got = gpu.index_contains(q)
    want = np.array([cpu.index_contains(3, h) for h in range(1, nxt)], dtype=np.uint8)
    assert np.array_equal(got, want)
    gpu.close()


def test_index_overflow_is_reported_not_silent():
    cfg = make_config(num_endpoints=4, max_batch=8, index_slots=64)
    gpu = EndpointPicker(cfg)
    ops = H.ops_array([(h, 1, abi.FI_OP_SET) for h in range(1, 200)])
    with pytest.raises(Exception) as ei:
        gpu.index_apply(ops)
        gpu.index_sync()
        gpu.index_apply(ops[:1])
    assert "index" in str(ei.value)
    gpu.close()


# ---------------------------------------------------------------------------------------
# match + score + pick
# ---------------------------------------------------------------------------------------
WEIGHTED = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]


@pytest.mark.parametrize("E", [1, 8, 33, 64, 100, 256, 500, 1024, 2048, 4096])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("holes", [False, True])
def test_pick_parity_over_pool_sizes(E, mode, holes):
    wl = H.small_workload(E=E, R=160, holes=holes, lru_capacity=300)
    cfg = H.config_for(wl, profiles=WEIGHTED, match_mode=mode)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    got, gch = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
    want, wch = cpu.pick_batch(tok, offs, wl.h0, want_chains=True)
    assert np.array_equal(gch, wch)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    if E >= 8:
        assert (want["match_blocks"] > 0).mean() > 0.3  # the case really exercises prefix hits
    gpu.close()


@pytest.mark.parametrize("scorers", [
    [(P, 100)], [(K, 100)], [(Q, 100)], [(K, 3), (P, 50), (Q, 11)], [(Q, 1), (K, 1), (P, 1)], [(P, 0), (K, 5)],
    [(P, 100), (P, 1), (K, 2), (Q, 3)],
])
def test_pick_parity_over_scorer_mixes(scorers):
    wl = H.small_workload(E=200, R=200)
    cfg = H.config_for(wl, profiles=[{"name": "default", "scorers": scorers}])
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    got = gpu.pick_batch(tok, offs, wl.h0)
    want = cpu.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    gpu.close()


def test_pick_ties_dead_endpoints_and_empty_pool():
    wl = H.small_workload(E=96, R=64)
    cfg = H.config_for(wl, profiles=[{"name": "default", "scorers": [(P, 100), (Q, 5)]}])
    tok, offs = wl.prompts()
    for alive_fn in (lambda e: e % 3 != 0, lambda e: e >= 64, lambda e: e < 0):
        gpu, cpu = _pair(cfg)
        st = wl.endpoint_states()
        st["flags"] = np.where(alive_fn(np.arange(wl.E)), abi.FI_ENDPOINT_ALIVE, 0)
        st["queue_depth"] = 4  # all equal → queue score 1.0 everywhere → mass ties → the requests' rotations decide
        _load(wl, gpu, cpu, states=st)
        got = gpu.pick_batch(tok, offs, wl.h0)
        want = cpu.pick_batch(tok, offs, wl.h0)
        assert H.picks_equal(got, want), H.describe_diff(got, want)
        gpu.close()
    assert (want["endpoint"] == abi.FI_NO_ENDPOINT).all()


def test_pick_pd_profiles_and_threshold():
    wl = H.small_workload(E=128, R=200, pd=True)
    profiles, _ = synth.baseline_profiles(5)
    tok, offs = wl.prompts()
    for thr in (0.0, 600.0, 1500.0, 1e9):
        cfg = H.config_for(wl, profiles=profiles, pd={"decode": 1, "prefill": 0, "threshold": thr})
        gpu, cpu = _pair(cfg)
        _load(wl, gpu, cpu)
        got = gpu.pick_batch(tok, offs, wl.h0)
        want = cpu.pick_batch(tok, offs, wl.h0)
        assert H.picks_equal(got, want), H.describe_diff(got, want)
        gpu.close()
        skipped = (want[:, 0]["endpoint"] == abi.FI_NO_ENDPOINT).mean()
        if thr == 0.0:
            assert skipped == 0.0
            assert (want[:, 0]["endpoint"] < 64).all() and (want[:, 1]["endpoint"] >= 64).all()  # role filters
        if thr == 1e9:
            assert skipped == 1.0


def test_pick_ragged_short_and_truncated_prompts():
    wl = H.small_workload(E=64, R=64, T=1024, max_blocks=16)  # 64 blocks of text, capped at 16
    cfg = H.config_for(wl, profiles=WEIGHTED, max_prompt_bytes=1 << 20)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, _ = wl.prompts()
    rng = np.random.default_rng(1)
    blobs = []
    for r in range(wl.R):
        n_tok = int(rng.choice([0, 3, 15, 16, 17, 100, 255, 256, 257, 1024]))
        blobs.append(tok[r, :n_tok].tobytes() + bytes(int(rng.integers(0, 4))))  # + ragged tail bytes
    data, offs = H.pack_prompts(blobs)
    got, gch = gpu.pick_batch(data, offs, wl.h0, want_chains=True)
    want, wch = cpu.pick_batch(data, offs, wl.h0, want_chains=True)
    assert np.array_equal(gch, wch)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    gpu.close()


def test_pick_reference_block_size_5_ascii():
    """The reference's own config: blockSize 5 over prompt text (strategy.go:57)."""
    rng = np.random.default_rng(9)
    E, R = 8, 64
    cfg = make_config(num_endpoints=E, block_bytes=5, max_blocks=256, max_batch=R, max_prompt_bytes=1 << 20)
    gpu, cpu = _pair(cfg)
    st = H.states_array(E)
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    alphabet = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz ,.", dtype=np.uint8)
    system = [alphabet[rng.integers(0, len(alphabet), size=400)].tobytes() for _ in range(4)]
    blobs = [system[int(rng.integers(0, 4))][: int(rng.integers(50, 400))] + alphabet[rng.integers(0, len(alphabet), size=int(rng.integers(0, 1500)))].tobytes()
             for _ in range(R)]
    data, offs = H.pack_prompts(blobs)
    h0 = synth.xxh64_py(b"meta-llama/Llama-3-8B")
    # warm the index the way upstream does: route, then Add(chain, picked endpoint)
    chains, nb = cpu.hash_batch(data, offs, h0)
    for r in range(0, R, 2):
        e = int(rng.integers(0, E))
        ops = H.ops_array([(int(h), e, abi.FI_OP_SET) for h in chains[r, : nb[r]]])
        gpu.index_apply(ops)
        cpu.index_apply(ops)
    got, gch = gpu.pick_batch(data, offs, h0, want_chains=True)
    want, wch = cpu.pick_batch(data, offs, h0, want_chains=True)
    assert np.array_equal(gch, wch)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    assert (want["match_blocks"] > 0).sum() >= R // 2
    gpu.close()


@pytest.mark.parametrize("device_lru", [0, 1])
def test_lru_add_chain_path_matches_oracle(device_lru):
    """Post-pick index maintenance (upstream PreRequest → indexer.Add), one chain per call, through the host LRU
    and through the device-resident LRU."""
    wl = H.small_workload(E=24, R=96, lru_capacity=0)
    cfg = H.config_for(wl, profiles=WEIGHTED, lru_capacity=400, index_slots=1 << 16)  # ~12 chains/endpoint: steady eviction
    gpu, cpu = _pair(cfg)
    gpu.set_option("device_lru", device_lru)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for batch in range(6):
        tok, offs = wl.prompts(batch=batch)
        got, gch = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        want, wch = cpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        assert np.array_equal(gch, wch)
        assert H.picks_equal(got, want), f"batch {batch}\n" + H.describe_diff(got, want)
        for r in range(wl.R):
            e = int(want[r, 0]["endpoint"])
            n = int(want[r, 0]["n_blocks"])
            gpu.index_add_chain(e, gch[r, :n])
            cpu.index_add_chain(e, wch[r, :n])
    assert (want["match_blocks"] > 0).any()
    stx = gpu.index_stats()
    assert stx.lru_entries <= 24 * 400 and stx.tombstones > 0  # evictions really happened
    gpu.close()


def test_device_resident_path_equals_host_path():
    import torch

    wl = H.small_workload(E=256, R=512, T=1024, max_blocks=64)
    cfg = H.config_for(wl, profiles=WEIGHTED)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    want = cpu.pick_batch(tok, offs, wl.h0)
    host = gpu.pick_batch(tok, offs, wl.h0)
    d_tok = torch.from_numpy(tok.view(np.int32)).cuda()
    d_off = torch.from_numpy(offs.view(np.int64)).cuda()
    d_h0 = torch.full((wl.R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(wl.R * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(wl.R * wl.max_blocks, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(3):  # idempotent
        gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), wl.R, tok.nbytes, d_out.data_ptr(),
                              d_ch.data_ptr(), s)
    torch.cuda.synchronize()
    dev = d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, 1)
    assert H.picks_equal(dev, host) and H.picks_equal(dev, want)
    gchain = d_ch.cpu().numpy().view(np.uint64).reshape(wl.R, wl.max_blocks)
    wchain, _ = cpu.hash_batch(tok, offs, wl.h0)
    assert np.array_equal(gchain, wchain)
    assert gpu.stats().kernel_launches > 0
    gpu.close()


def test_batch_limits_are_enforced():
    cfg = make_config(num_endpoints=4, max_batch=4, max_prompt_bytes=1024)
    gpu = EndpointPicker(cfg)
    data, offs = H.pack_prompts([bytes(64)] * 5)
    with pytest.raises(Exception) as ei:
        gpu.pick_batch(data, offs, 1)
    assert "max_batch" in str(ei.value)
    data, offs = H.pack_prompts([bytes(2048)])
    with pytest.raises(Exception) as ei:
        gpu.pick_batch(data, offs, 1)
    assert "max_prompt_bytes" in str(ei.value)
    gpu.close()


def _random_lora_states(E, rng, n_adapters=12):
    from fusioninfer_b200 import LORA_DTYPE

    st = np.zeros(E, dtype=LORA_DTYPE)
    st["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 5)), int(rng.integers(0, 3))
        ids = rng.permutation(n_adapters)[: na + nw] + 1000
        st[e]["n_active"], st[e]["n_waiting"] = na, nw
        st[e]["active"][:na] = ids[:na]
        st[e]["waiting"][:nw] = ids[na:]
        st[e]["max_active"] = int(rng.integers(0, 7))
    return st


@pytest.mark.parametrize("E", [8, 100, 1024, 2048])
@pytest.mark.parametrize("scorers", [[(abi.FI_SCORER_LORA, 100)],
                                     [(P, 60), (abi.FI_SCORER_LORA, 30), (K, 5), (Q, 5)]])
def test_pick_parity_lora_affinity(E, scorers):
    rng = np.random.default_rng(E)
    wl = H.small_workload(E=E, R=128)
    cfg = H.config_for(wl, profiles=[{"name": "default", "scorers": scorers}])
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    lora = _random_lora_states(E, rng)
    gpu.update_endpoints_lora(lora)
    cpu.update_endpoints_lora(lora)
    tok, offs = wl.prompts()
    adapters = (rng.integers(0, 14, size=wl.R) + 1000).astype(np.uint64)  # includes ids nobody holds
    got = gpu.pick_batch(tok, offs, wl.h0, adapters=adapters)
    want = cpu.pick_batch(tok, offs, wl.h0, adapters=adapters)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    # without adapters every request uses id 0
    got0 = gpu.pick_batch(tok, offs, wl.h0)
    want0 = cpu.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got0, want0), H.describe_diff(got0, want0)
    gpu.close()


@pytest.mark.parametrize("slices", ["1", "3", "8", "16"])
def test_host_path_sliced_feed_is_exact(slices, monkeypatch):
    """fi_epp_pick_batch copies the prompts in slices and runs hash/walk/match per slice while the next
    slice is in flight (>= 8 MB of prompts): ragged prompt lengths, a batch size that is not a multiple of
    the slice size, PD profiles, chains_out — all equal to the oracle and to the single-copy path."""
    monkeypatch.setenv("FI_EPP_FEED_SLICES", slices)
    wl = synth.Workload(R=1000, E=96, T=4096, seed=synth.SEEDS[1], lru_capacity=2000, pd=True)
    profiles, pd = synth.baseline_profiles(5)
    pd = dict(pd, threshold=9000.0)
    cfg = H.config_for(wl, profiles=profiles, pd=pd, max_prompt_bytes=wl.R * wl.T * 4)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    tok, offs = wl.prompts()
    # ragged: cut a pseudo-random tail off every prompt (keeps 4-byte token alignment, some become empty)
    rng = np.random.default_rng(7)
    keep = rng.integers(0, wl.T + 1, size=wl.R)
    keep[::9] = wl.T
    keep[5] = 0
    blobs = [tok[r, : keep[r]].tobytes() for r in range(wl.R)]
    data, offs = H.pack_prompts(blobs)
    assert len(data) >= (8 << 20)
    got, gch = gpu.pick_batch(data, offs, wl.h0, want_chains=True)
    want, wch = cpu.pick_batch(data, offs, wl.h0, want_chains=True)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    assert np.array_equal(gch, wch)
    gpu.close()


@pytest.mark.parametrize("order", ["shuffled", "reversed", "interleaved"])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_pick_parity_whatever_the_insertion_order(order, mode):
    """The index numbers its nodes in insertion order and the match kernel first tries "next block = next
    node"; a prefix whose keys arrived out of chain order (shuffled op stream, reversed chains, two
    endpoints' ops interleaved) must fall back to table lookups and still give the oracle's answer."""
    wl = H.small_workload(E=96, R=256, holes=True, lru_capacity=600)
    cfg = H.config_for(wl, profiles=[{"name": "default", "scorers": [(P, 100), (K, 9), (Q, 5)]}], match_mode=mode)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    ops = np.concatenate(list(wl.index_ops()))
    rng = np.random.default_rng(11)
    if order == "shuffled":
        ops = ops[rng.permutation(len(ops))]
    elif order == "reversed":
        ops = ops[::-1].copy()
    else:  # odd and even positions of the stream swapped pairwise: runs of length one
        idx = np.arange(len(ops))
        idx[: len(ops) // 2 * 2] = idx[: len(ops) // 2 * 2].reshape(-1, 2)[:, ::-1].reshape(-1)
        ops = ops[idx]
    for lo in range(0, len(ops), 5000):  # several launches: node ranges of different launches interleave
        gpu.index_apply(ops[lo:lo + 5000])
    cpu.index_apply(ops)
    tok, offs = wl.prompts()
    got = gpu.pick_batch(tok, offs, wl.h0)
    want = cpu.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    assert int((got["match_blocks"] > 0).sum()) > 50
    gpu.close()


def test_pick_parity_after_churn_and_rebuild():
    """Chains are retired (every endpoint drops them: their nodes die), re-added for other endpoints in a
    different order, and the small table is forced through rebuilds (which compact the live nodes in node
    order); picks must follow the oracle through every phase."""
    wl = H.small_workload(E=48, R=192, lru_capacity=400)
    profiles = [{"name": "default", "scorers": [(P, 100), (K, 7), (Q, 3)]}]
    ops0 = np.concatenate(list(wl.index_ops()))
    uniq = len(np.unique(ops0["hash"]))
    slots = 256
    while slots * 0.55 < uniq:  # live keys stay under 60 % but tombstones push `used` over 70 %
        slots *= 2
    cfg = H.config_for(wl, profiles=profiles, index_slots=slots)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    tok, offs = wl.prompts()

    def check(tag):
        got = gpu.pick_batch(tok, offs, wl.h0)
        want = cpu.pick_batch(tok, offs, wl.h0)
        assert H.picks_equal(got, want), tag + "\n" + H.describe_diff(got, want)
        return got

    for arr in np.array_split(ops0, 7):
        gpu.index_apply(arr)
        cpu.index_apply(arr)
    first = check("initial")
    assert int((first["match_blocks"] > 0).sum()) > 40
    rng = np.random.default_rng(5)
    for phase in range(6):
        # drop everything a random third of the endpoints hold, then give the same hashes to other endpoints
        victims = rng.choice(wl.E, size=wl.E // 3, replace=False)
        sel = ops0[np.isin(ops0["endpoint"], victims)]
        clr = sel.copy()
        clr["op"] = abi.FI_OP_CLEAR
        gpu.index_apply(clr)
        cpu.index_apply(clr)
        check(f"phase {phase} after clears")
        re = sel[rng.permutation(len(sel))[: len(sel) // 2]].copy()
        re["endpoint"] = (re["endpoint"] + 1 + phase) % wl.E
        gpu.index_apply(re)
        cpu.index_apply(re)
        check(f"phase {phase} after re-adds")
        back = sel.copy()  # the victims get their chains back, in chain order
        gpu.index_apply(back)
        cpu.index_apply(back)
    check("final")
    assert gpu.index_stats().rebuilds >= 1
    gpu.close()


def test_pipelined_submit_equals_oracle_with_index_updates_in_between():
    """fi_epp_pick_submit keeps two batches in flight (batch k+1 is hashed while batch k is matched).  Seven
    different batches of different sizes are submitted back to back, index updates and a pod-state refresh
    are interleaved (each batch must see the index and the pod states as of ITS submit call), stream-ordered
    picks are mixed in; after one fi_epp_pick_wait every output equals the oracle's."""
    import torch

    wl = H.small_workload(E=128, R=384, T=1024, max_blocks=64, lru_capacity=500, pd=True)
    profiles, pd = synth.baseline_profiles(5)
    pd = dict(pd, threshold=900.0)
    cfg = H.config_for(wl, profiles=profiles, pd=pd)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    all_ops = np.concatenate(list(wl.index_ops()))
    parts = np.array_split(all_ops, 8)
    gpu.index_apply(parts[0])
    cpu.index_apply(parts[0])
    s = torch.cuda.current_stream().cuda_stream
    sizes = [384, 100, 1, 383, 64, 384, 200]
    keep, wants, outs = [], [], []
    rng = np.random.default_rng(3)
    for k, R in enumerate(sizes):
        tok, offs = wl.prompts(batch=k)
        tok = np.ascontiguousarray(tok[:R])
        offs = offs[: R + 1].copy()
        d_tok = torch.from_numpy(tok.view(np.int32)).cuda()
        d_off = torch.from_numpy(offs.view(np.int64)).cuda()
        d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
        d_out = torch.zeros(R * 2 * 16, dtype=torch.uint8, device="cuda")
        keep.append((d_tok, d_off, d_h0))
        wants.append(cpu.pick_batch(tok, offs, wl.h0))
        if k == 4:  # a stream-ordered pick in the middle of the pipeline
            gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_out.data_ptr(), 0, s)
        else:
            gpu.pick_submit(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_out.data_ptr(), s)
        outs.append(d_out)
        # the NEXT batch sees more of the index, some clears, and (once) refreshed pod states
        nxt = parts[k + 1]
        gpu.index_apply(nxt)
        cpu.index_apply(nxt)
        clr = parts[k][rng.permutation(len(parts[k]))[:200]].copy()
        clr["op"] = abi.FI_OP_CLEAR
        gpu.index_apply(clr)
        cpu.index_apply(clr)
        if k == 2:
            st2 = st.copy()
            st2["queue_depth"] = st2["queue_depth"][::-1].copy()
            st2["kv_util"] = 1.0 - st2["kv_util"]
            gpu.update_endpoints(st2)
            cpu.update_endpoints(st2)
    gpu.pick_wait(s)
    torch.cuda.synchronize()
    for k, R in enumerate(sizes):
        got = outs[k].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 2)
        assert H.picks_equal(got, wants[k]), f"batch {k}\n" + H.describe_diff(got, wants[k])
    gpu.close()


def test_tie_rotation_spreads_cold_requests_and_matches_the_rule():
    """ADVICE r1: with the reference's default profile (prefix scorer only, strategy.go:51-68) every request
    without a cached prefix ties on all endpoints; the rotation must spread them (not endpoint 0) and follow the
    rule of include/fi_epp.h, checked here against the independent python statement of it (tests/restate.py)."""
    from tests import restate

    wl = H.small_workload(E=200, R=256)
    cfg = H.config_for(wl)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    tok, offs = wl.prompts()
    got, chains = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
    want = cpu.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    assert len(np.unique(got[:, 0]["endpoint"])) > 60  # (requests of one Zipf group share their first block: same endpoint)
    for r in range(wl.R):
        assert got[r, 0]["endpoint"] == restate.tie_start(int(got[r, 0]["n_blocks"]), int(chains[r, 0]), wl.h0, r, wl.E)
    # short prompts (no block): rotation by (h0, request index); sliced and unsliced host feeds agree (r_base)
    data, offs2 = H.pack_prompts([bytes(10)] * 64)
    got2 = gpu.pick_batch(data, offs2, wl.h0)
    assert H.picks_equal(got2, cpu.pick_batch(data, offs2, wl.h0))
    assert len(np.unique(got2[:, 0]["endpoint"])) > 30
    gpu.close()


@pytest.mark.parametrize("lpm", [False, True])
def test_gpu_equals_the_second_restatement(lpm):
    """The kernels against tests/restate.py (python dicts / floats / the xxhash wheel; shares no code with the
    oracle): cfg 1 of BASELINE.json and a hole-y pool with the weighted PD profiles."""
    from tests import restate

    for wl, profiles, pd in (
        (synth.baseline_workload(1, lru_capacity=300),) + synth.baseline_profiles(1),
        (H.small_workload(E=48, R=96, holes=True, pd=True, lru_capacity=250),) + tuple(
            x if i == 0 else dict(x, threshold=700.0) for i, x in enumerate(synth.baseline_profiles(5))),
    ):
        cfg = H.config_for(wl, profiles=profiles, pd=pd, match_mode=abi.FI_MATCH_LPM if lpm else abi.FI_MATCH_UPSTREAM)
        gpu = EndpointPicker(cfg)
        ref = restate.from_config(cfg)
        st = wl.endpoint_states()
        gpu.update_endpoints(st)
        ref.update_endpoints(st)
        for ops in wl.index_ops():
            gpu.index_apply(ops)
            ref.apply(ops)
        tok, offs = wl.prompts()
        got = gpu.pick_batch(tok, offs, wl.h0)
        want = ref.pick(tok, offs, wl.h0)
        assert H.picks_equal(got, want), H.describe_diff(got, want)
        gpu.close()


@pytest.mark.parametrize("threads", ["1", "5", "device"])
def test_add_chains_batch_equals_sequential_oracle(threads, monkeypatch):
    """fi_epp_index_add_chains equals the oracle adding the chains one request at a time — over several steps
    with LRU churn (capacity far below one batch's inserts per endpoint), and the picks stay bit-exact.  Host LRU
    walked on a worker pool (segments where a hash is re-added after its eviction inside the same batch), and the
    device-resident LRU (the batch is cut into sub-batches of at most `capacity` touches per endpoint)."""
    if threads != "device":
        monkeypatch.setenv("FI_EPP_LRU_THREADS", threads)
    wl = H.small_workload(E=12, R=160, T=768, max_blocks=48, lru_capacity=70)
    prof = [{"name": "d", "scorers": [(P, 100), (K, 9), (Q, 5)]}]
    cfg = H.config_for(wl, profiles=prof, lru_capacity=70, index_slots=1 << 16)
    gpu, cpu = _pair(cfg)
    gpu.set_option("device_lru", 1 if threads == "device" else 0)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for step in range(6):
        tok, offs = wl.prompts(batch=step % 3)  # batches recur: prefixes are re-touched after evictions
        got, ch = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        want, wch = cpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        assert H.picks_equal(got, want), f"step {step}\n" + H.describe_diff(got, want)
        gpu.index_add_chains(got[:, 0]["endpoint"], ch, got[:, 0]["n_blocks"])
        cpu.index_add_chains(want[:, 0]["endpoint"], wch, want[:, 0]["n_blocks"])
    gpu.index_sync()
    # membership round trip on a sample of (endpoint, hash) pairs both ways
    q = [(int(wch[r, i]), int(e), 0) for r in range(0, wl.R, 7) for i in range(0, 48, 5) for e in range(wl.E)]
    have = gpu.index_contains(H.ops_array(q))
    for (hh, e, _), g in zip(q, have):
        assert bool(g) == cpu.index_contains(e, hh)
    stt = gpu.index_stats()
    assert stt.lru_entries <= wl.E * 70 and stt.tombstones > 0
    gpu.close()


def test_chained_label_filters_third_label():
    """by-label generalised (SURVEY §8(f)3): profiles with several ANDed filters over component-type AND two
    other labels' bits; disjoint filters admit nothing.  GPU == oracle."""
    wl = H.small_workload(E=200, R=128)
    prof = [{"name": "a", "role_mask": 1 | 4, "more_filters": [8 | 16, 32], "scorers": [(P, 60), (Q, 40)]},
            {"name": "b", "role_mask": 2, "more_filters": [4], "scorers": [(K, 1)]},
            {"name": "c", "role_mask": 0, "more_filters": [16], "scorers": [(P, 100), (K, 3)]}]
    cfg = H.config_for(wl, profiles=prof)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    rng = np.random.default_rng(9)
    st["role_mask"] = (1 << rng.integers(0, 3, size=wl.E)) | (8 << rng.integers(0, 2, size=wl.E)) | np.where(rng.random(wl.E) < 0.7, 32, 0)
    _load(wl, gpu, cpu, states=st)
    tok, offs = wl.prompts()
    got = gpu.pick_batch(tok, offs, wl.h0)
    want = cpu.pick_batch(tok, offs, wl.h0)
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    ok = ((st["role_mask"] & 5) != 0) & ((st["role_mask"] & 24) != 0) & ((st["role_mask"] & 32) != 0)
    assert ok[got[:, 0]["endpoint"]].all() and (got[:, 1]["endpoint"] == abi.FI_NO_ENDPOINT).all()
    assert ((st["role_mask"][got[:, 2]["endpoint"]] & 16) != 0).all()
    gpu.close()


class _PyLru:
    """hashicorp/golang-lru semantics, the plainest way: an ordered dict per endpoint (oldest first)."""

    def __init__(self, cap):
        from collections import OrderedDict

        self.cap, self.d = cap, OrderedDict()

    def add_chain(self, keys):
        for k in keys:
            k = int(k)
            if k in self.d:
                self.d.move_to_end(k)
            else:
                self.d[k] = True
                if len(self.d) > self.cap:
                    self.d.popitem(last=False)


def _device_lru_handle(E, cap, max_blocks, max_batch=256):
    wl = H.small_workload(E=E, R=8, T=max_blocks * 16, max_blocks=max_blocks, lru_capacity=0)
    cfg = H.config_for(wl, lru_capacity=cap, index_slots=1 << 17, max_batch=max_batch)
    gpu = EndpointPicker(cfg)
    gpu.set_option("device_lru", 1)
    gpu.set_option("lru_table_slots", 1)  # the minimum (4 x capacity): hot endpoints overflow their table
    return gpu


def _check_lru_state(gpu, ref, E):
    """recency order AND index membership equal the sequential reference"""
    for e in range(E):
        got = gpu.lru_dump(e)
        want = np.array(list(ref[e].d.keys()), dtype=np.uint64)
        assert np.array_equal(got, want), f"endpoint {e}: {len(got)} vs {len(want)} entries"
    # membership: every key ever seen, at every endpoint
    seen = np.array(sorted({k for l in ref for k in l.d} | getattr(_check_lru_state, "extra", set())), dtype=np.uint64)
    q = np.zeros(len(seen) * E, dtype=H.OP_DTYPE)  # every (key, endpoint) pair, key-major
    q["hash"] = np.repeat(seen, E)
    q["endpoint"] = np.tile(np.arange(E, dtype=np.uint32), len(seen))
    have = gpu.index_contains(q)
    want = np.stack([np.isin(seen, np.array(list(ref[e].d), dtype=np.uint64)) for e in range(E)], axis=1).ravel()
    assert np.array_equal(have.astype(bool), want)


def test_device_lru_order_and_membership_random_batches():
    """The device-resident LRU against a sequential ordered-dict LRU: random batches with shared prefixes, keys
    re-touched within and across batches, hot endpoints that force several sub-batches, enough churn for the
    log compaction / table rebuild to run many times; recency order (fi_epp_lru_dump) and index membership
    are compared after every batch."""
    _device_lru_random_batches(cap=90, M=24)


@pytest.mark.parametrize("cap,M", [(1023, 1023), (1100, 1023)])
def test_device_lru_random_batches_long_chains(cap, M):
    """The same with chains of up to 1023 blocks: a single chain can fill (cap = M) or nearly fill an LRU."""
    _device_lru_random_batches(cap, M)


def _device_lru_random_batches(cap, M):
    E = 6
    gpu = _device_lru_handle(E, cap, M)
    ref = [_PyLru(cap) for _ in range(E)]
    rng = np.random.default_rng(2024)
    ever = set()
    # a pool of prefix chains; requests take a prefix of a pool chain plus a private tail
    pool = rng.integers(1, 1 << 62, size=(40, M), dtype=np.uint64)
    for step in range(40):
        R = int(rng.integers(1, 60))
        chains = np.zeros((R, M), dtype=np.uint64)
        nb = rng.integers(0, M + 1, size=R).astype(np.uint32)
        eps = rng.integers(0, E, size=R).astype(np.uint32)
        if step % 5 == 0:
            eps[:] = eps[0]  # hot spot: one endpoint takes the whole batch
        eps[rng.random(R) < 0.05] = abi.FI_NO_ENDPOINT
        for r in range(R):
            c = pool[rng.integers(0, len(pool))]
            cut = int(rng.integers(0, M + 1))
            chains[r, :cut] = c[:cut]
            chains[r, cut:] = rng.integers(1, 1 << 62, size=M - cut, dtype=np.uint64)
            if rng.random() < 0.1 and nb[r] >= 2:
                chains[r, nb[r] - 1] = chains[r, 0]  # the same key twice in one chain
        gpu.index_add_chains(eps, chains, nb)
        for r in range(R):
            if eps[r] != abi.FI_NO_ENDPOINT:
                ref[eps[r]].add_chain(chains[r, : nb[r]])
                ever.update(int(k) for k in chains[r, : nb[r]])
        if step % 4 == 3 or step < 3:
            _check_lru_state.extra = set(list(ever)[:: max(1, len(ever) // 400)])
            _check_lru_state(gpu, ref, E)
    _check_lru_state.extra = ever
    _check_lru_state(gpu, ref, E)
    st = gpu.index_stats()
    assert st.lru_entries == sum(len(l.d) for l in ref) and st.tombstones > 0
    c = gpu.lru_counters()
    # every path ran: keys gone again within their batch, an endpoint whose table refused a batch (rolled back and
    # re-run in capacity-sized sub-batches), log compactions / table rebuilds
    assert c["doomed"] > 0 and c["deferred_requests"] > 0 and c["maintained"] > 0 and c["sub_batches"] > 40, c
    assert c["sets"] >= st.lru_entries and c["clears"] >= c["doomed"]  # (doomed keys are CLEARed whether they were entries or not)
    gpu.close()


def test_device_lru_edge_cases():
    """capacity hit exactly; a chain as long as the capacity; the hashes 0 and ~0 (the tables' own markers);
    single-chain calls interleaved with batches; empty calls."""
    _device_lru_edge_cases(cap=16, M=16)


@pytest.mark.parametrize("cap,M", [(1023, 1023), (1100, 1023)])
def test_device_lru_edge_cases_long_chains(cap, M):
    """The same with 1023-key chains: one chain fills the LRU exactly (cap = M) or nearly (M < cap)."""
    _device_lru_edge_cases(cap, M)


def _device_lru_edge_cases(cap, M):
    E = 3
    gpu = _device_lru_handle(E, cap, M)
    ref = [_PyLru(cap) for _ in range(E)]
    ever = set()

    def add(eps, chains, nb):
        eps = np.asarray(eps, dtype=np.uint32)
        chains = np.asarray(chains, dtype=np.uint64).reshape(len(eps), -1)
        nb = np.asarray(nb, dtype=np.uint32)
        gpu.index_add_chains(eps, chains, nb)
        for r in range(len(eps)):
            ref[eps[r]].add_chain(chains[r, : nb[r]])
            ever.update(int(k) for k in chains[r, : nb[r]])
        _check_lru_state.extra = ever
        _check_lru_state(gpu, ref, E)

    a = np.arange(1, M + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    add([0], [a], [M])                       # fills endpoint 0 exactly (M = cap)
    add([0], [a[::-1].copy()], [M])          # same keys, reversed recency: no eviction
    b = a + np.uint64(7)
    add([0, 0], [b, a], [M, M])              # a chain of `capacity` new keys evicts everything, then back again
    special = np.array([0, 0xFFFFFFFFFFFFFFFF, 5, 0, 9, 0xFFFFFFFFFFFFFFFF] + [11] * (M - 6), dtype=np.uint64)
    add([1, 2], [special, special], [6, 4])  # the hashes 0 and ~0 are ordinary members
    for i in range(cap + 4):                 # push them out again, one new key per call (single-chain entry point)
        k = np.array([1000 + i], dtype=np.uint64)
        gpu.index_add_chain(1, k)
        ref[1].add_chain(k)
        ever.add(1000 + i)
    _check_lru_state.extra = ever
    _check_lru_state(gpu, ref, E)
    add([1], [special], [6])                 # and in again
    gpu.index_add_chains(np.zeros(0, np.uint32), np.zeros((0, M), np.uint64), np.zeros(0, np.uint32))
    add([2, 2, 2], [a, b, a], [0, 3, 0])     # zero-length chains are skipped
    gpu.close()


def test_device_lru_from_device_chains():
    """fi_epp_index_add_chains_device: the chains stay in device memory (chains_out of the device pick); same
    chains and picks as the oracle over several churn steps."""
    _device_lru_from_device_chains(max_blocks=32, T=512, cap=300, slots=1 << 17)


def test_device_lru_from_device_chains_long_prompts():
    """The same at max_blocks = 1023: chains_out's pitch (1023) is not the device buffers' (1024)."""
    _device_lru_from_device_chains(max_blocks=1023, T=16 * 1024, cap=3000, slots=1 << 20)


def _device_lru_from_device_chains(max_blocks, T, cap, slots):
    import torch

    wl = H.small_workload(E=40, R=256, T=T, max_blocks=max_blocks, lru_capacity=0)
    prof = [{"name": "d", "scorers": [(P, 100), (K, 9), (Q, 5)]}]
    cfg = H.config_for(wl, profiles=prof, lru_capacity=cap, index_slots=slots, max_prompt_bytes=wl.R * wl.T * 4)
    gpu, cpu = _pair(cfg)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    d_out = torch.zeros(wl.R * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(wl.R * wl.max_blocks, dtype=torch.int64, device="cuda")
    for step in range(5):
        tok, offs = wl.prompts(batch=step % 2)
        d_tok = torch.from_numpy(tok.view(np.int32)).cuda()
        d_off = torch.from_numpy(offs.view(np.int64)).cuda()
        d_h0 = torch.full((wl.R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), wl.R, tok.nbytes, d_out.data_ptr(),
                              d_chains=d_ch.data_ptr(), stream=stream)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, 1)
        want, wch = cpu.pick_batch(tok, offs, wl.h0, want_chains=True)
        assert H.picks_equal(got, want), f"step {step}\n" + H.describe_diff(got, want)
        assert np.array_equal(d_ch.cpu().numpy().view(np.uint64).reshape(wl.R, wl.max_blocks), wch), f"step {step}"
        gpu.index_add_chains_device(got[:, 0]["endpoint"], d_ch.data_ptr(), wl.max_blocks, got[:, 0]["n_blocks"], stream=stream)
        cpu.index_add_chains(want[:, 0]["endpoint"], wch, want[:, 0]["n_blocks"])
    assert gpu.index_stats().tombstones > 0
    gpu.close()


@pytest.mark.parametrize("block_tokens,max_blocks", [
    pytest.param(16, 128, id="64B-128"), pytest.param(16, 1023, id="64B-1023"),
    pytest.param(24, 128, id="96B-128"), pytest.param(24, 1023, id="96B-1023"),
])
def test_pipelined_back_to_back_batches(block_tokens, max_blocks):
    """Twelve batches of different sizes submitted back to back with nothing in between (so that the pipeline really
    has its two batches in flight and reuses every slot buffer several times), one wait at the end, every output
    equal to the oracle's; then the same again after a stream-ordered pick.  Stage A is one hash_chain launch:
    hash_chain<2, WALK> at 64-byte blocks, the run-time stripe count hash_chain<0, WALK> at 96-byte blocks.
    max_blocks = 1023: prompts past the cap with a partial last block, chain pitch 1024."""
    import torch

    if max_blocks == 128:
        wl = H.small_workload(E=200, R=512, T=128 * block_tokens, max_blocks=128, block_tokens=block_tokens)
    else:
        wl = H.small_workload(E=200, R=512, T=block_tokens * (max_blocks + 1) + 5, max_blocks=max_blocks,
                              groups_per_endpoint=2, block_tokens=block_tokens)
    cfg = H.config_for(wl, profiles=WEIGHTED, max_prompt_bytes=wl.R * wl.T * 4)
    gpu, cpu = _pair(cfg)
    _load(wl, gpu, cpu)
    s = torch.cuda.current_stream().cuda_stream
    sizes = [512, 37, 512, 1, 300, 512, 512, 64, 511, 512, 200, 512]
    for rnd in range(2):
        keep, wants, outs = [], [], []
        for k, R in enumerate(sizes):
            tok, offs = wl.prompts(batch=k + 20 * rnd)
            tok = np.ascontiguousarray(tok[:R])
            offs = offs[: R + 1].copy()
            d_tok = torch.from_numpy(tok.view(np.int32)).cuda()
            d_off = torch.from_numpy(offs.view(np.int64)).cuda()
            d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
            d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
            keep.append((d_tok, d_off, d_h0))
            wants.append(cpu.pick_batch(tok, offs, wl.h0))
            outs.append(d_out)
        torch.cuda.synchronize()
        for k, R in enumerate(sizes):
            d_tok, d_off, d_h0 = keep[k]
            gpu.pick_submit(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(d_tok.numel()) * 4, outs[k].data_ptr(), s)
        gpu.pick_wait(s)
        torch.cuda.synchronize()
        for k, R in enumerate(sizes):
            got = outs[k].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
            assert H.picks_equal(got, wants[k]), f"round {rnd} batch {k}\n" + H.describe_diff(got, wants[k])
        if rnd == 0:  # a stream-ordered pick between the two pipelined rounds
            tok, offs = wl.prompts(batch=99)
            assert H.picks_equal(gpu.pick_batch(tok, offs, wl.h0), cpu.pick_batch(tok, offs, wl.h0))
    assert not gpu.pipeline_info()["partitioned"]
    gpu.close()


@pytest.mark.parametrize("name", ["pipe_partition", "pipe_hash_ctas", "pipe_match_ctas"])
def test_removed_pipeline_options_are_unknown(name):
    """The SM partition of the pipelined path and its per-SM CTA caps are gone: their option names are unknown."""
    wl = H.small_workload(E=8, R=4)
    gpu = EndpointPicker(H.config_for(wl))
    with pytest.raises(FiEppError) as ei:
        gpu.set_option(name, 0)
    assert ei.value.status == abi.FI_ERR_INVALID
    assert "unknown option" in str(ei.value)
    gpu.close()


def test_device_lru_next_to_direct_index_ops():
    """fi_epp_index_apply bypasses the LRU (as in upstream, where only PreRequest feeds it).  A key that is in the
    index that way, is then touched by an Add and pushed out of the LRU again within the same batch must end up
    ABSENT (sequential Adds: SET — a no-op — then CLEAR), exactly like the oracle's index."""
    wl = H.small_workload(E=4, R=8, T=256, max_blocks=16, lru_capacity=0)
    cfg = H.config_for(wl, lru_capacity=20, index_slots=1 << 14, max_batch=64)
    gpu, cpu = _pair(cfg)
    gpu.set_option("device_lru", 1)
    rng = np.random.default_rng(11)
    direct = rng.integers(1, 1 << 62, size=16, dtype=np.uint64)
    ops = H.ops_array([(int(h), e, abi.FI_OP_SET) for h in direct for e in (0, 1)])
    gpu.index_apply(ops)
    cpu.index_apply(ops)
    # endpoint 0: the direct keys first, then 40 fresh ones in the same batch (capacity 20: the direct keys are
    # touched, inserted into the LRU, and evicted again); endpoint 1: only a few fresh keys (direct keys stay)
    fresh = rng.integers(1, 1 << 62, size=(3, 16), dtype=np.uint64)
    chains = np.stack([direct, fresh[0], fresh[1], fresh[2]])
    eps = np.array([0, 0, 0, 1], dtype=np.uint32)
    nb = np.array([16, 16, 16, 5], dtype=np.uint32)
    gpu.index_add_chains(eps, chains, nb)
    cpu.index_add_chains(eps, chains, nb)
    q = [(int(h), e, 0) for h in np.concatenate([direct, fresh.ravel()]) for e in range(4)]
    have = gpu.index_contains(H.ops_array(q))
    want = np.array([cpu.index_contains(e, h) for h, e, _ in q], dtype=bool)
    assert np.array_equal(have.astype(bool), want)
    assert not have[: 16 * 4].reshape(16, 4)[:, 0].any()   # the direct keys are gone from endpoint 0 ...
    assert have[: 16 * 4].reshape(16, 4)[:, 1].all()       # ... and still on endpoint 1
    assert gpu.lru_counters()["doomed"] >= 16
    gpu.close()
