"""GPU (-m gpu): the ranked pick (fi_epp_pick_batch_ranked / _device_ranked, docs/SPEC.md S.6a).

Every comparison is bit-exact (scores as raw 64-bit patterns): k = 1 against the single pick of the same handle,
k > 1 against the CPU oracle's ranked pick (tests/ext_oracle.cpp), on every row shape of the match kernel.
"""
import ctypes as C
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
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
NOBODY = 64  # a label bit no endpoint carries

CASES = {
    "weighted": dict(profiles=[{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]),
    # chained by-label filters; the second profile admits nobody
    "filters": dict(profiles=[{"name": "a", "role_mask": 3, "more_filters": [12], "scorers": [(P, 10), (Q, 3)]},
                              {"name": "none", "role_mask": NOBODY, "scorers": [(P, 1)]},
                              {"name": "c", "role_mask": 16, "scorers": [(P, 5), (K, 1)]}]),
    "pd": dict(profiles=[{"name": "prefill", "role_mask": 1, "scorers": [(P, 50), (K, 5)]},
                         {"name": "decode", "role_mask": 2, "scorers": [(P, 50), (Q, 5)]}],
               pd={"prefill": 0, "decode": 1}),
    "lora": dict(profiles=[{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5), (Q, 5)]}]),
}


def _states(wl, rng, roles=True):
    st = wl.endpoint_states()
    if roles:
        st["role_mask"] = rng.integers(1, 32, wl.E).astype(np.uint32)
    st["flags"] = np.where(rng.random(wl.E) < 0.15, 0, abi.FI_ENDPOINT_ALIVE)  # dead endpoints
    return st


def _lora(E, rng):
    from fusioninfer_b200 import LORA_DTYPE

    st = np.zeros(E, dtype=LORA_DTYPE)
    st["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 5)), int(rng.integers(0, 3))
        ids = rng.permutation(12)[: na + nw] + 1000
        st[e]["n_active"], st[e]["n_waiting"] = na, nw
        st[e]["active"][:na] = ids[:na]
        st[e]["waiting"][:nw] = ids[na:]
        st[e]["max_active"] = int(rng.integers(0, 7))
    return st


def _setup(wl, case, mode, rng, **kw):
    spec = dict(CASES[case])
    if case == "pd":  # a threshold that splits the batch between prefill and skip
        spec["pd"] = dict(spec["pd"], threshold=0.6 * wl.T * 4)
    cfg = H.config_for(wl, match_mode=mode, max_prompt_bytes=wl.R * wl.T * 4, **spec, **kw)
    gpu, cpu = EndpointPicker(cfg), ExtOracle(cfg)
    st = _states(wl, rng)
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    if case == "lora":
        lo = _lora(wl.E, rng)
        gpu.update_endpoints_lora(lo)
        cpu.update_endpoints_lora(lo)
    for ops in wl.index_ops():
        gpu.index_apply(ops)
        cpu.index_apply(ops)
    return gpu, cpu


def _cold(offs, n=8, nbytes=20):
    """the first n requests become prompts shorter than one block: every prefix total ties"""
    offs = offs.copy()
    offs[1:n + 1] = offs[0] + np.arange(1, n + 1, dtype=np.uint64) * nbytes
    return offs


def _eq(got, want, what):
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("max_blocks", [256, 1023])
def test_k1_equals_the_single_pick(case, mode, max_blocks):
    rng = np.random.default_rng(max_blocks + mode)
    T = 16 * max_blocks + 40  # the longest prompts run past the cap and end in a partial block
    wl = H.small_workload(E=100, R=96, T=T, max_blocks=max_blocks, holes=True, lru_capacity=max_blocks)
    gpu, cpu = _setup(wl, case, mode, rng)
    tok, offs = wl.prompts()
    offs = _cold(offs)
    ad = (rng.integers(0, 14, wl.R) + 1000).astype(np.uint64) if case == "lora" else None
    single = gpu.pick_batch(tok, offs, wl.h0, adapters=ad)
    ranked = gpu.pick_batch_ranked(tok, offs, wl.h0, 1, adapters=ad)
    assert ranked.shape == (wl.R, len(CASES[case]["profiles"]), 1)
    _eq(np.ascontiguousarray(ranked[:, :, 0]), single, "ranked k = 1 vs fi_epp_pick_batch")
    _eq(ranked, cpu.pick_batch_ranked(tok, offs, wl.h0, 1, adapters=ad), "ranked k = 1 vs the oracle")
    if case == "pd":  # the threshold splits the batch
        skipped = ranked[:, 0, 0]["endpoint"] == abi.FI_NO_ENDPOINT
        assert skipped.any() and not skipped.all()
    gpu.close()


@pytest.mark.parametrize("E", [1, 3, 40, 100, 200, 500, 1024, 2048, 4096])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_ranked_equals_the_oracle_on_every_row_shape(E, mode):
    """Pools of 1 to 4 096 endpoints (1 to 128 words per row); fewer eligible endpoints than k; a profile that
    admits nobody; cold prompts whose totals all tie, so the list is the request's rotation."""
    rng = np.random.default_rng(E * 3 + mode)
    wl = H.small_workload(E=E, R=96, holes=True)
    profiles = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]},
                {"name": "prefix", "role_mask": 3, "scorers": [(P, 100)]},
                {"name": "none", "role_mask": NOBODY, "scorers": [(P, 1)]}]
    cfg = H.config_for(wl, match_mode=mode, profiles=profiles)
    gpu, cpu = EndpointPicker(cfg), ExtOracle(cfg)
    st = _states(wl, rng, roles=False)
    st["role_mask"] = rng.integers(1, 8, E).astype(np.uint32)
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for ops in wl.index_ops():
        gpu.index_apply(ops)
        cpu.index_apply(ops)
    tok, offs = wl.prompts()
    offs = _cold(offs, n=16)
    for k in (2, 4, 16):
        got = gpu.pick_batch_ranked(tok, offs, wl.h0, k)
        _eq(got, cpu.pick_batch_ranked(tok, offs, wl.h0, k), f"E={E} k={k}")
        assert (got[:, 2]["endpoint"] == abi.FI_NO_ENDPOINT).all()
        if E > 16:  # the cold requests of the prefix-only profile: its eligible endpoints in rotation order
            assert (got[:16, 1, :]["endpoint"] != abi.FI_NO_ENDPOINT).all()
    gpu.close()


def _device_batch(tok, offs, h0, R, k, P):
    import torch

    d_tok = torch.from_numpy(np.ascontiguousarray(tok[:R]).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs[: R + 1].copy().view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * P * k * 16, dtype=torch.uint8, device="cuda")
    return d_tok, d_off, d_h0, d_out


@pytest.mark.parametrize("case", ["weighted", "lora"])
def test_host_and_device_entry_points_agree(case):
    import torch

    rng = np.random.default_rng(5)
    wl = H.small_workload(E=200, R=128, holes=True)
    gpu, cpu = _setup(wl, case, abi.FI_MATCH_UPSTREAM, rng)
    tok, offs = wl.prompts()
    ad = (rng.integers(0, 14, wl.R) + 1000).astype(np.uint64) if case == "lora" else None
    k, Pn = 4, len(CASES[case]["profiles"])
    host, chains = gpu.pick_batch_ranked(tok, offs, wl.h0, k, want_chains=True, adapters=ad)
    _eq(host, cpu.pick_batch_ranked(tok, offs, wl.h0, k, adapters=ad), "host ranked vs the oracle")
    assert np.array_equal(chains, cpu.hash_batch(tok, offs, wl.h0)[0])
    b = _device_batch(tok, offs, wl.h0, wl.R, k, Pn)
    d_ad = torch.from_numpy(ad.view(np.int64)).cuda() if ad is not None else None
    d_chains = torch.zeros(wl.R * wl.max_blocks, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    gpu.pick_batch_device_ranked(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), wl.R, tok.nbytes, k, b[3].data_ptr(),
                                 d_chains.data_ptr(), s, d_ad.data_ptr() if d_ad is not None else 0)
    torch.cuda.synchronize()
    dev = b[3].cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, Pn, k)
    _eq(dev, host, "device ranked vs host ranked")
    assert np.array_equal(d_chains.cpu().numpy().view(np.uint64).reshape(wl.R, wl.max_blocks), chains)
    gpu.close()


def test_sliced_host_feed_agrees_with_the_unsliced_one():
    """>= 8 MiB of prompts and R >= 64 * slices: the host call copies and matches slice by slice"""
    rng = np.random.default_rng(11)
    wl = H.small_workload(E=64, R=2048, T=1100, max_blocks=64, holes=True)
    gpu, cpu = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng)
    tok, offs = wl.prompts()
    assert int(offs[-1]) >= 8 << 20
    sliced = gpu.pick_batch_ranked(tok, offs, wl.h0, 8)
    gpu.set_option("feed_slices", 1)
    whole = gpu.pick_batch_ranked(tok, offs, wl.h0, 8)
    _eq(sliced, whole, "sliced vs unsliced feed")
    _eq(whole, cpu.pick_batch_ranked(tok, offs, wl.h0, 8), "vs the oracle")
    gpu.close()


def test_ranked_after_pipelined_submits_and_removal():
    import torch

    rng = np.random.default_rng(3)
    wl = H.small_workload(E=64, R=256, holes=True)
    gpu, _ = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng)
    s = torch.cuda.current_stream().cuda_stream
    batches = [wl.prompts(batch=i) for i in range(3)]
    dev = [_device_batch(t, o, wl.h0, wl.R, 1, 1) for t, o in batches]
    torch.cuda.synchronize()
    for (t, _), b in zip(batches, dev):  # still in flight when the ranked call is made
        gpu.pick_submit(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), wl.R, t.nbytes, b[3].data_ptr(), s)
    tok, offs = batches[0]
    ranked = gpu.pick_batch_ranked(tok, offs, wl.h0, 4)
    gpu.pick_wait(s)
    torch.cuda.synchronize()
    single = gpu.pick_batch(tok, offs, wl.h0)
    _eq(np.ascontiguousarray(ranked[:, :, 0]), single, "ranked after pipelined submits")
    sub = dev[0][3].cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, 1)
    _eq(sub, single, "the submitted batch")
    victims = sorted(set(int(e) for e in single[:40, 0]["endpoint"]))
    gpu.remove_endpoints(victims)  # asynchronous: the ranked call is ordered after it
    ranked = gpu.pick_batch_ranked(tok, offs, wl.h0, 4)
    single = gpu.pick_batch(tok, offs, wl.h0)
    _eq(np.ascontiguousarray(ranked[:, :, 0]), single, "ranked after remove_endpoints")
    assert not np.isin(ranked["endpoint"][ranked["match_blocks"] > 0], victims).any()
    gpu.close()


def test_add_chains_device_after_a_ranked_call_takes_its_chains():
    """upstream PreRequest after a ranked pick: the device LRU adds the chains of the ranked call"""
    rng = np.random.default_rng(4)
    wl = H.small_workload(E=40, R=128, lru_capacity=300)
    gpu, cpu = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng, lru_capacity=300)
    tok, offs = wl.prompts(batch=0)
    got = gpu.pick_batch_ranked(tok, offs, wl.h0, 3)
    want = cpu.pick_batch_ranked(tok, offs, wl.h0, 3)
    _eq(got, want, "ranked before the Add")
    chains = cpu.hash_batch(tok, offs, wl.h0)[0]
    eps, nb = got[:, 0, 0]["endpoint"], got[:, 0, 0]["n_blocks"]
    gpu.index_add_chains_device(eps, 0, 0, nb)
    cpu.index_add_chains(eps, chains, nb)
    for e in sorted(set(int(x) for x in eps if x != abi.FI_NO_ENDPOINT))[:8]:
        held = gpu.lru_dump(e)
        assert all(cpu.index_contains(e, int(h)) for h in held)
    tok2, offs2 = wl.prompts(batch=1)
    _eq(gpu.pick_batch_ranked(tok2, offs2, wl.h0, 3), cpu.pick_batch_ranked(tok2, offs2, wl.h0, 3), "after the Add")
    gpu.close()


def test_sub_range_handle_reports_global_endpoints():
    """one rank over endpoints [begin, begin + count) of the pool: the oracle sees the others as dead"""
    rng = np.random.default_rng(6)
    wl = H.small_workload(E=300, R=128, holes=True)
    begin, count = 100, 150
    profiles = [{"name": "default", "scorers": [(P, 100), (K, 13)]}]
    gpu = EndpointPicker(H.config_for(wl, profiles=profiles, endpoint_begin=begin, endpoint_count=count))
    cpu = ExtOracle(H.config_for(wl, profiles=profiles))
    st = _states(wl, rng, roles=False)
    gpu.update_endpoints(st)
    st = st.copy()
    st["flags"][:begin] = 0
    st["flags"][begin + count:] = 0
    cpu.update_endpoints(st)
    for ops in wl.index_ops(begin, begin + count):
        gpu.index_apply(ops)
        cpu.index_apply(ops)
    tok, offs = wl.prompts()
    got = gpu.pick_batch_ranked(tok, offs, wl.h0, 5)
    _eq(got, cpu.pick_batch_ranked(tok, offs, wl.h0, 5), "sub-range handle")
    real = got["endpoint"][got["endpoint"] != abi.FI_NO_ENDPOINT]
    assert real.min() >= begin and real.max() < begin + count
    gpu.close()


def test_bad_arguments_are_rejected():
    wl = H.small_workload(E=40, R=16)
    gpu = EndpointPicker(H.config_for(wl))
    tok, offs = wl.prompts()
    for k in (0, abi.FI_EPP_MAX_RANKED + 1):
        with pytest.raises(FiEppError) as ei:
            gpu.pick_batch_ranked(tok, offs, wl.h0, k)
        assert ei.value.status == abi.FI_ERR_INVALID
    lib = abi.load()
    tok = np.ascontiguousarray(tok)
    h0 = np.full(wl.R, wl.h0, dtype=np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert lib.fi_epp_pick_batch_ranked(gpu._h, p(tok), p(offs), p(h0), None, wl.R, 2, None, None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_pick_batch_device_ranked(gpu._h, None, p(offs), p(h0), None, wl.R, 0, 2, None, None,
                                               None) == abi.FI_ERR_INVALID
    assert gpu.pick_batch_ranked(tok, offs, wl.h0, abi.FI_EPP_MAX_RANKED).shape == (wl.R, 1, abi.FI_EPP_MAX_RANKED)
    gpu.close()


def test_sharded_pool_is_refused(gpu_count):
    if gpu_count < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    wl = H.small_workload(E=64, R=32)
    uid = EndpointPicker.comm_unique_id()
    status = [None] * world
    errors = []
    tok, offs = wl.prompts()

    def worker(rank):
        try:
            begin, count = shard_range(wl.E, rank, world)
            p = EndpointPicker(H.config_for(wl, device=rank, endpoint_begin=begin, endpoint_count=count))
            p.comm_init(uid, rank, world)
            try:
                p.pick_batch_ranked(tok, offs, wl.h0, 2)
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
