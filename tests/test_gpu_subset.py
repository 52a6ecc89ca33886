"""GPU (-m gpu): subset picks (fi_epp_pick_batch_subset / _device_subset, docs/SPEC.md S.5a).

Every comparison is bit-exact (scores as raw 64-bit patterns): no subset and all-ones subsets against the ranked and
single picks of the same handle, random subsets against the subset CPU oracle (tests/subset_oracle.cpp), on every
row shape of the match kernel.
"""
import ctypes as C

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import helpers as H
from tests.subset_oracle import SubsetOracle
from tests.test_gpu_ranked import CASES, _cold, _device_batch, _eq, _lora, _states

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q


def _setup(wl, case, mode, rng, **kw):
    spec = dict(CASES[case])
    if case == "pd":  # a threshold that splits the batch between prefill and skip
        spec["pd"] = dict(spec["pd"], threshold=0.6 * wl.T * 4)
    cfg = H.config_for(wl, match_mode=mode, max_prompt_bytes=wl.R * wl.T * 4, **spec, **kw)
    gpu, cpu = EndpointPicker(cfg), SubsetOracle(cfg)
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


def _random_subsets(R, E, rng):
    """request r gets a random subset of size (0, 1, 8, E/2, E)[r % 5] (capped at E)"""
    sizes = [0, 1, 8, E // 2, E]
    return subset_bitsets([rng.choice(E, min(sizes[r % 5], E), replace=False).tolist() for r in range(R)], E)


def _adapters(case, R, rng):
    return (rng.integers(0, 14, R) + 1000).astype(np.uint64) if case == "lora" else None


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("max_blocks", [256, 1023])
def test_no_subset_and_all_ones_equal_the_ranked_and_single_picks(case, mode, max_blocks):
    rng = np.random.default_rng(max_blocks + mode + 17)
    T = 16 * max_blocks + 40  # the longest prompts run past the cap and end in a partial block
    wl = H.small_workload(E=100, R=96, T=T, max_blocks=max_blocks, holes=True, lru_capacity=max_blocks)
    gpu, cpu = _setup(wl, case, mode, rng)
    tok, offs = wl.prompts()
    offs = _cold(offs)
    ad = _adapters(case, wl.R, rng)
    ones = subset_bitsets([None] * wl.R, wl.E)
    single = gpu.pick_batch(tok, offs, wl.h0, adapters=ad)
    for k in (1, 4):
        ranked = gpu.pick_batch_ranked(tok, offs, wl.h0, k, adapters=ad)
        _eq(gpu.pick_batch_subset(tok, offs, wl.h0, None, k, adapters=ad), ranked, f"NULL subsets vs ranked, k={k}")
        _eq(gpu.pick_batch_subset(tok, offs, wl.h0, ones, k, adapters=ad), ranked, f"all-ones subsets vs ranked, k={k}")
    got = gpu.pick_batch_subset(tok, offs, wl.h0, ones, 1, adapters=ad)
    _eq(np.ascontiguousarray(got[:, :, 0]), single, "all-ones subsets, k = 1 vs the single pick")
    # random subsets on the long prompts (the variant's own shared-memory opt-in at 1 023 blocks)
    sub = _random_subsets(wl.R, wl.E, rng)
    _eq(gpu.pick_batch_subset(tok, offs, wl.h0, sub, 4, adapters=ad), cpu.pick_batch_subset(tok, offs, wl.h0, sub, 4, ad),
        "random subsets vs the oracle")
    gpu.close()
    cpu.close()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("E", [1, 3, 40, 100, 200, 500, 1024, 2048, 4096])
def test_random_subsets_equal_the_oracle_on_every_row_shape(case, E):
    """Pools of 1 to 4 096 endpoints (1 to 128 words per row), subsets of 0, 1, 8, E/2 and E endpoints, both match
    modes, k = 1, 4 and 16; cold prompts whose prefix totals all tie"""
    for mode in (abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM):
        rng = np.random.default_rng(E * 5 + mode)
        wl = H.small_workload(E=E, R=96, holes=True)
        gpu, cpu = _setup(wl, case, mode, rng)
        tok, offs = wl.prompts()
        offs = _cold(offs, n=16)
        ad = _adapters(case, wl.R, rng)
        sub = _random_subsets(wl.R, E, rng)
        for k in (1, 4, 16):
            got = gpu.pick_batch_subset(tok, offs, wl.h0, sub, k, adapters=ad)
            _eq(got, cpu.pick_batch_subset(tok, offs, wl.h0, sub, k, ad), f"E={E} mode={mode} k={k}")
        empty = np.arange(wl.R) % 5 == 0
        assert (got["endpoint"][empty] == abi.FI_NO_ENDPOINT).all()
        gpu.close()
        cpu.close()


def test_queue_normalisation_over_the_subset():
    """queues [0, 10, 5, 20] with subset {1, 3}: endpoint 1 scores 1.0 (the whole pool would give 0.5)"""
    wl = H.small_workload(E=4, R=8)
    gpu = EndpointPicker(H.config_for(wl, profiles=[{"name": "q", "scorers": [(Q, 1)]}]))
    gpu.update_endpoints(H.states_array(4, queue=np.array([0, 10, 5, 20])))
    tok, offs = wl.prompts()
    got = gpu.pick_batch_subset(tok, offs, wl.h0, subset_bitsets([[1, 3]] * wl.R, 4), 2)
    assert (got["endpoint"][:, 0] == [[1, 3]] * wl.R).all()
    assert (got["score"][:, 0] == [[1.0, 0.0]] * wl.R).all()
    whole = gpu.pick_batch_subset(tok, offs, wl.h0, None, 4)
    assert (whole["endpoint"][:, 0] == [[0, 2, 1, 3]] * wl.R).all()
    gpu.close()


def _d_subsets(sub):
    import torch

    return torch.from_numpy(np.ascontiguousarray(sub).view(np.int32)).cuda()


@pytest.mark.parametrize("case", ["weighted", "lora"])
def test_host_and_device_entry_points_agree(case):
    import torch

    rng = np.random.default_rng(5)
    wl = H.small_workload(E=200, R=128, holes=True)
    gpu, cpu = _setup(wl, case, abi.FI_MATCH_UPSTREAM, rng)
    tok, offs = wl.prompts()
    ad = _adapters(case, wl.R, rng)
    sub = _random_subsets(wl.R, wl.E, rng)
    k, Pn = 4, len(CASES[case]["profiles"])
    host, chains = gpu.pick_batch_subset(tok, offs, wl.h0, sub, k, adapters=ad, want_chains=True)
    _eq(host, cpu.pick_batch_subset(tok, offs, wl.h0, sub, k, ad), "host subset vs the oracle")
    assert np.array_equal(chains, cpu.hash_batch(tok, offs, wl.h0)[0])
    b = _device_batch(tok, offs, wl.h0, wl.R, k, Pn)
    d_ad = torch.from_numpy(ad.view(np.int64)).cuda() if ad is not None else None
    d_sub = _d_subsets(sub)
    d_chains = torch.zeros(wl.R * wl.max_blocks, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    gpu.pick_batch_device_subset(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), wl.R, tok.nbytes, k, b[3].data_ptr(),
                                 d_sub.data_ptr(), d_chains.data_ptr(), s, d_ad.data_ptr() if d_ad is not None else 0)
    torch.cuda.synchronize()
    dev = b[3].cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, Pn, k)
    _eq(dev, host, "device subset vs host subset")
    assert np.array_equal(d_chains.cpu().numpy().view(np.uint64).reshape(wl.R, wl.max_blocks), chains)
    # NULL device subsets: the ranked device call's bytes
    b2 = _device_batch(tok, offs, wl.h0, wl.R, k, Pn)
    gpu.pick_batch_device_subset(b2[0].data_ptr(), b2[1].data_ptr(), b2[2].data_ptr(), wl.R, tok.nbytes, k,
                                 b2[3].data_ptr(), 0, 0, s, d_ad.data_ptr() if d_ad is not None else 0)
    torch.cuda.synchronize()
    dev0 = b2[3].cpu().numpy().view(H.PICK_DTYPE).reshape(wl.R, Pn, k)
    _eq(dev0, gpu.pick_batch_ranked(tok, offs, wl.h0, k, adapters=ad), "NULL device subsets vs ranked")
    gpu.close()
    cpu.close()


def test_sliced_host_feed_agrees_with_the_unsliced_one():
    """>= 8 MiB of prompts and R >= 64 * slices: the host call copies and matches slice by slice, each slice with its
    own rows of the bitsets"""
    rng = np.random.default_rng(11)
    wl = H.small_workload(E=64, R=2048, T=1100, max_blocks=64, holes=True)
    gpu, cpu = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng)
    tok, offs = wl.prompts()
    assert int(offs[-1]) >= 8 << 20
    sub = _random_subsets(wl.R, wl.E, rng)
    sliced = gpu.pick_batch_subset(tok, offs, wl.h0, sub, 8)
    gpu.set_option("feed_slices", 1)
    whole = gpu.pick_batch_subset(tok, offs, wl.h0, sub, 8)
    _eq(sliced, whole, "sliced vs unsliced feed")
    _eq(whole, cpu.pick_batch_subset(tok, offs, wl.h0, sub, 8), "vs the oracle")
    gpu.close()
    cpu.close()


def test_ops_submits_and_removals_before_a_call_are_seen():
    import torch

    rng = np.random.default_rng(3)
    wl = H.small_workload(E=64, R=256, holes=True)
    gpu, cpu = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng)
    tok, offs = wl.prompts()
    sub = _random_subsets(wl.R, wl.E, rng)
    # index ops submitted right before the call
    chains = cpu.hash_batch(tok, offs, wl.h0)[0]
    ops = H.ops_array([(int(chains[r, 0]), (r * 7) % wl.E, abi.FI_OP_SET) for r in range(0, wl.R, 3)])
    gpu.index_apply(ops)
    cpu.index_apply(ops)
    _eq(gpu.pick_batch_subset(tok, offs, wl.h0, sub, 4), cpu.pick_batch_subset(tok, offs, wl.h0, sub, 4),
        "after index_apply")
    # pipelined submits still in flight
    s = torch.cuda.current_stream().cuda_stream
    batches = [wl.prompts(batch=i) for i in range(3)]
    dev = [_device_batch(t, o, wl.h0, wl.R, 1, 1) for t, o in batches]
    torch.cuda.synchronize()
    for (t, _), b in zip(batches, dev):
        gpu.pick_submit(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), wl.R, t.nbytes, b[3].data_ptr(), s)
    got = gpu.pick_batch_subset(tok, offs, wl.h0, sub, 4)
    gpu.pick_wait(s)
    torch.cuda.synchronize()
    _eq(got, cpu.pick_batch_subset(tok, offs, wl.h0, sub, 4), "after pipelined submits")
    # a removal: asynchronous, the subset call is ordered after it
    victims = sorted(set(int(e) for e in got[:40, 0, 0]["endpoint"] if e != abi.FI_NO_ENDPOINT))
    gpu.remove_endpoints(victims)
    got = gpu.pick_batch_subset(tok, offs, wl.h0, subset_bitsets([None] * wl.R, wl.E), 4)
    _eq(got, gpu.pick_batch_ranked(tok, offs, wl.h0, 4), "all-ones after remove_endpoints vs ranked")
    got = gpu.pick_batch_subset(tok, offs, wl.h0, sub, 4)
    assert not np.isin(got["endpoint"][got["match_blocks"] > 0], victims).any()
    gpu.close()
    cpu.close()


def test_add_chains_device_after_a_subset_call_takes_its_chains():
    """upstream PreRequest after a subset pick: the device LRU adds the chains of the subset call"""
    rng = np.random.default_rng(4)
    wl = H.small_workload(E=40, R=128, lru_capacity=300)
    gpu, cpu = _setup(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng, lru_capacity=300)
    tok, offs = wl.prompts(batch=0)
    sub = _random_subsets(wl.R, wl.E, rng)
    got = gpu.pick_batch_subset(tok, offs, wl.h0, sub, 3)
    _eq(got, cpu.pick_batch_subset(tok, offs, wl.h0, sub, 3), "subset before the Add")
    chains = cpu.hash_batch(tok, offs, wl.h0)[0]
    eps, nb = got[:, 0, 0]["endpoint"], got[:, 0, 0]["n_blocks"]
    gpu.index_add_chains_device(eps, 0, 0, nb)
    cpu.index_add_chains(eps, chains, nb)
    for e in sorted(set(int(x) for x in eps if x != abi.FI_NO_ENDPOINT))[:8]:
        held = gpu.lru_dump(e)
        assert all(cpu.index_contains(e, int(h)) for h in held)
    tok2, offs2 = wl.prompts(batch=1)
    _eq(gpu.pick_batch_subset(tok2, offs2, wl.h0, sub, 3), cpu.pick_batch_subset(tok2, offs2, wl.h0, sub, 3),
        "after the Add")
    gpu.close()
    cpu.close()


def test_bad_arguments_are_rejected():
    wl = H.small_workload(E=40, R=16)
    gpu = EndpointPicker(H.config_for(wl))
    tok, offs = wl.prompts()
    sub = subset_bitsets([None] * wl.R, wl.E)
    for k in (0, abi.FI_EPP_MAX_RANKED + 1):
        with pytest.raises(FiEppError) as ei:
            gpu.pick_batch_subset(tok, offs, wl.h0, sub, k)
        assert ei.value.status == abi.FI_ERR_INVALID
    lib = abi.load()
    tok = np.ascontiguousarray(tok)
    h0 = np.full(wl.R, wl.h0, dtype=np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert lib.fi_epp_pick_batch_subset(gpu._h, p(tok), p(offs), p(h0), None, p(sub), wl.R, 2, None,
                                        None) == abi.FI_ERR_INVALID
    assert lib.fi_epp_pick_batch_device_subset(gpu._h, None, p(offs), p(h0), None, None, wl.R, 0, 2, None, None,
                                               None) == abi.FI_ERR_INVALID
    b = _device_batch(tok, offs, wl.h0, wl.R, 2, 1)
    d_sub = _d_subsets(sub)
    assert lib.fi_epp_pick_batch_device_subset(gpu._h, b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), None,
                                               d_sub.data_ptr(), wl.R + 1, 0, 2, b[3].data_ptr(), None,
                                               None) == abi.FI_ERR_CAPACITY
    assert gpu.pick_batch_subset(tok, offs, wl.h0, sub, abi.FI_EPP_MAX_RANKED).shape == (wl.R, 1, abi.FI_EPP_MAX_RANKED)
    with pytest.raises(ValueError):
        gpu.pick_batch_subset(tok, offs, wl.h0, sub[:, :1].copy() if sub.shape[1] > 1 else sub[:-1], 1)
    gpu.close()


def test_a_handle_over_part_of_the_pool_refuses_subsets():
    wl = H.small_workload(E=300, R=32, holes=True)
    gpu = EndpointPicker(H.config_for(wl, endpoint_begin=100, endpoint_count=150))
    gpu.update_endpoints(wl.endpoint_states())
    tok, offs = wl.prompts()
    with pytest.raises(FiEppError) as ei:
        gpu.pick_batch_subset(tok, offs, wl.h0, subset_bitsets([None] * wl.R, wl.E), 2)
    assert ei.value.status == abi.FI_ERR_STATE
    # without subsets it is the ranked pick, sub-range handles included
    _eq(gpu.pick_batch_subset(tok, offs, wl.h0, None, 2), gpu.pick_batch_ranked(tok, offs, wl.h0, 2), "NULL subsets")
    gpu.close()
