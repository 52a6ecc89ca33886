"""GPU (-m gpu): handle lifecycle.  Several handles are created, driven through every buffer group a handle allocates
on first use (both pipeline slots, both fi_epp_index_add_submitted buffers, the device LRU and its resize staging, the
removal buffer, the diagnostics temporaries, the ranked and subset staging, the spare index tables, the trace event and
the event pool) and closed, one after another in one process.  Every call must succeed, and every handle must return
what the first one returned on the same inputs, whichever LRU serves it.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.test_gpu_ranked import _device_batch

pytestmark = pytest.mark.gpu

E, R, CAP, HOT = 16, 160, 64, 3
PROFILES = [{"name": "default", "scorers": [(H.P, 100), (H.K, 10), (H.Q, 10)]}]


def _route(picks):
    """the endpoints the batch is added to: half of it to one endpoint, many times the touch bound"""
    eps = picks[:, 0]["endpoint"].copy()
    eps[: R // 2] = HOT
    return eps, picks[:, 0]["n_blocks"].astype(np.uint32)


def _session(wl, device_lru):
    """one handle's whole life -> what its calls returned, by call"""
    import torch

    cfg = H.config_for(wl, profiles=PROFILES, lru_capacity=CAP, index_slots=4096, max_prompt_bytes=wl.R * wl.T * 4)
    got = {}
    g = EndpointPicker(cfg)
    g.set_option("device_lru", device_lru)
    g.update_endpoints(wl.endpoint_states())
    host = [wl.prompts(batch=i) for i in range(4)]
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream

    # pipelined submits in both slots; their chains also come back for the host LRU's Adds
    dev = [_device_batch(tok, offs, wl.h0, R, 1, 1) for tok, offs in host[:2]]
    chains = [torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda") for _ in dev]
    tickets = [g.pick_submit_ex(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), R, host[i][0].nbytes, d[3].data_ptr(),
                                d_chains=chains[i].data_ptr(), stream=s) for i, d in enumerate(dev)]
    g.pick_wait_batch(tickets[1], s)
    stream.synchronize()
    for i, d in enumerate(dev):
        picks = d[3].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        got[f"submit {i}"] = picks
        eps, nb = _route(picks)
        if device_lru:
            g.index_add_submitted(tickets[i], eps, nb)  # Add j stages through buffer j & 1
        else:
            g.index_add_chains(eps, chains[i].cpu().numpy().view(np.uint64).reshape(R, wl.max_blocks), nb)

    # a stream-ordered pick and the Add of its chains from host memory
    picks, ch = g.pick_batch(*host[2], wl.h0, want_chains=True)
    got["pick 2"] = picks
    eps, nb = _route(picks)
    g.index_add_chains(eps, ch, nb)

    got["evicted"] = g.set_lru_capacities([HOT, 0, 1], [wl.max_blocks] * 3, want_evicted=True)
    assert got["evicted"] > 0, "the shrink must evict"
    got["removed"] = g.remove_endpoints([5], count=True)
    if device_lru:
        got["lru dump"] = g.lru_dump(HOT)
    got["contains"] = g.index_contains(H.ops_array(
        [(int(ch[r, j]), int(eps[r]), abi.FI_OP_SET) for r in range(R) if eps[r] != abi.FI_NO_ENDPOINT
         for j in range(int(nb[r]))]))

    got["ranked"] = g.pick_batch_ranked(*host[3], wl.h0, k=4)
    rng = np.random.default_rng(7)
    bits = subset_bitsets([rng.choice(E, size=5, replace=False) for _ in range(R)], E)
    got["subset"] = g.pick_batch_subset(*host[3], wl.h0, bits, k=2)

    # SET / CLEAR churn: tombstones until the index is rebuilt into its spare tables
    rng = np.random.default_rng(11)
    for _ in range(20):
        keys, owners = rng.integers(1, 2**63, size=500, dtype=np.uint64), rng.integers(0, E, size=500)
        for op in (abi.FI_OP_SET, abi.FI_OP_CLEAR):
            g.index_apply(H.ops_array([(int(k), int(e), op) for k, e in zip(keys, owners)]))
        g.index_sync()
        if g.index_stats().rebuilds:
            break
    assert g.index_stats().rebuilds >= 1
    got["pick 3"] = g.pick_batch(*host[3], wl.h0)
    g.index_sync()  # reports a broken device-LRU invariant, if any
    g.close()
    return got


def test_handles_allocate_everything_and_close_one_after_another(monkeypatch):
    wl = H.small_workload(E=E, R=R, T=600, max_blocks=32, lru_capacity=CAP)
    first = _session(wl, device_lru=1)
    runs = {"again": lambda: _session(wl, device_lru=1), "host LRU": lambda: _session(wl, device_lru=0)}

    def traced():
        monkeypatch.setenv("FI_EPP_TRACE", "0")  # read at create: the first three submits are traced
        try:
            return _session(wl, device_lru=1)
        finally:
            monkeypatch.delenv("FI_EPP_TRACE")

    runs["traced"] = traced
    for name, run in runs.items():
        got = run()
        for what, want in first.items():
            if what == "lru dump" and what not in got:
                continue  # the host LRU has no device LRU to dump
            if isinstance(want, np.ndarray):
                assert want.tobytes() == got[what].tobytes(), f"{name}: {what} differs from the first handle's"
            else:
                assert want == got[what], f"{name}: {what} differs from the first handle's"
