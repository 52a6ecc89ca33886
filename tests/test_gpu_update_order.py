"""GPU (-m gpu): the device work of every kind of index update, pinned.

One fixed sequence of calls runs on a device-LRU handle and on a host-LRU handle (device_lru = 0): index_apply,
index_add_chain, index_add_chains, index_add_chains_device(.., NULL, ..) and pick_submit_ex + index_add_submitted
(device LRU only), set_lru_capacities lowering and raising capacities, index_remove_endpoints, resize_pool shrinking
and growing (device LRU only), an index filled with tombstones until the next update rebuilds it, and picks of every
kind between them.  After each call the deltas of fi_epp_get_stats' kernel_launches, h2d_bytes and d2h_bytes must be
the pinned ones below, and index membership (index_contains) and every pick must equal the oracle extension's
(tests/resize_oracle.py).

The pinned deltas are what the library gave before every update was ordered through update_begin / update_end
(engine_index.cu), measured by running this file with FI_EPP_LIB=<that build of libfi_epp.so>: the same kernels and the
same copies in the same order.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.resize_oracle import ResizeOracle

pytestmark = pytest.mark.gpu
P, K, Q = H.P, H.K, H.Q
PROFILES = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]
E, R, MB, CAP, KR = 40, 64, 32, 120, 4
SLOTS = 1 << 14

# (call, kernel launches, H2D bytes, D2H bytes) of the sequence, per device_lru
PINNED = {
    1: [
        ('index_apply', 1, 48000, 0), ('pick_batch', 3, 133064, 1024), ('index_add_chain', 8, 600, 0),
        ('index_add_chains', 8, 17988, 0), ('index_contains', 1, 0, 0), ('pick_batch', 2, 132104, 1024),
        ('index_add_chains_device', 8, 1604, 0), ('pick_batch_device', 2, 0, 0), ('pick_submit_ex k', 2, 0, 0),
        ('pick_submit_ex', 2, 0, 0), ('index_add_submitted', 8, 1604, 0), ('index_contains', 1, 0, 0),
        ('set_lru_capacities lower', 2, 192, 0), ('pick_batch', 2, 132104, 1024),
        ('set_lru_capacities raise', 0, 160, 0), ('pick_batch', 2, 132104, 1024), ('index_add_chains', 8, 17988, 0),
        ('index_remove_endpoints', 2, 8, 0), ('index_contains', 1, 0, 0), ('resize_pool shrink', 3, 32, 0),
        ('pick_batch', 3, 137480, 1024), ('index_contains', 1, 0, 0), ('resize_pool grow', 1, 0, 0),
        ('pick_batch', 3, 142280, 1024), ('index_add_chains', 8, 17988, 0), ('index_apply tombstones', 2, 293472, 0),
        ('index_apply rebuild', 2, 8000, 0), ('index_contains', 1, 0, 0), ('pick_batch', 2, 132104, 1024),
        ('pick_batch_ranked', 2, 132104, 4096), ('pick_batch_subset', 2, 132616, 4096), ('pick_batch_device', 2, 0, 0),
        ('pick_submit_ex k', 2, 0, 0), ('pick_submit_ex', 2, 0, 0), ('index_add_submitted', 16, 1928, 0),
        ('index_contains', 1, 0, 0),
    ],
    0: [
        ('index_apply', 1, 48000, 0), ('pick_batch', 3, 133064, 1024), ('index_add_chain', 0, 0, 0),
        ('index_add_chains', 8, 43312, 0), ('index_contains', 3, 2864, 0), ('pick_batch_device', 2, 0, 0),
        ('pick_submit_ex k', 2, 0, 0), ('pick_submit_ex', 2, 0, 0), ('index_contains', 1, 0, 0),
        ('set_lru_capacities lower', 0, 0, 0), ('pick_batch', 3, 135432, 1024), ('set_lru_capacities raise', 0, 0, 0),
        ('pick_batch', 2, 132104, 1024), ('index_add_chains', 22, 46752, 0), ('index_remove_endpoints', 3, 2768, 0),
        ('index_contains', 1, 0, 0), ('index_apply tombstones', 2, 203296, 0), ('index_apply rebuild', 2, 8000, 0),
        ('index_contains', 1, 0, 0), ('pick_batch', 2, 132104, 1024), ('pick_batch_ranked', 2, 132104, 4096),
        ('pick_batch_subset', 2, 132616, 4096), ('pick_batch_device', 2, 0, 0), ('pick_submit_ex k', 2, 0, 0),
        ('pick_submit_ex', 2, 0, 0), ('index_contains', 1, 0, 0),
    ],
}


def _torch():
    import torch

    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a).view(np.uint8).ravel().copy()).cuda()


class _Seq:
    """a handle and the oracle fed the same calls; log = the stats deltas of every call to the handle"""

    def __init__(self, device_lru):
        self.wl = H.small_workload(E=E, R=R, T=512, max_blocks=MB, lru_capacity=0)
        cfg = H.config_for(self.wl, profiles=PROFILES, lru_capacity=CAP, index_slots=SLOTS)
        self.g, self.o = EndpointPicker(cfg), ResizeOracle(cfg, track_removal=True)
        self.g.set_option("device_lru", device_lru)
        self.st = self.wl.endpoint_states()
        self.g.update_endpoints(self.st)
        self.o.update_endpoints(self.st)
        self.E, self.h0 = E, np.full(R, self.wl.h0, dtype=np.uint64)
        self.rng = np.random.default_rng(7)
        self.ever = set()
        self.log = []

    def call(self, what, f, *args, **kw):
        a = self.g.stats()
        r = f(*args, **kw)
        b = self.g.stats()
        self.log.append((what, b.kernel_launches - a.kernel_launches, b.h2d_bytes - a.h2d_bytes, b.d2h_bytes - a.d2h_bytes))
        return r

    def both(self, what, name, *args):
        self.call(what, getattr(self.g, name), *args)
        getattr(self.o, name)(*args)

    def batch(self, b):
        tok, offs = self.wl.prompts(batch=b)
        chains, nb = self.o.hash_batch(tok, offs, self.h0)
        for r in range(R):
            self.ever.update(int(x) for x in chains[r, : nb[r]])
        return tok, offs, chains, nb

    def pick(self, what, b):
        """a host pick of batch b -> its inputs, the oracle's chains and the picked endpoints"""
        tok, offs, chains, nb = self.batch(b)
        got = self.call(what, self.g.pick_batch, tok, offs, self.h0)
        want = self.o.pick_batch(tok, offs, self.h0)
        assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)
        return tok, offs, chains, nb, got[:, 0]["endpoint"].copy()

    def members(self, what):
        hashes = np.array(sorted(self.ever), dtype=np.uint64)
        hashes = hashes[self.rng.permutation(len(hashes))[:1500]]
        q = np.zeros(len(hashes) * self.E, dtype=H.OP_DTYPE)
        q["hash"] = np.repeat(hashes, self.E)
        q["endpoint"] = np.tile(np.arange(self.E, dtype=np.uint32), len(hashes))
        got = self.call(what, self.g.index_contains, q)
        want = np.array([self.o.index_contains(int(e), int(h)) for h, e in zip(q["hash"], q["endpoint"])], dtype=np.uint8)
        assert np.array_equal(got, want), f"{what}: {int((got != want).sum())} of {len(q)} memberships differ"
        assert want.any()

    def device_picks(self, b, device_lru):
        """pick_batch_device and pick_submit_ex (k = 0, and k = KR with subsets) of batch b; on the device LRU the
        submitted batch is then added with index_add_submitted"""
        torch = _torch()
        tok, offs, chains, nb = self.batch(b)
        sub = subset_bitsets([self.rng.choice(self.E, [1, 8, self.E // 2][r % 3], replace=False).tolist()
                              for r in range(R)], self.E)
        d = [_dev(tok), _dev(offs), _dev(self.h0), _dev(sub)]
        out = torch.empty(R * KR * 16, dtype=torch.uint8, device="cuda")
        p = [x.data_ptr() for x in d]

        def read(k):
            torch.cuda.synchronize()
            return out[: R * max(k, 1) * 16].cpu().numpy().view(H.PICK_DTYPE).reshape((R, 1, k) if k else (R, 1))

        want = self.o.pick_batch(tok, offs, self.h0)
        self.call("pick_batch_device", self.g.pick_batch_device, p[0], p[1], p[2], R, tok.nbytes, out.data_ptr())
        got = read(0)
        assert H.picks_equal(got, want), "pick_batch_device\n" + H.describe_diff(got, want)
        want_sub = self.o.pick_batch_subset(tok, offs, self.h0, sub, KR)
        t = self.call("pick_submit_ex k", self.g.pick_submit_ex, p[0], p[1], p[2], R, tok.nbytes, out.data_ptr(), k=KR,
                      d_subsets=p[3])
        self.g.pick_wait_batch(t)
        got = read(KR)
        assert H.picks_equal(got, want_sub), "pick_submit_ex k\n" + H.describe_diff(got, want_sub)
        t = self.call("pick_submit_ex", self.g.pick_submit_ex, p[0], p[1], p[2], R, tok.nbytes, out.data_ptr())
        self.g.pick_wait_batch(t)
        got = read(0)
        assert H.picks_equal(got, want), "pick_submit_ex\n" + H.describe_diff(got, want)
        if device_lru:
            eps = got[:, 0]["endpoint"].copy()
            self.call("index_add_submitted", self.g.index_add_submitted, t, eps, nb)
            self.o.index_add_chains(eps, chains, nb)

    def host_picks(self, b):
        tok, offs, _, _ = self.batch(b)
        sub = subset_bitsets([self.rng.choice(self.E, [2, self.E // 3][r % 2], replace=False).tolist()
                              for r in range(R)], self.E)
        for what, f, args in (("pick_batch_ranked", "pick_batch_ranked", (KR,)),
                               ("pick_batch_subset", "pick_batch_subset", (sub, KR))):
            got = self.call(what, getattr(self.g, f), tok, offs, self.h0, *args)
            want = getattr(self.o, f)(tok, offs, self.h0, *args)
            assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)

    def close(self):
        self.g.close()
        self.o.close()


@pytest.mark.parametrize("device_lru", [1, 0])
def test_update_device_work_is_pinned(device_lru):
    s = _Seq(device_lru)
    g = s.g
    ops = next(iter(s.wl.index_ops()))[:3000]
    s.ever.update(int(x) for x in ops["hash"])
    s.both("index_apply", "index_apply", ops)
    tok, offs, chains, nb, eps = s.pick("pick_batch", 0)
    s.both("index_add_chain", "index_add_chain", int(eps[0]), chains[0, : nb[0]].copy())
    s.both("index_add_chains", "index_add_chains", eps, chains, nb)
    s.members("index_contains")
    if device_lru:
        tok, offs, chains, nb, eps = s.pick("pick_batch", 1)
        s.call("index_add_chains_device", g.index_add_chains_device, eps, 0, 0, nb)
        s.o.index_add_chains(eps, chains, nb)
    s.device_picks(2, device_lru)
    s.members("index_contains")
    low = [3, 7, 11, 19, int(eps[1])]
    s.both("set_lru_capacities lower", "set_lru_capacities", low, [MB] * len(low))
    s.pick("pick_batch", 3)
    s.both("set_lru_capacities raise", "set_lru_capacities", low, [0] * len(low))
    _, _, chains, nb, eps = s.pick("pick_batch", 4)
    s.both("index_add_chains", "index_add_chains", eps, chains, nb)
    s.both("index_remove_endpoints", "remove_endpoints", [5, int(eps[2])])
    s.members("index_contains")
    if device_lru:
        removed = s.call("resize_pool shrink", g.resize_pool, E - 8, count=True)
        assert removed == s.o.resize(E - 8)
        s.E = E - 8
        s.pick("pick_batch", 5)
        s.members("index_contains")
        s.call("resize_pool grow", g.resize_pool, E)
        s.o.resize(E)
        s.E = E
        for x in (g, s.o):
            x.update_endpoints(s.st)
        _, _, chains, nb, eps = s.pick("pick_batch", 6)
        s.both("index_add_chains", "index_add_chains", eps, chains, nb)
    # fill the index with tombstones past its rebuild threshold (70% of the slots used, at most 60% live): the SETs and
    # CLEARs of fresh keys in one group, then the next update rebuilds
    st0 = g.index_stats()
    fresh = s.rng.integers(1, 2**63, int(SLOTS * 0.7) - st0.used + 200, dtype=np.int64).astype(np.uint64)
    tight = np.zeros(2 * len(fresh), dtype=H.OP_DTYPE)
    tight["hash"] = np.concatenate([fresh, fresh])
    tight["endpoint"] = 9
    tight["op"] = [abi.FI_OP_SET] * len(fresh) + [abi.FI_OP_CLEAR] * len(fresh)
    s.both("index_apply tombstones", "index_apply", tight)
    s.both("index_apply rebuild", "index_apply", ops[:500])
    assert g.index_stats().rebuilds == st0.rebuilds + 1
    s.members("index_contains")
    s.pick("pick_batch", 7)
    s.host_picks(8)
    s.device_picks(9, device_lru)
    s.members("index_contains")
    log = s.log
    s.close()
    assert log == PINNED[device_lru], "stats deltas per call:\n" + repr(log)
