"""GPU (-m gpu): several threads and several handles on one GPU at once.

ctypes releases the GIL around every library call, so Python threads run the library concurrently.  Every thread's
script is generated up front from a seed and the oracle's results are computed in the main thread before the threads
start; results are compared, bit for bit, after every thread has joined.

* One handle per thread, several handles on one device: configurations whose match kernels need different amounts of
  shared memory (all above 48 KiB) but share the same variants (one pool-width class), so their launches race on the
  variants' shared-memory opt-in.  The same scripts also run interleaved step by step on one thread, which separates
  "interleaving" from "concurrency" when a case fails.
* Several threads on one handle: each thread owns a slice of the endpoints and its own chain seed, so that its keys
  never meet another thread's; its picks then equal an oracle fed only its own script.
"""
import ctypes as C
import threading

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests.ext_oracle import ExtOracle
from tests.test_gpu_ranked import _lora, _states

pytestmark = pytest.mark.gpu
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
PROFILES = [{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5), (Q, 5)]}]
R, STEPS, KR = 32, 6, 3


def _torch():
    import torch

    return torch


def _dev(a, dtype=np.int64):
    return _torch().from_numpy(np.ascontiguousarray(a).view(dtype).ravel().copy()).cuda()


def _eq(got, want, what):
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)


def _run(scripts, threaded):
    """every script's steps, each script on its own thread (threaded) or all interleaved step by step on this one"""
    errors = []

    def body(sc, steps):
        try:
            for i in steps:
                sc.step(i)
        except Exception as e:  # pragma: no cover - reported below
            errors.append(f"{sc.name}: {type(e).__name__}: {e}")

    if threaded:
        ths = [threading.Thread(target=body, args=(sc, range(STEPS))) for sc in scripts]
        for t in ths:
            t.start()
        for t in ths:
            t.join(timeout=600)
        assert not any(t.is_alive() for t in ths), "a thread did not finish"
    else:
        for i in range(STEPS):
            for sc in scripts:
                body(sc, [i])
    assert not errors, "\n".join(errors)


class Script:
    """One thread's calls on handle g: per step, host picks of every variant, a device pick on the thread's own
    stream, a pipelined submit_ex -> wait_batch -> add_submitted, index_apply and index_add_chains, all on endpoints
    `mine` with prompts of chain seed h0.  `oracle` is fed the same calls in the main thread, which records every
    expected result before any thread starts."""

    def __init__(self, name, g, oracle, wl, mine, h0, seed, batch0=0, removals=False, capacities=False):
        torch = _torch()
        self.name, self.g, self.mine = name, g, np.asarray(mine, dtype=np.uint32)
        rng = np.random.default_rng(seed)
        E = int(g.cfg.num_endpoints)
        self.max_blocks = int(g.cfg.max_blocks)
        self.stream = torch.cuda.Stream()
        self.steps, self.want, self.got, self.pairs = [], [], [], set()
        for i in range(STEPS):
            tok, offs = wl.prompts(batch=batch0 + i)
            hv = np.full(R, h0, dtype=np.uint64)
            ad = (rng.integers(0, 14, R) + 1000).astype(np.uint64)
            sub = subset_bitsets([rng.choice(self.mine, min(len(self.mine), [1, 4, 64][r % 3]), replace=False).tolist()
                                  for r in range(R)], E)
            chains, nb = oracle.hash_batch(tok, offs, hv)
            # Adds go to the first half of the endpoints, direct SET / CLEAR ops to the second: a direct CLEAR of a
            # pair the endpoint's LRU still holds is left out (the LRU does not re-SET it on a later touch)
            adds, direct = self.mine[: (len(self.mine) + 1) // 2], self.mine[(len(self.mine) + 1) // 2:]
            eps = rng.choice(adds, R).astype(np.uint32)
            eps2 = rng.choice(adds, R).astype(np.uint32)
            ops = H.ops_array([(int(chains[r, j]), int(rng.choice(direct)), abi.FI_OP_SET if r % 3 else abi.FI_OP_CLEAR)
                               for r in range(0, R, 4) for j in range(int(nb[r]) // 2)])
            st = dict(tok=tok, offs=offs, h0=hv, ad=ad, sub=sub, chains=chains, nb=nb, eps=eps, eps2=eps2, ops=ops,
                      remove=rng.choice(self.mine, 2, replace=False).astype(np.uint32) if removals and i % 3 == 2 else None,
                      caps=(rng.choice(self.mine, 3, replace=False).astype(np.uint32),
                            np.uint32(self.max_blocks) if i % 2 == 0 else np.uint32(0)) if capacities else None,
                      d=[_dev(tok, np.int32), _dev(offs), _dev(hv), _dev(ad)],
                      out=torch.zeros(R * 16, dtype=torch.uint8, device="cuda"),
                      out2=torch.zeros(R * 16, dtype=torch.uint8, device="cuda"))
            # the oracle, in the order step() makes the calls
            w = {"lora": oracle.pick_batch(tok, offs, hv, adapters=ad),
                 "ranked": oracle.pick_batch_ranked(tok, offs, hv, KR, adapters=ad),
                 "subset": oracle.pick_batch_subset(tok, offs, hv, sub, KR, adapters=ad)}
            w["device"] = w["submit"] = w["lora"]
            oracle.index_add_chains(eps, chains, nb)
            oracle.index_apply(ops)
            oracle.index_add_chains(eps2, chains, nb)
            if st["remove"] is not None:
                oracle.remove_endpoints(st["remove"])
            if st["caps"] is not None:
                oracle.set_lru_capacities(st["caps"][0], np.full(3, st["caps"][1], dtype=np.uint32))
            for e, x in ((eps, chains), (eps2, chains)):
                self.pairs.update((int(x[r, j]), int(e[r])) for r in range(R) for j in range(int(nb[r])))
            self.pairs.update((int(o["hash"]), int(o["endpoint"])) for o in ops)
            self.steps.append(st)
            self.want.append(w)
        self.late_adds = 0  # add_submitted refused (FI_ERR_STATE) and replaced by index_add_chains

    def step(self, i):
        g, st, s = self.g, self.steps[i], self.stream
        tok, offs, hv, ad = st["tok"], st["offs"], st["h0"], st["ad"]
        got = {"lora": g.pick_batch(tok, offs, hv, adapters=ad),
               "ranked": g.pick_batch_ranked(tok, offs, hv, KR, adapters=ad),
               "subset": g.pick_batch_subset(tok, offs, hv, st["sub"], KR, adapters=ad)}
        d = [x.data_ptr() for x in st["d"]]
        lib = abi.load()
        g._check(lib.fi_epp_pick_batch_device_lora(g._h, d[0], d[1], d[2], d[3], R, tok.nbytes, st["out"].data_ptr(),
                                                    None, s.cuda_stream), "fi_epp_pick_batch_device_lora")
        t = g.pick_submit_ex(d[0], d[1], d[2], R, tok.nbytes, st["out2"].data_ptr(), d_adapters=d[3], stream=s.cuda_stream)
        g.pick_wait_batch(t, s.cuda_stream)
        s.synchronize()
        got["device"] = st["out"].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        got["submit"] = st["out2"].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        # the raw call: fi_epp_last_error is not meaningful while other threads use the handle
        eps, nb = np.ascontiguousarray(st["eps"]), np.ascontiguousarray(st["nb"])
        rc = lib.fi_epp_index_add_submitted(g._h, t, eps.ctypes.data_as(C.c_void_p), nb.ctypes.data_as(C.c_void_p), R)
        if rc == abi.FI_ERR_STATE:  # the batch's chains were reclaimed by later submits, or it was not pipelined
            self.late_adds += 1
            g.index_add_chains(eps, st["chains"], nb)
        elif rc != abi.FI_OK:
            raise AssertionError(f"fi_epp_index_add_submitted: status {rc}")
        g.index_apply(st["ops"])
        g.index_add_chains(st["eps2"], st["chains"], nb)
        if st["remove"] is not None:
            g.remove_endpoints(st["remove"])
        if st["caps"] is not None:
            g.set_lru_capacities(st["caps"][0], np.full(3, st["caps"][1], dtype=np.uint32))
        self.got.append(got)

    def check(self, oracle, what, picks=True):
        if picks:
            assert len(self.got) == STEPS, f"{self.name}: {len(self.got)} of {STEPS} steps ran"
            for i, (got, want) in enumerate(zip(self.got, self.want)):
                for k in want:
                    _eq(got[k], want[k], f"{what}, {self.name} step {i}: {k}")
        q = H.ops_array([(h, e, abi.FI_OP_SET) for h, e in sorted(self.pairs)])
        want = np.array([oracle.index_contains(e, h) for h, e in sorted(self.pairs)], dtype=np.uint8)
        assert np.array_equal(self.g.index_contains(q), want), f"{what}, {self.name}: index membership"
        for e in self.mine.tolist():
            assert np.array_equal(self.g.lru_dump(e), oracle.lru(e)), f"{what}, {self.name}: LRU of endpoint {e}"


# (max_blocks, block_bytes, match mode, pool size): match smem 8 * MP * 20 bytes is 160, 80 and 50 KiB; every pool
# is 33..64 endpoints, so all of them launch the same match variants
HANDLES = [(1023, 64, abi.FI_MATCH_UPSTREAM, 64), (512, 32, abi.FI_MATCH_LPM, 48), (320, 40, abi.FI_MATCH_UPSTREAM, 40),
           (1023, 32, abi.FI_MATCH_LPM, 56)]


@pytest.mark.parametrize("threaded", [True, False], ids=["threads", "interleaved"])
def test_handles_on_one_device(threaded):
    """one handle per thread, four handles with different match shared-memory sizes on one GPU"""
    torch = _torch()
    scripts, oracles = [], []
    for n, (mb, bb, mode, E) in enumerate(HANDLES):
        wl = H.small_workload(E=E, R=R, T=600, max_blocks=mb, block_tokens=bb // 4, holes=True, lru_capacity=mb + 64,
                              seed=0xA110 + n)
        cfg = H.config_for(wl, profiles=PROFILES, match_mode=mode, lru_capacity=mb + 64, max_prompt_bytes=R * wl.T * 4)
        g, o = EndpointPicker(cfg), ExtOracle(cfg)
        rng = np.random.default_rng(n)
        st, lo = _states(wl, rng, roles=False), _lora(E, rng)
        for x in (g, o):
            x.update_endpoints(st)
            x.update_endpoints_lora(lo)
            for ops in wl.index_ops():
                x.index_apply(ops)
        scripts.append(Script(f"handle {n} (max_blocks {mb}, block_bytes {bb})", g, o, wl, range(E), wl.h0, n))
        oracles.append(o)
    torch.cuda.synchronize()
    _run(scripts, threaded)
    torch.cuda.synchronize()
    for sc, o in zip(scripts, oracles):
        sc.check(o, "threads" if threaded else "interleaved")
        # only the handle whose block size is not a multiple of 32 serves its submits stream-ordered
        assert (sc.late_adds > 0) == (sc.g.cfg.block_bytes % 32 != 0), sc.name
        sc.g.close()
        o.close()


@pytest.mark.parametrize("threaded", [True, False], ids=["threads", "interleaved"])
def test_threads_on_one_handle(threaded):
    """four threads on one handle, each on its own endpoints and keys, with removals, capacity changes and a small
    index that rebuilds during the run; a reader thread polls the counters.  Between two such phases the main thread
    grows the pool."""
    torch = _torch()
    T, E, cap, mb = 4, 96, 64, 32
    wl = H.small_workload(E=E, R=R, T=600, max_blocks=mb, holes=True, lru_capacity=cap)
    # about 35 000 keys pass through an index of 16 384 slots, at most about 7 000 of them live: tombstones force rebuilds
    cfg = H.config_for(wl, profiles=PROFILES, lru_capacity=cap, max_prompt_bytes=R * wl.T * 4, index_slots=16384)
    g = EndpointPicker(cfg)
    rng = np.random.default_rng(7)
    st, lo = _states(wl, rng, roles=False), _lora(E, rng)
    g.update_endpoints(st)
    g.update_endpoints_lora(lo)
    oracles = []
    for t in range(T):  # each oracle: the common state, then only thread t's calls
        o = ExtOracle(cfg, track_removal=True)
        o.update_endpoints(st)
        o.update_endpoints_lora(lo)
        oracles.append(o)
    slices = [range(t * E // T, (t + 1) * E // T) for t in range(T)]
    seeds = [0x5EED0000 + t for t in range(T)]
    torch.cuda.synchronize()
    stop = threading.Event()

    def reader():
        while not stop.is_set():
            g.index_stats()
            g.lru_counters()
            g.stats()

    for phase in range(2):
        scripts = [Script(f"thread {t}", g, oracles[t], wl, slices[t], seeds[t], 100 + t + 10 * phase, batch0=10 * phase,
                          removals=True, capacities=True) for t in range(T)]
        torch.cuda.synchronize()
        stop.clear()
        rd = threading.Thread(target=reader)
        rd.start()
        try:
            _run(scripts, threaded)
        finally:
            stop.set()
            rd.join()
        torch.cuda.synchronize()
        for sc, o in zip(scripts, oracles):
            sc.check(o, f"phase {phase}")
        assert g.index_stats().lru_entries == sum(o.lru_size(e) for o in oracles for e in range(o.E))
        if phase == 0:
            g.resize_pool(E + 40)
            for o in oracles:
                o.resize(E + 40)
            for sc, o in zip(scripts, oracles):
                sc.check(o, "after the resize", picks=False)
    assert g.index_stats().rebuilds > 0
    g.index_sync()
    g.close()
    for o in oracles:
        o.close()
