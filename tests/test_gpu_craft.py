"""GPU (-m gpu): picks on crafted chains, bit for bit against the CPU oracle.

tests/craft.py runs the block-hash chain backwards, so a request's h0 can put any value at any block of its prompt
and start its tie rotation at any endpoint.  Random prompts never reach two kinds of input:

  A / B. a block hash of exactly 0 or ~0.  These are the index table's EMPTY / TOMB markers; they own the fixed nodes
     C and C + 1 instead of a slot, and every reader has a branch for them: the speculation and klog check of
     match_kernels.cu resolve_request_nodes, the prefetched home bucket of match_pick, the presence test of index_find,
     the early-exit checker of hash_kernels.cu (whose zero-filled tails must never verify), SET / CLEAR, the index
     rebuild and the device LRU.
  C. a tie rotation that starts at a chosen endpoint: 0, E - 1, either side of a 32-endpoint word boundary, with
     holes at the start, ranked lists that wrap, subsets on both sides of the start.

Every scene asserts that the crafting happened (fi_epp_hash_batch holds the marker where it was put, the index holds
the markers the scene designed, early exit really stopped requests, the rotation really decided), so a scene that
degenerates fails instead of checking nothing.
"""
from collections import OrderedDict

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, make_config, subset_bitsets
from fusioninfer_b200 import _abi as abi
from tests import craft as K
from tests import helpers as H
from tests.ext_oracle import ExtOracle
from tests.test_gpu_early_exit import _big_R
from tests.test_gpu_ranked import CASES, _lora

pytestmark = pytest.mark.gpu
UP, LPM = abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM
MODES = [UP, LPM]
SET, CLEAR = abi.FI_OP_SET, abi.FI_OP_CLEAR
NOEP = abi.FI_NO_ENDPOINT
Z, T = K.MARKERS  # 0 (EMPTY) and ~0 (TOMB)


def _eq(got, want, what):
    assert H.picks_equal(got, want), what + "\n" + H.describe_diff(got, want)


def _ops(triples):
    a = np.zeros(len(triples), dtype=H.OP_DTYPE)
    if triples:
        a["hash"] = np.array([t[0] for t in triples], dtype=np.uint64)
        a["endpoint"] = [t[1] for t in triples]
        a["op"] = [t[2] for t in triples]
    return a


def _contains(gpu, keys, E):
    q = np.zeros(len(keys) * E, dtype=H.OP_DTYPE)
    q["hash"] = np.repeat(np.asarray(keys, dtype=np.uint64), E)
    q["endpoint"] = np.tile(np.arange(E, dtype=np.uint32), len(keys))
    return gpu.index_contains(q).reshape(len(keys), E).astype(bool)


def _check_markers(gpu, ref, E, want=None, what=""):
    """index_contains of 0 and ~0 at every endpoint: the oracle's, and (want: {marker: holders}) the designed one"""
    got = _contains(gpu, [Z, T], E)
    for i, m in enumerate((Z, T)):
        exp = np.array([ref.index_contains(e, m) for e in range(E)])
        assert np.array_equal(got[i], exp), f"{what}: marker {m:#x} held by {np.flatnonzero(got[i])}, oracle " \
                                            f"{np.flatnonzero(exp)}"
        if want is not None:
            assert set(np.flatnonzero(exp).tolist()) == set(want[m]), f"{what}: marker {m:#x} not as designed"


def _torch():
    import torch

    return torch


def _dev(a, dtype=None):
    torch = _torch()
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(dtype) if dtype is not None else a).cuda()


# ---- A. markers on the pick path --------------------------------------------------------------------------------------
# Per marker, who holds it: "one" endpoint, "many", nobody ("none"), SET and CLEARed again ("cleared"), or one endpoint
# with the speculated node free ("L1": the marker is the block right after the last node the index allocated) or
# retired ("L2": a stand-in regular key held that node, then left).  Marker 0 is the one a klog check can confuse with
# a free or retired node (klog == 0); ~0 takes a complementary layout in the same handle.
LAYOUTS = {"held": ("one", "many"), "unheld": ("none", "cleared"), "L1": ("L1", "many"), "L2": ("L2", "one")}
HOLDERS = {Z: {"one": [3], "many": [3, 9, 17, 22, 30, 38], "L1": [3], "L2": [3]},
           T: {"one": [5], "many": [5, 11, 19, 26, 33, 39], "L1": [5], "L2": [5]}}
CHAIN_OWNER = {Z: 3, T: 5}  # the endpoint that holds the regular blocks when nobody holds the marker
E_A, M_A = 40, 128


def _specs():
    """(n_blocks, position, blocks held) per case, for either marker: block 0 (the tie seed and the prefetched bucket),
    interior blocks inside and past the first speculation round, the last block, and the last block of each hashing
    group 8g + 7 with held blocks after it and a miss three blocks before the end; two long prompts whose held
    prefix ends early, so that early exit saves most of their blocks"""
    out = [(12, 0, 12), (20, 5, 15), (100, 70, 90), (33, 32, 33), (128, 3, 8), (128, 20, 24)]
    out += [(8 * g + 16, 8 * g + 7, 8 * g + 13) for g in range(15)]
    return out


class _MarkerScene:
    """One handle, its oracle, and crafted requests: every case of _specs() for both markers, each request's regular
    blocks [0, held) held by the marker's holders (or its chain owner), its first p blocks by a rival endpoint"""

    def __init__(self, B, mode, layout, case="weighted", tail=0, seed=1):
        self.B, self.mode, self.E = B, mode, E_A
        rng = np.random.default_rng(seed * 1000 + B)
        lay = dict(zip((Z, T), LAYOUTS[layout]))
        self.lay = lay
        specs, self.held = [], []
        for m in (Z, T):
            for n, p, held in _specs():
                specs.append((n, p, m))
                self.held.append(held)
        if lay[Z] == "L1":  # the last request: its chain is SET last and ends in the marker
            specs.append((16, 15, Z))
            self.held.append(16)
        self.specs = specs
        self.sc = K.scene(specs, B, rng, tail=tail)
        spec = dict(CASES[case])
        if case == "pd":
            spec["pd"] = dict(spec["pd"], threshold=float(np.median([n for n, _, _ in specs]) * B))
        self.case, self.P = case, len(spec["profiles"])
        R_big = _big_R()
        copies = -(-R_big // self.sc.R)
        self.big = self.sc.tiled(copies)
        self.cfg = make_config(num_endpoints=self.E, block_bytes=B, max_blocks=M_A, lru_capacity=0, max_batch=self.big.R,
                               match_mode=mode, index_slots=1 << 16, max_prompt_bytes=int(self.big.offs[-1]) + 64, **spec)
        self.gpu, self.ref = EndpointPicker(self.cfg), ExtOracle(self.cfg)
        self.gpu.set_option("feed_slices", 1)
        st = H.states_array(self.E, kv=rng.integers(300, 900, self.E) / 1024.0, queue=rng.integers(0, 16, self.E),
                            roles=np.full(self.E, 3))
        for m in (Z, T):
            for e in HOLDERS[m]["many"]:
                st["kv_util"][e], st["queue_depth"][e] = 0.1, 0  # the holders score best: a pick's match_blocks
                # shows the holder's count
        self.gpu.update_endpoints(st)
        self.ref.update_endpoints(st)
        if case == "lora":
            lo = _lora(self.E, rng)
            self.gpu.update_endpoints_lora(lo)
            self.ref.update_endpoints_lora(lo)
        self.rng = rng
        chains, nb = self.ref.hash_batch(self.sc.tok, self.sc.offs, self.sc.h0)
        self.chains = chains
        self._fill(chains)

    def holders(self, m):
        return HOLDERS[m].get(self.lay[m], [])

    def apply(self, triples):
        ops = _ops(triples)
        self.gpu.index_apply(ops)
        self.ref.index_apply(ops)

    def _fill(self, chains):
        """Each request's chain is SET in chain order in a call of its own (< 256 ops: one CTA, consecutive nodes), by
        its first holder; the other holders, the rivals and the markers follow."""
        later, stand_ins = [], []
        for r in range(self.sc.R):  # (the L1 request is the last one: no SET after it claims a new key)
            n, p, m = self.specs[r]
            hs = self.holders(m) or [CHAIN_OWNER[m]]
            first = []
            for j in range(self.held[r]):
                h = int(chains[r, j])
                if j == p:
                    if self.lay[m] == "L2":
                        s = int(self.rng.integers(1, 1 << 62))
                        stand_ins.append(s)
                        first.append((s, hs[0], SET))
                    continue
                first.append((h, hs[0], SET))
            self.apply(first)
            later += [(int(chains[r, j]), e, SET) for e in hs[1:] for j in range(self.held[r]) if j != p]
            rival = (r * 7 + 1) % self.E
            if rival not in HOLDERS[Z]["many"] + HOLDERS[T]["many"]:
                later += [(int(chains[r, j]), rival, SET) for j in range(p)]
        if stand_ins:
            self.apply([(s, HOLDERS[Z]["L2"][0], CLEAR) for s in stand_ins])
        marks = []
        for m in (Z, T):
            marks += [(m, e, SET) for e in self.holders(m)]
            if self.lay[m] == "cleared":
                marks += [(m, e, SET) for e in (1, 2, 4)]
        self.apply(marks)
        if any(self.lay[m] == "cleared" for m in (Z, T)):
            self.apply([(m, e, CLEAR) for m in (Z, T) if self.lay[m] == "cleared" for e in (1, 2, 4)])
        self.apply(later)  # keys already present: no new nodes

    def check_design(self):
        """the GPU's own hashing holds each marker where it was crafted; the index holds the markers as designed"""
        chains, nb = self.gpu.hash_batch(self.sc.tok, self.sc.offs, self.sc.h0)
        for r, (n, p, m) in enumerate(self.specs):
            assert int(nb[r]) == n and int(chains[r, p]) == m, f"request {r}: the marker is not at block {p}"
        _check_markers(self.gpu, self.ref, self.E, {m: self.holders(m) for m in (Z, T)}, "design")

    def check_decisive(self, picks):
        """upstream: each request of a held marker is won by a holder whose count includes the marker"""
        if self.mode != UP or self.case != "weighted":
            return
        for r, (n, p, m) in enumerate(self.specs):
            if self.holders(m):
                assert int(picks[r, 0]["endpoint"]) in self.holders(m), r
                assert int(picks[r, 0]["match_blocks"]) == self.held[r], (r, picks[r, 0])

    def close(self):
        self.gpu.close()
        self.ref.close()


def _entry_points(s, sc, what, big):
    """every pick entry point on one crafted batch, each against the oracle; the early-exit pick also against the
    whole-chain one.  -> the single pick"""
    torch = _torch()
    gpu, ref, tok, offs, h0, R, P = s.gpu, s.ref, sc.tok, sc.offs, sc.h0, sc.R, s.P
    ad = (s.rng.integers(0, 14, R) + 1000).astype(np.uint64) if s.case == "lora" else None
    subsets = [sorted({int(x) for x in s.rng.choice(s.E, 6, replace=False)} | set(s.holders(Z)[:1]) |
                      set(s.holders(T)[-1:])) for _ in range(R)]
    sub = subset_bitsets(subsets, s.E)
    want = ref.pick_batch(tok, offs, h0, adapters=ad)
    if big:
        gpu.set_profiling(True)
        gpu.reset_stats()
    got = gpu.pick_batch(tok, offs, h0, adapters=ad)
    if big:
        st = gpu.stats()
        gpu.set_profiling(False)
        total = int(want[:, 0]["n_blocks"].astype(np.int64).sum())
        assert st.hashed_blocks < total, f"{what}: early exit did not run ({st.hashed_blocks} of {total} blocks)"
    _eq(got, want, f"{what}: pick_batch")
    full, chains = gpu.pick_batch(tok, offs, h0, want_chains=True, adapters=ad)
    _eq(full, got, f"{what}: pick_batch with chains_out vs without")
    assert np.array_equal(chains, ref.hash_batch(tok, offs, h0)[0]), f"{what}: chains_out"
    want_r = ref.pick_batch_ranked(tok, offs, h0, 4, adapters=ad)
    _eq(gpu.pick_batch_ranked(tok, offs, h0, 4, adapters=ad), want_r, f"{what}: ranked k=4")
    want_s = ref.pick_batch_subset(tok, offs, h0, sub, 3, adapters=ad)
    _eq(gpu.pick_batch_subset(tok, offs, h0, sub, 3, adapters=ad), want_s, f"{what}: subset k=3")
    _eq(gpu.pick_batch_subset(tok, offs, h0, sub, 3, adapters=ad, want_chains=True)[0], want_s,
        f"{what}: subset k=3 with chains_out")
    # device buffers: the ranked call with chains_out, the subset call without, pipelined submits of both kinds
    d_tok, d_off, d_h0 = _dev(tok), _dev(offs, np.int64), _dev(h0, np.int64)
    d_ad = _dev(ad, np.int64) if ad is not None else None
    d_sub = _dev(sub, np.int32)
    nbytes = int(offs[-1])
    stream = torch.cuda.current_stream().cuda_stream
    d_out = torch.zeros(R * P * 4 * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(R * M_A, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    gpu.pick_batch_device_ranked(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, 4, d_out.data_ptr(),
                                 d_ch.data_ptr(), stream, d_ad.data_ptr() if d_ad is not None else 0)
    torch.cuda.synchronize()
    _eq(d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, P, 4), want_r, f"{what}: device ranked")
    assert np.array_equal(d_ch.cpu().numpy().view(np.uint64).reshape(R, M_A), chains), f"{what}: device chains_out"
    d_out.zero_()
    gpu.pick_batch_device_subset(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, 3, d_out.data_ptr(),
                                 d_sub.data_ptr(), 0, stream, d_ad.data_ptr() if d_ad is not None else 0)
    torch.cuda.synchronize()
    _eq(d_out.cpu().numpy()[: R * P * 3 * 16].view(H.PICK_DTYPE).reshape(R, P, 3), want_s, f"{what}: device subset")
    outs = [torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda"),
            torch.zeros(R * P * 4 * 16, dtype=torch.uint8, device="cuda")]
    d_ch.zero_()
    t0 = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, outs[0].data_ptr(), k=0,
                            d_adapters=d_ad.data_ptr() if d_ad is not None else 0, stream=stream)
    t1 = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, outs[1].data_ptr(), k=4,
                            d_adapters=d_ad.data_ptr() if d_ad is not None else 0, d_chains=d_ch.data_ptr(),
                            stream=stream)
    assert t1 > t0
    gpu.pick_wait_batch(t1, stream)
    torch.cuda.synchronize()
    _eq(outs[0].cpu().numpy().view(H.PICK_DTYPE).reshape(R, P), want, f"{what}: pick_submit_ex k=0")
    _eq(outs[1].cpu().numpy().view(H.PICK_DTYPE).reshape(R, P, 4), want_r, f"{what}: pick_submit_ex k=4")
    assert np.array_equal(d_ch.cpu().numpy().view(np.uint64).reshape(R, M_A), chains), f"{what}: submit chains_out"
    return want


@pytest.mark.parametrize("case", ["weighted", "pd", "lora"])
@pytest.mark.parametrize("mode", MODES, ids=["upstream", "lpm"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_markers_on_every_pick_path(layout, mode, case):
    """64-byte blocks (hash_chain<2>): whole-SM tiles with whole chains (the distinct requests) and half-SM tiles with
    early exit (the requests tiled past 64 per SM), through every entry point"""
    s = _MarkerScene(64, mode, layout, case)
    s.check_design()
    want = _entry_points(s, s.sc, f"{layout} {case} mode={mode} small", big=False)
    s.check_decisive(want)
    _entry_points(s, s.big, f"{layout} {case} mode={mode} big", big=True)
    s.close()


# (block bytes, junk bytes after each prompt): hash_chain<1>, <4>, run-time stripes, hash_generic, one unaligned feed
SIZES = [(32, 0), (128, 0), (96, 0), (40, 0), (8, 0), (64, 3)]


@pytest.mark.parametrize("mode", MODES, ids=["upstream", "lpm"])
@pytest.mark.parametrize("size", SIZES, ids=[f"B{b}" + ("u" if t else "") for b, t in SIZES])
def test_markers_at_every_block_size(size, mode):
    B, tail = size
    for layout in sorted(LAYOUTS):
        s = _MarkerScene(B, mode, layout, tail=tail, seed=2)
        s.check_design()
        what = f"B={B} tail={tail} {layout} mode={mode}"
        for sc, big in ((s.sc, False), (s.big, True)):
            want = s.ref.pick_batch(sc.tok, sc.offs, sc.h0)
            if big:
                s.gpu.set_profiling(True)
                s.gpu.reset_stats()
            got = s.gpu.pick_batch(sc.tok, sc.offs, sc.h0)
            if big:
                st = s.gpu.stats()
                s.gpu.set_profiling(False)
                if B % 32 == 0:  # hash_chain: early exit (hash_generic hashes whole chains)
                    assert st.hashed_blocks < int(want[:, 0]["n_blocks"].astype(np.int64).sum()), what
            _eq(got, want, what + (" big" if big else " small"))
            _eq(s.gpu.pick_batch(sc.tok, sc.offs, sc.h0, want_chains=True)[0], want, what + " chains_out")
            _eq(s.gpu.pick_batch_ranked(sc.tok, sc.offs, sc.h0, 4), s.ref.pick_batch_ranked(sc.tok, sc.offs, sc.h0, 4),
                what + " ranked")
            if not big:
                s.check_decisive(want)
        s.close()


# ---- B. markers entering the index from hashed chains (device LRU) ------------------------------------------------------
class _Lru:
    """ordered dicts (oldest first) with per-endpoint capacities: hashicorp/golang-lru, plainly"""

    def __init__(self, E, cap):
        self.cap = [cap] * E
        self.d = [OrderedDict() for _ in range(E)]

    def add(self, e, keys):
        d = self.d[e]
        for k in keys:
            k = int(k)
            if k in d:
                d.move_to_end(k)
            else:
                d[k] = True
                while len(d) > self.cap[e]:
                    d.popitem(last=False)

    def resize(self, e, cap):
        self.cap[e] = cap
        while len(self.d[e]) > cap:
            self.d[e].popitem(last=False)

    def clear(self, e):
        self.d[e].clear()


def test_markers_through_the_device_lru_and_two_rebuilds():
    torch = _torch()
    E, C, M, B = 8, 48, 32, 64
    cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=C, max_batch=256, index_slots=1 << 12,
                      profiles=[{"name": "default", "scorers": [(H.P, 100), (H.K, 13), (H.Q, 7)]}])
    gpu, ref, model = EndpointPicker(cfg), ExtOracle(cfg, track_removal=True), _Lru(E, C)
    gpu.set_option("device_lru", 1)
    rng = np.random.default_rng(77)
    st = H.states_array(E, kv=rng.integers(0, 1024, E) / 1024.0, queue=rng.integers(0, 8, E))
    gpu.update_endpoints(st)
    ref.update_endpoints(st)
    sc = K.scene([(n, p, m) for m in (Z, T) for n, p in ((12, 0), (16, 5), (9, 8), (32, 20))], B, rng)
    chains, nb = ref.hash_batch(sc.tok, sc.offs, sc.h0)
    for r, (n, p, m) in enumerate(zip(sc.n, sc.pos, sc.target)):
        assert int(chains[r, p]) == m
    stream = torch.cuda.current_stream().cuda_stream

    def check(what, design=None):
        for e in range(E):
            got = gpu.lru_dump(e)
            assert np.array_equal(got, ref.lru(e)), f"{what}: LRU of endpoint {e} vs the oracle"
            assert np.array_equal(got, np.array(list(model.d[e]), dtype=np.uint64)), f"{what}: LRU {e} vs the model"
        _check_markers(gpu, ref, E, design, what)
        _eq(gpu.pick_batch(sc.tok, sc.offs, sc.h0), ref.pick_batch(sc.tok, sc.offs, sc.h0), f"{what}: picks")
        _eq(gpu.pick_batch_ranked(sc.tok, sc.offs, sc.h0, 3), ref.pick_batch_ranked(sc.tok, sc.offs, sc.h0, 3),
            f"{what}: ranked picks")

    def added(eps, ch, nbk):
        ref.index_add_chains(eps, ch, nbk)
        for r, e in enumerate(eps):
            if e != NOEP:
                model.add(int(e), ch[r, : nbk[r]])

    # 1. the chains_out of a crafted device pick, added through fi_epp_index_add_chains_device
    R = sc.R
    d_tok, d_off, d_h0 = _dev(sc.tok), _dev(sc.offs, np.int64), _dev(sc.h0, np.int64)
    d_out = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(R * M, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(sc.offs[-1]), d_out.data_ptr(),
                          d_ch.data_ptr(), stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_ch.cpu().numpy().view(np.uint64).reshape(R, M), chains)
    eps = np.array([0, 1, 2, 3, 0, 1, 2, 3], dtype=np.uint32)  # requests 0-3 carry marker 0, 4-7 marker ~0
    gpu.index_add_chains_device(eps, d_ch.data_ptr(), M, nb, stream)
    added(eps, chains, nb)
    check("chains_out Add", {Z: [0, 1, 2, 3], T: [0, 1, 2, 3]})
    # 2. a pipelined submit whose chains the handle keeps, added through fi_epp_index_add_submitted
    t = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(sc.offs[-1]), d_out.data_ptr(),
                           stream=stream)
    eps2 = np.array([4, 5, 6, 7, NOEP, 4, NOEP, 6], dtype=np.uint32)
    gpu.index_add_submitted(t, eps2, nb)
    gpu.pick_wait_batch(t, stream)
    torch.cuda.synchronize()
    added(eps2, chains, nb)
    check("submitted Add", {Z: [0, 1, 2, 3, 4, 5, 6, 7], T: [0, 1, 2, 3, 4, 6]})

    def fresh_chains(n_req, n):
        return rng.integers(1, 1 << 63, (n_req, M), dtype=np.uint64), np.full(n_req, n, dtype=np.uint32)

    # 3. later Adds evict the markers from endpoints 0 and 4 (endpoint 1 gets 12 more keys, 44 of its 48)
    ch, nbk = fresh_chains(3, M)
    nbk[2] = 12
    e3 = np.array([0, 4, 1], dtype=np.uint32)
    gpu.index_add_chains(e3, ch, nbk)
    added(e3, ch, nbk)
    ch, nbk = fresh_chains(2, M)
    gpu.index_add_chains(e3[:2], ch, nbk)
    added(e3[:2], ch, nbk)
    check("evicted from 0 and 4", {Z: [1, 2, 3, 5, 6, 7], T: [1, 2, 3, 6]})
    # 4. shrinking endpoint 1 to 32 evicts its 12 oldest keys: request 1's first blocks, marker 0 among them
    gone = gpu.set_lru_capacities([1], [M], want_evicted=True)
    assert gone == len(ref.set_lru_capacities([1], [M])) == 12
    model.resize(1, M)
    check("endpoint 1 shrunk", {Z: [2, 3, 5, 6, 7], T: [1, 2, 3, 6]})
    # 5. removing holders of both markers
    gpu.remove_endpoints([2, 6])
    ref.remove_endpoints([2, 6])
    model.clear(2)
    model.clear(6)
    check("endpoints 2 and 6 removed", {Z: [3, 5, 7], T: [1, 3]})

    # 6. two rebuilds: junk keys SET and CLEARed on endpoint 7 (outside the LRU) fill the table with tombstones
    def churn(what):
        before = gpu.index_stats().rebuilds
        for i in range(12):
            junk = rng.integers(1, 1 << 63, 700, dtype=np.uint64)
            gpu.index_apply(_ops([(int(k), 7, SET) for k in junk]))
            gpu.index_apply(_ops([(int(k), 7, CLEAR) for k in junk]))
            gpu.index_sync()
            if gpu.index_stats().rebuilds > before:
                return
        raise AssertionError(f"{what}: no rebuild")

    churn("first rebuild")
    check("after the first rebuild, markers held", {Z: [3, 5, 7], T: [1, 3]})
    gpu.remove_endpoints([1, 3, 5, 7])
    ref.remove_endpoints([1, 3, 5, 7])
    for e in (1, 3, 5, 7):
        model.clear(e)
    check("markers held by nobody", {Z: [], T: []})
    churn("second rebuild")  # into the spare, whose special rows were live before the first
    check("after the second rebuild, markers held by nobody", {Z: [], T: []})
    assert gpu.index_stats().rebuilds >= 2
    gpu.close()
    ref.close()


# ---- C. the tie rotation started where the test chooses ------------------------------------------------------------------
def _starts(E):
    if E <= 1024:
        return list(range(E))
    return sorted({0, 1, E - 2, E - 1} | {32 * k + d for k in range(1, E // 32) for d in (-1, 0, 1)})


def _rot_order(s, E, ok):
    """the endpoints e with ok[e] (a bool array), in rotated order from s"""
    idx = (s + np.arange(E)) % E
    return idx[ok[idx]].tolist()


@pytest.mark.parametrize("E", [1, 3, 40, 64, 100, 1024, 2048, 4096])
def test_tie_rotation_starts(E):
    """One PD handle (prefill admits every alive endpoint, decode has role holes at 31-33, at the pool's ends and at
    every fifth endpoint, some of them dead), one request per start for each scene: (i)/(ii) cold requests, (iii) a
    prefix held on both sides of the start, (iv) ranked lists, (v) subsets across the start, (vi) requests without
    blocks, (vii) the PD pair.  Every total ties; the rotation alone decides."""
    B, M = 64, 8
    starts = _starts(E)
    S = len(starts)
    rng = np.random.default_rng(E)
    holes = {e for e in range(E) if e % 5 == 0} | {31, 32, 33, E - 1, 1} if E > 3 else set()
    dead = {e for e in holes if e % 2 == 0}
    roles = np.array([1 | (0 if e in holes else 2) for e in range(E)], dtype=np.uint32)
    alive = np.array([0 if e in dead else abi.FI_ENDPOINT_ALIVE for e in range(E)], dtype=np.uint32)
    ok = [(alive != 0) & ((roles & 1) != 0), (alive != 0) & ((roles & 2) != 0)]
    profiles = [{"name": "prefill", "role_mask": 1, "scorers": [(H.P, 100), (H.K, 13), (H.Q, 7)]},
                {"name": "decode", "role_mask": 2, "scorers": [(H.P, 100), (H.K, 13)]}]
    R = 4 * S
    cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=0, max_batch=R, profiles=profiles,
                      pd={"prefill": 0, "decode": 1, "threshold": 0.0}, index_slots=1 << 16)
    gpu, ref = EndpointPicker(cfg), ExtOracle(cfg)
    st = H.states_array(E, roles=roles, alive=alive)  # equal kv and queue everywhere
    gpu.update_endpoints(st)
    ref.update_endpoints(st)
    # requests [0, S): cold; [S, 2S): no blocks; [2S, 3S): a prefix held on both sides; [3S, 4S): cold, with subsets
    blobs, h0, sides = [], [], []
    for q in range(4):
        for i, s in enumerate(starts):
            r = q * S + i
            if q == 1:
                raw, blocks = b"\x07" * (1 + r % (B - 1)), []
            else:
                raw = rng.integers(0, 256, 3 * B, dtype=np.uint8).tobytes()
                blocks = [raw[j * B:(j + 1) * B] for j in range(3)]
            blobs.append(raw)
            h0.append(K.h0_for_start(s, E, r, blocks, low=0x51ED * r + q))  # no two share a first block
    tok, offs = H.pack_prompts(blobs)
    h0 = np.array(h0, dtype=np.uint64)
    chains, nb = ref.hash_batch(tok, offs, h0)
    assert np.array_equal(gpu.hash_batch(tok, offs, h0)[0], chains)
    for r in range(R):  # the crafting happened
        s = starts[r % S]
        seed = int(chains[r, 0]) if nb[r] else int(h0[r]) ^ ((r + 1) * K.GOLDEN & K.MASK64)
        assert K.tie_start(seed, E) == s, (r, s)
    # (iii): the prefix of request 2S + i held by a pair of endpoints around its start, one before and one after
    triples = []
    for i, s in enumerate(starts):
        r = 2 * S + i
        pair = sorted({(s - 1 - i % 3) % E, (s + 2 + i % 5) % E})
        sides.append(pair)
        triples += [(int(chains[r, j]), e, SET) for e in pair for j in range(2)]
    ops = _ops(triples)
    gpu.index_apply(ops)
    ref.index_apply(ops)
    subsets = [None] * (3 * S) + [sorted({(s + d) % E for d in (-3, -1, 1, 4)}) for s in starts]
    sub = subset_bitsets(subsets, E)

    want1 = ref.pick_batch(tok, offs, h0)
    _eq(gpu.pick_batch(tok, offs, h0), want1, f"E={E} pick_batch")
    want_s = ref.pick_batch_subset(tok, offs, h0, sub, 2)
    _eq(gpu.pick_batch_subset(tok, offs, h0, sub, 2), want_s, f"E={E} subset k=2")
    ranked = {}
    for k in (2, 4, 8):
        ranked[k] = ref.pick_batch_ranked(tok, offs, h0, k)
        _eq(gpu.pick_batch_ranked(tok, offs, h0, k), ranked[k], f"E={E} ranked k={k}")

    # the expected winners, computed here: the tied endpoints in rotated order from the start
    for q in range(4):
        for i, s in enumerate(starts):
            r = q * S + i
            for pi in (0, 1):
                if q == 2:
                    held = [e for e in sides[i] if ok[pi][e]]
                    mine = np.isin(np.arange(E), held)
                    order = _rot_order(s, E, mine) + _rot_order(s, E, ok[pi] & ~mine)
                elif q == 3:
                    order = _rot_order(s, E, ok[pi] & np.isin(np.arange(E), subsets[r]))
                else:
                    order = _rot_order(s, E, ok[pi])
                exp = order[0] if order else NOEP
                got = want_s[r, pi, 0]["endpoint"] if q == 3 else want1[r, pi]["endpoint"]
                assert int(got) == exp, f"E={E} scene {q} start {s} profile {pi}: {int(got)} != {exp}"
                if q != 3:
                    for k in (2, 4, 8):
                        lst = [int(x) for x in ranked[k][r, pi, :]["endpoint"]]
                        assert lst == (order[:k] + [NOEP] * k)[:k], f"E={E} scene {q} start {s} k={k}"
                        if q == 2 and len(held) == 2 and k == 2:  # the pair really tied
                            sc = ranked[k][r, pi, :]["score"]
                            assert sc[0] == sc[1] and ranked[k][r, pi, 0]["match_blocks"] == 2
    # the cold scenes tied: one total for every decided request of a profile
    for pi in (0, 1):
        cold = want1[: 2 * S, pi]
        cold = cold[cold["endpoint"] != NOEP]
        assert len(np.unique(cold["score"])) <= 1 and (cold["match_blocks"] == 0).all()
    # the ranked lists wrap from E - 1 to 0 somewhere
    if E >= 8:
        lst = ranked[8][:S, 0, :]["endpoint"].astype(np.int64)
        assert any((np.diff(row[row != NOEP]) < 0).any() for row in lst)
    # the device and pipelined entry points on the same batch
    torch = _torch()
    d_tok, d_off, d_h0 = _dev(tok), _dev(offs, np.int64), _dev(h0, np.int64)
    d_out = torch.zeros(R * 2 * 4 * 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    t = gpu.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(offs[-1]), d_out.data_ptr(), k=4,
                           stream=stream)
    gpu.pick_wait_batch(t, stream)
    torch.cuda.synchronize()
    _eq(d_out.cpu().numpy().view(H.PICK_DTYPE).reshape(R, 2, 4), ranked[4], f"E={E} pick_submit_ex k=4")
    d_out.zero_()
    gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, int(offs[-1]), d_out.data_ptr(), 0,
                          stream)
    torch.cuda.synchronize()
    _eq(d_out.cpu().numpy()[: R * 2 * 16].view(H.PICK_DTYPE).reshape(R, 2), want1, f"E={E} pick_batch_device")
    gpu.close()
    ref.close()
