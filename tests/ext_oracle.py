"""ctypes wrapper of the CPU oracle's test-side extension (tests/ext_oracle.cpp, built by `make` into build/) — test
infrastructure only.  ExtOracle is the oracle of oracle/epp_oracle.py with:
  * the ranked pick (docs/SPEC.md S.6a): every profile's eligible endpoints ordered by (total desc, the request's tie
    rotation), the first k of them, over each request's candidate subset (S.5a) with pick_batch_subset;
  * per-endpoint LRU capacities (S.2b): its Adds evict against each endpoint's own capacity, set_lru_capacities
    resizes, lru(e) dumps an endpoint's LRU.  remove_endpoints (S.2a) CLEARs every hash ever aimed at an endpoint, so
    the handle has to be created with track_removal=True to use it;
  * the shard view (S.2e), ExtOracle(cfg, shard=(b, c)): what a single-rank handle created with endpoint_begin = b,
    endpoint_count = c computes.  Its index and LRUs hold only pairs of endpoints in [b, b + c): ops, Adds, capacity
    changes and removals addressed elsewhere are dropped.  Its picks (single, LoRA, ranked) rank only the shard's
    eligible endpoints, with the queue scorer's min / max over the eligible endpoints of the whole pool, the tie
    rotation of the whole pool, and the PD rule on the shard's own decode pick;
  * match_counts: fi_epp_match_counts (S.3a), every endpoint's match count of the picks' walk, one column per endpoint
    of the shard (of the pool without one);
  * resize(E'), the pool resize of S.2c: a shrink is remove_endpoints of the tail followed by truncating the
    per-endpoint state, a grow appends fresh endpoints.  A shrink removes, so it needs track_removal=True;
  * the state of an index snapshot (S.2d): state() reads the pair set, every endpoint's LRU (least recently used
    first) and every capacity, and load_state(...) replaces them, leaving endpoint states and adapters as they are.
A shard view refuses resize, state and load_state with ValueError, as the product refuses a handle over part of the
pool."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle
from oracle.epp_oracle import _ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_ext_oracle.so")
_lib = None
_P = C.c_void_p


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_ext_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    # the same epo_* functions: take their signatures from the oracle's binding (ctypes caches each bound function)
    for name, g in vars(epp_oracle.load()).items():
        if name.startswith("epo_"):
            f = getattr(lib, name)
            f.restype, f.argtypes = g.restype, g.argtypes
    for name, res, args in (
            ("epx_create", _P, [C.POINTER(abi.fi_epp_config)]),
            ("epx_destroy", None, [_P]),
            ("epx_set_shard", C.c_int, [_P, C.c_uint32, C.c_uint32]),
            ("epx_pick_batch_ranked", C.c_int, [_P, _P, _P, _P, _P, _P, C.c_uint32, C.c_uint32, _P]),
            ("epx_add_chain", C.c_int, [_P, C.c_uint32, _P, C.c_uint32]),
            ("epx_add_chains", C.c_int, [_P, _P, _P, C.c_uint32, _P, C.c_uint32]),
            ("epx_set_lru_capacities", C.c_int, [_P, _P, _P, C.c_uint32, _P, _P, C.c_uint64, C.POINTER(C.c_uint64)]),
            ("epx_lru_dump", C.c_uint32, [_P, C.c_uint32, _P, C.c_uint32]),
            ("epx_lru_clear", C.c_int, [_P, C.c_uint32]),
            ("epx_match_counts", C.c_int, [_P, _P, _P, _P, C.c_uint32, _P, _P]),
            ("epx_resize", C.c_int, [_P, C.c_uint32]),
            ("epx_index_pairs", C.c_uint64, [_P, _P, _P, C.c_uint64]),
            ("epx_lru_capacities", C.c_int, [_P, _P]),
            ("epx_load_state", C.c_int, [_P, C.c_uint64, _P, _P, _P, _P, _P])):
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    _lib = lib
    return lib


class ExtOracle(epp_oracle.Oracle):
    shard = None  # (b, c) on a shard view

    def __init__(self, cfg: abi.fi_epp_config, track_removal: bool = False, shard=None):
        self._lib = load()
        self.cfg = abi.fi_epp_config.from_buffer_copy(cfg)
        self._h = self._lib.epx_create(C.byref(self.cfg))
        if not self._h:
            raise RuntimeError("epx_create failed (see stderr)")
        self.P = cfg.n_profiles
        self.M = cfg.max_blocks
        self.E = cfg.num_endpoints
        self.C = cfg.lru_capacity
        self._seen = [set() for _ in range(self.E)] if track_removal else None
        if shard is not None:
            b, c = int(shard[0]), int(shard[1])
            if self._lib.epx_set_shard(self._h, b, c) != 0:
                raise ValueError(f"shard {shard} is not a non-empty range of the {self.E} endpoints")
            self.shard = (b, c)

    def mine(self, endpoints) -> np.ndarray:
        """which of the endpoints lie in the shard (all of them without one)"""
        e = np.asarray(endpoints, dtype=np.int64)
        if self.shard is None:
            return np.ones(e.shape, dtype=bool)
        return (e >= self.shard[0]) & (e < self.shard[0] + self.shard[1])

    # ---- the single pick: on a shard view, rank 0 of the ranked pick -------------------------------------------
    def pick_batch(self, prompts, offsets, h0, want_chains=False, nthreads=1, adapters=None):
        if self.shard is None:
            return super().pick_batch(prompts, offsets, h0, want_chains, nthreads, adapters)
        picks = np.ascontiguousarray(self.pick_batch_ranked(prompts, offsets, h0, 1, adapters)[:, :, 0])
        return (picks, self.hash_batch(prompts, offsets, h0)[0]) if want_chains else picks

    def close(self):
        if self._h:
            self._lib.epx_destroy(self._h)
            self._h = None

    # ---- the ranked pick ------------------------------------------------------------------------------------------
    def pick_batch_ranked(self, prompts, offsets, h0, k: int, adapters=None):
        """-> picks [R, n_profiles, k] (PICK_DTYPE)"""
        return self.pick_batch_subset(prompts, offsets, h0, None, k, adapters)

    def pick_batch_subset(self, prompts, offsets, h0, subsets, k: int = 1, adapters=None):
        """subsets: [R, ceil(E / 32)] uint32 bitsets or None -> picks [R, n_profiles, k] (PICK_DTYPE)"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        picks = np.zeros((R, self.P, k), dtype=epp_oracle.PICK_DTYPE)
        ad = None if adapters is None else np.ascontiguousarray(np.broadcast_to(np.asarray(adapters, dtype=np.uint64), (R,)))
        sub = None
        if subsets is not None:
            assert self.shard is None, "a handle over part of the pool takes no subsets"
            sub = np.ascontiguousarray(subsets, dtype=np.uint32)
            assert sub.shape == (R, (self.E + 31) // 32), sub.shape
        rc = self._lib.epx_pick_batch_ranked(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), _ptr(ad), _ptr(sub), R, k,
                                             _ptr(picks))
        assert rc == 0, rc
        return picks

    # ---- per-endpoint LRU capacities --------------------------------------------------------------------------------
    def _see(self, e, hashes):
        if self._seen is not None and self.mine(e):
            self._seen[int(e)].update(int(h) for h in hashes)

    def index_apply(self, ops):
        ops = np.ascontiguousarray(ops, dtype=epp_oracle.OP_DTYPE)
        if self.shard is not None:
            bad = ops["endpoint"] >= self.E
            assert not bad.any(), "index op endpoint out of range"
            ops = np.ascontiguousarray(ops[self.mine(ops["endpoint"])])
        for e in np.unique(ops["endpoint"]):
            self._see(e, ops["hash"][ops["endpoint"] == e])
        super().index_apply(ops)

    def index_add_chain(self, endpoint: int, hashes):
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        self._see(endpoint, hashes)
        rc = self._lib.epx_add_chain(self._h, endpoint, _ptr(hashes), len(hashes))
        assert rc == 0, rc

    def index_add_chains(self, endpoints, chains, nblocks):
        endpoints = np.ascontiguousarray(endpoints, dtype=np.uint32)
        nblocks = np.ascontiguousarray(nblocks, dtype=np.uint32)
        chains = np.ascontiguousarray(chains, dtype=np.uint64)
        if self._seen is not None:
            for r, e in enumerate(endpoints):
                if e != abi.FI_NO_ENDPOINT:
                    self._see(e, chains[r, : nblocks[r]])
        rc = self._lib.epx_add_chains(self._h, _ptr(endpoints), _ptr(chains), chains.shape[1], _ptr(nblocks),
                                      len(endpoints))
        assert rc == 0, rc

    def set_lru_capacities(self, endpoints, capacities):
        """-> the (hash, endpoint) pairs evicted, oldest first per endpoint, endpoints in order of first appearance.
        ValueError (and nothing changes) for the arguments fi_epp_set_lru_capacities rejects with FI_ERR_INVALID."""
        eps = np.ascontiguousarray(np.atleast_1d(np.asarray(endpoints, dtype=np.int64)))
        if (eps < 0).any() or (eps >= self.E).any():
            raise ValueError("endpoint out of range")
        eps = eps.astype(np.uint32)
        caps = np.ascontiguousarray(np.atleast_1d(np.asarray(capacities, dtype=np.uint32)))
        room = int(sum(self.lru_size(int(e)) for e in set(eps.tolist())))
        ev_h = np.zeros(max(room, 1), dtype=np.uint64)
        ev_e = np.zeros(max(room, 1), dtype=np.uint32)
        n = C.c_uint64(0)
        rc = self._lib.epx_set_lru_capacities(self._h, _ptr(eps), _ptr(caps), len(eps), _ptr(ev_h), _ptr(ev_e),
                                              len(ev_h), C.byref(n))
        if rc == abi.FI_ERR_INVALID:
            raise ValueError("invalid endpoint or capacity")
        assert rc == 0, rc
        return [(int(h), int(e)) for h, e in zip(ev_h[: n.value], ev_e[: n.value])]

    def remove_endpoints(self, endpoints):
        """upstream indexer.RemovePod (S.2a): every pair of the endpoints leaves the index, their LRUs become empty and
        keep their capacities"""
        assert self._seen is not None, "create the oracle with track_removal=True"
        for e in {int(x) for x in np.atleast_1d(endpoints)}:
            ops = np.zeros(len(self._seen[e]), dtype=epp_oracle.OP_DTYPE)
            ops["hash"] = sorted(self._seen[e])
            ops["endpoint"] = e
            ops["op"] = abi.FI_OP_CLEAR
            epp_oracle.Oracle.index_apply(self, ops)
            self._seen[e] = set()
            rc = self._lib.epx_lru_clear(self._h, e)
            assert rc == 0, rc

    def lru_size(self, e: int) -> int:
        return int(self._lib.epx_lru_dump(self._h, e, None, 0))

    def lru(self, e: int) -> np.ndarray:
        """endpoint e's keys, least recently used first"""
        n = self.lru_size(e)
        out = np.zeros(max(n, 1), dtype=np.uint64)
        self._lib.epx_lru_dump(self._h, e, _ptr(out), n)
        return out[:n].copy()

    # ---- match counts -----------------------------------------------------------------------------------------------
    def match_counts(self, prompts, offsets, h0):
        """-> (counts uint16 [R, c], nblocks uint32 [R]) of fi_epp_match_counts"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        c = self.E if self.shard is None else self.shard[1]
        counts = np.zeros((R, c), dtype=np.uint16)
        nb = np.zeros(R, dtype=np.uint32)
        rc = self._lib.epx_match_counts(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(counts), _ptr(nb))
        assert rc == 0, rc
        return counts, nb

    # ---- pool resize and snapshot state: a handle over the whole pool -------------------------------------------
    def _whole_pool(self, what):
        if self.shard is not None:
            raise ValueError(f"{what} needs a handle over the whole pool, not a shard view")

    def resize(self, num_endpoints: int) -> int:
        """fi_epp_resize_pool (S.2c).  -> the (endpoint, hash) pairs a shrink removed."""
        self._whole_pool("resize")
        En = int(num_endpoints)
        if En < 1 or En > 4096:
            raise ValueError("num_endpoints out of range")
        removed = 0
        if En < self.E:
            removed = sum(self.index_contains(e, h) for e in range(En, self.E) for h in self._seen[e])
            self.remove_endpoints(range(En, self.E))
        rc = self._lib.epx_resize(self._h, En)
        assert rc == 0, rc
        if self._seen is not None:
            self._seen = self._seen[:En] + [set() for _ in range(En - len(self._seen))]
        self.E = self.cfg.num_endpoints = self.cfg.endpoint_count = En
        return int(removed)

    def index_pairs(self) -> set:
        """{(endpoint, hash)}"""
        n = int(self._lib.epx_index_pairs(self._h, None, None, 0))
        hs = np.zeros(max(n, 1), dtype=np.uint64)
        es = np.zeros(max(n, 1), dtype=np.uint32)
        self._lib.epx_index_pairs(self._h, _ptr(hs), _ptr(es), n)
        return set(zip(es[:n].tolist(), hs[:n].tolist()))

    def capacities(self) -> list:
        out = np.zeros(self.E, dtype=np.uint32)
        self._lib.epx_lru_capacities(self._h, _ptr(out))
        return out.tolist()

    def state(self):
        """(pair set, [LRU of each endpoint, least recently used first], [capacity of each endpoint])"""
        self._whole_pool("state")
        lrus = [self.lru(e) if self.C else np.zeros(0, np.uint64) for e in range(self.E)]
        return self.index_pairs(), lrus, self.capacities()

    def load_state(self, pairs, lrus, caps):
        self._whole_pool("load_state")
        pairs = sorted(pairs)
        es = np.array([e for e, _ in pairs], dtype=np.uint32)
        hs = np.array([h for _, h in pairs], dtype=np.uint64)
        lens = np.array([len(x) for x in lrus], dtype=np.uint32)
        keys = np.concatenate([np.asarray(x, dtype=np.uint64) for x in lrus] + [np.zeros(1, np.uint64)])
        caps = np.ascontiguousarray(caps, dtype=np.uint32)
        rc = self._lib.epx_load_state(self._h, len(pairs), _ptr(hs), _ptr(es), _ptr(lens), _ptr(keys), _ptr(caps))
        assert rc == 0, rc
        if self._seen is not None:
            self._seen = [set() for _ in range(self.E)]
            for e, h in pairs:
                self._seen[e].add(int(h))
            for e, x in enumerate(lrus):
                self._seen[e].update(int(h) for h in x)
