"""ctypes wrapper of the capacity CPU oracle (tests/capacity_oracle.cpp, built by `make` into build/) — test
infrastructure only.  CapacityOracle is the oracle of oracle/epp_oracle.py with per-endpoint LRU capacities
(docs/SPEC.md S.2b): its Adds evict against each endpoint's own capacity, set_lru_capacities resizes, lru(e) dumps an
endpoint's LRU.  remove_endpoints (S.2a) CLEARs every hash ever aimed at an endpoint, so the handle has to be created
with track_removal=True to use it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_capacity_oracle.so")
_lib = None
_P = C.c_void_p


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_capacity_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    base = epp_oracle.load()  # the same epo_* functions: take their signatures from the oracle's binding
    for name in ("epo_endpoints_update", "epo_endpoints_lora_update", "epo_index_reserve", "epo_index_apply",
                 "epo_index_keys", "epo_index_contains", "epo_hash_batch", "epo_pick_batch", "epo_pick_batch_lora"):
        f, g = getattr(lib, name), getattr(base, name)
        f.restype, f.argtypes = g.restype, g.argtypes
    lib.epo_cap_create.restype = _P
    lib.epo_cap_create.argtypes = [C.POINTER(abi.fi_epp_config)]
    lib.epo_cap_destroy.restype = None
    lib.epo_cap_destroy.argtypes = [_P]
    lib.epo_cap_add_chain.restype = C.c_int
    lib.epo_cap_add_chain.argtypes = [_P, C.c_uint32, _P, C.c_uint32]
    lib.epo_cap_add_chains.restype = C.c_int
    lib.epo_cap_add_chains.argtypes = [_P, _P, _P, C.c_uint32, _P, C.c_uint32]
    lib.epo_cap_set_lru_capacities.restype = C.c_int
    lib.epo_cap_set_lru_capacities.argtypes = [_P, _P, _P, C.c_uint32, _P, _P, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.epo_cap_lru_dump.restype = C.c_uint32
    lib.epo_cap_lru_dump.argtypes = [_P, C.c_uint32, _P, C.c_uint32]
    lib.epo_cap_lru_clear.restype = None
    lib.epo_cap_lru_clear.argtypes = [_P, C.c_uint32]
    _lib = lib
    return lib


class CapacityOracle(epp_oracle.Oracle):
    def __init__(self, cfg: abi.fi_epp_config, track_removal: bool = False):
        self._lib = load()
        self.cfg = abi.fi_epp_config.from_buffer_copy(cfg)
        self._h = self._lib.epo_cap_create(C.byref(self.cfg))
        if not self._h:
            raise RuntimeError("epo_cap_create failed (see stderr)")
        self.P = cfg.n_profiles
        self.M = cfg.max_blocks
        self.E = cfg.num_endpoints
        self.C = cfg.lru_capacity
        self._seen = [set() for _ in range(self.E)] if track_removal else None

    def close(self):
        if self._h:
            self._lib.epo_cap_destroy(self._h)
            self._h = None

    def _see(self, e, hashes):
        if self._seen is not None:
            self._seen[int(e)].update(int(h) for h in hashes)

    def index_apply(self, ops):
        ops = np.ascontiguousarray(ops, dtype=epp_oracle.OP_DTYPE)
        for e in np.unique(ops["endpoint"]):
            self._see(e, ops["hash"][ops["endpoint"] == e])
        super().index_apply(ops)

    def index_add_chain(self, endpoint: int, hashes):
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        self._see(endpoint, hashes)
        rc = self._lib.epo_cap_add_chain(self._h, endpoint, epp_oracle._ptr(hashes), len(hashes))
        assert rc == 0, rc

    def index_add_chains(self, endpoints, chains, nblocks):
        endpoints = np.ascontiguousarray(endpoints, dtype=np.uint32)
        nblocks = np.ascontiguousarray(nblocks, dtype=np.uint32)
        chains = np.ascontiguousarray(chains, dtype=np.uint64)
        if self._seen is not None:
            for r, e in enumerate(endpoints):
                if e != abi.FI_NO_ENDPOINT:
                    self._see(e, chains[r, : nblocks[r]])
        rc = self._lib.epo_cap_add_chains(self._h, epp_oracle._ptr(endpoints), epp_oracle._ptr(chains), chains.shape[1],
                                          epp_oracle._ptr(nblocks), len(endpoints))
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
        rc = self._lib.epo_cap_set_lru_capacities(self._h, epp_oracle._ptr(eps), epp_oracle._ptr(caps), len(eps),
                                                  epp_oracle._ptr(ev_h), epp_oracle._ptr(ev_e), len(ev_h), C.byref(n))
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
            self._lib.epo_cap_lru_clear(self._h, e)

    def lru_size(self, e: int) -> int:
        return int(self._lib.epo_cap_lru_dump(self._h, e, None, 0))

    def lru(self, e: int) -> np.ndarray:
        """endpoint e's keys, least recently used first"""
        n = self.lru_size(e)
        out = np.zeros(max(n, 1), dtype=np.uint64)
        self._lib.epo_cap_lru_dump(self._h, e, epp_oracle._ptr(out), n)
        return out[:n].copy()
