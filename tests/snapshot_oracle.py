"""ctypes wrapper of tests/snapshot_oracle.cpp (built by `make` into build/) — test infrastructure only.
SnapshotOracle is the ResizeOracle of tests/resize_oracle.py plus the state of an index snapshot (docs/SPEC.md S.2d):
state() reads the pair set, every endpoint's LRU (least recently used first) and every capacity, and load_state(...)
replaces them, leaving endpoint states and adapters as they are."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle.epp_oracle import _ptr
from tests import resize_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_snapshot_oracle.so")
_lib = None
_P = C.c_void_p


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_snapshot_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    # the same epo_* / epx_* functions: take their signatures from the resize extension's binding
    for name, g in vars(resize_oracle.load()).items():
        if name.startswith(("epo_", "epx_")):
            f = getattr(lib, name)
            f.restype, f.argtypes = g.restype, g.argtypes
    for name, res, args in (("epx_index_pairs", C.c_uint64, [_P, _P, _P, C.c_uint64]),
                            ("epx_lru_capacities", C.c_int, [_P, _P]),
                            ("epx_load_state", C.c_int, [_P, C.c_uint64, _P, _P, _P, _P, _P])):
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    _lib = lib
    return lib


class SnapshotOracle(resize_oracle.ResizeOracle):
    def __init__(self, cfg: abi.fi_epp_config, track_removal: bool = False):
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
        lrus = [self.lru(e) if self.C else np.zeros(0, np.uint64) for e in range(self.E)]
        return self.index_pairs(), lrus, self.capacities()

    def load_state(self, pairs, lrus, caps):
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
