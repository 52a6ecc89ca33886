"""ctypes wrapper of tests/resize_oracle.cpp (built by `make` into build/) — test infrastructure only.  ResizeOracle is
the ExtOracle of tests/ext_oracle.py plus resize(E'), the pool resize of docs/SPEC.md S.2c: a shrink is remove_endpoints
of the tail followed by truncating the per-endpoint state, a grow appends fresh endpoints.  A shrink removes, so the
handle has to be created with track_removal=True to shrink."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from fusioninfer_b200 import _abi as abi
from tests import ext_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_resize_oracle.so")
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_resize_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    # the same epo_* / epx_* functions: take their signatures from the extension's binding
    for name, g in vars(ext_oracle.load()).items():
        if name.startswith(("epo_", "epx_")):
            f = getattr(lib, name)
            f.restype, f.argtypes = g.restype, g.argtypes
    lib.epx_resize.restype, lib.epx_resize.argtypes = C.c_int, [C.c_void_p, C.c_uint32]
    _lib = lib
    return lib


class ResizeOracle(ext_oracle.ExtOracle):
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

    def resize(self, num_endpoints: int) -> int:
        """fi_epp_resize_pool (S.2c).  -> the (endpoint, hash) pairs a shrink removed."""
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
