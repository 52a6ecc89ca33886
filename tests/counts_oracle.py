"""ctypes wrapper of tests/counts_oracle.cpp (built by `make` into build/) — test infrastructure only.  CountsOracle is
the ExtOracle of tests/ext_oracle.py, shard view included, plus match_counts: fi_epp_match_counts (docs/SPEC.md S.3a),
every endpoint's match count of the picks' walk, one column per endpoint of the shard (of the pool without one)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle.epp_oracle import _ptr
from tests import ext_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_counts_oracle.so")
_lib = None
_P = C.c_void_p


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_counts_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    # the same epo_* / epx_* functions: take their signatures from the extension's binding
    for name, g in vars(ext_oracle.load()).items():
        if name.startswith(("epo_", "epx_")):
            f = getattr(lib, name)
            f.restype, f.argtypes = g.restype, g.argtypes
    lib.epx_match_counts.restype = C.c_int
    lib.epx_match_counts.argtypes = [_P, _P, _P, _P, C.c_uint32, _P, _P]
    _lib = lib
    return lib


class CountsOracle(ext_oracle.ExtOracle):
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

    def match_counts(self, prompts, offsets, h0):
        """-> (counts uint16 [R, c], nblocks uint32 [R]) of fi_epp_match_counts"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        c = self.E if self.shard is None else self.shard[1]
        counts = np.zeros((R, c), dtype=np.uint16)
        nb = np.zeros(R, dtype=np.uint32)
        rc = self._lib.epx_match_counts(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(counts), _ptr(nb))
        assert rc == 0, rc
        return counts, nb
