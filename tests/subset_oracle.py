"""ctypes wrapper of the subset CPU oracle (tests/subset_oracle.cpp, built by `make` into build/) — test
infrastructure only.  SubsetOracle is the oracle of oracle/epp_oracle.py with one more call, pick_batch_subset: the
ranked pick of docs/SPEC.md S.6a over each request's candidate subset (S.5a)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "build", "libepp_subset_oracle.so")
_lib = None
_P = C.c_void_p


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        subprocess.run(["make", "-C", ROOT, "build/libepp_subset_oracle.so"], check=True, capture_output=True)
    lib = C.CDLL(LIB_PATH)
    base = epp_oracle.load()  # the same epo_* functions: take their signatures from the oracle's binding
    for name in ("epo_create", "epo_destroy", "epo_endpoints_update", "epo_endpoints_lora_update", "epo_index_reserve",
                 "epo_index_apply", "epo_index_add_chain", "epo_index_add_chains", "epo_index_keys",
                 "epo_index_contains", "epo_hash_batch", "epo_pick_batch", "epo_pick_batch_lora"):
        f, g = getattr(lib, name), getattr(base, name)
        f.restype, f.argtypes = g.restype, g.argtypes
    lib.epo_pick_batch_subset.restype = C.c_int
    lib.epo_pick_batch_subset.argtypes = [_P, _P, _P, _P, _P, _P, C.c_uint32, C.c_uint32, _P]
    _lib = lib
    return lib


class SubsetOracle(epp_oracle.Oracle):
    def __init__(self, cfg: abi.fi_epp_config):
        self._lib = load()
        self.cfg = abi.fi_epp_config.from_buffer_copy(cfg)
        self._h = self._lib.epo_create(C.byref(self.cfg))
        if not self._h:
            raise RuntimeError("epo_create failed (see stderr)")
        self.P = cfg.n_profiles
        self.M = cfg.max_blocks
        self.E = cfg.num_endpoints

    def pick_batch_subset(self, prompts, offsets, h0, subsets, k: int = 1, adapters=None):
        """subsets: [R, ceil(E / 32)] uint32 bitsets or None -> picks [R, n_profiles, k] (PICK_DTYPE)"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        picks = np.zeros((R, self.P, k), dtype=epp_oracle.PICK_DTYPE)
        ad = None if adapters is None else np.ascontiguousarray(np.broadcast_to(np.asarray(adapters, dtype=np.uint64), (R,)))
        sub = None
        if subsets is not None:
            sub = np.ascontiguousarray(subsets, dtype=np.uint32)
            assert sub.shape == (R, (self.E + 31) // 32), sub.shape
        rc = self._lib.epo_pick_batch_subset(self._h, epp_oracle._ptr(prompts), epp_oracle._ptr(offsets),
                                             epp_oracle._ptr(h0), epp_oracle._ptr(ad), epp_oracle._ptr(sub), R, k,
                                             epp_oracle._ptr(picks))
        assert rc == 0, rc
        return picks
