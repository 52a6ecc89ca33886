"""Shared helpers for the tests (host side only; no GPU needed to import)."""
from __future__ import annotations

import json
import os
from collections import OrderedDict

import numpy as np

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import make_config, synth

HERE = os.path.dirname(os.path.abspath(__file__))
PICK_DTYPE, OP_DTYPE, ENDPOINT_DTYPE = abi.np_dtypes()
P, K, Q = abi.FI_SCORER_PREFIX, abi.FI_SCORER_KV_UTIL, abi.FI_SCORER_QUEUE


def golden():
    with open(os.path.join(HERE, "golden", "xxh64_chain_golden.json")) as f:
        return json.load(f)


def pack_prompts(blobs):
    """list of bytes -> (uint8 array, offsets uint64 [R+1])"""
    offs = np.zeros(len(blobs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for b in blobs])
    data = np.frombuffer(b"".join(blobs) + b"\0" * 16, dtype=np.uint8).copy()
    return data, offs


def ops_array(triples):
    """[(hash, endpoint, op)] -> OP_DTYPE array"""
    a = np.zeros(len(triples), dtype=OP_DTYPE)
    for i, (h, e, o) in enumerate(triples):
        a[i] = (h, e, o)
    return a


def states_array(E, kv=None, queue=None, roles=None, alive=None):
    s = np.zeros(E, dtype=ENDPOINT_DTYPE)
    s["endpoint"] = np.arange(E)
    s["kv_util"] = 0.0 if kv is None else kv
    s["queue_depth"] = 0 if queue is None else queue
    s["role_mask"] = abi.FI_ROLE_WORKER if roles is None else roles
    s["flags"] = abi.FI_ENDPOINT_ALIVE if alive is None else alive
    return s


def picks_equal(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def describe_diff(got, want, limit=5):
    bad = np.argwhere((got["endpoint"] != want["endpoint"]) | (got["match_blocks"] != want["match_blocks"])
                      | (got["n_blocks"] != want["n_blocks"]) | (got["score"].view(np.uint64) != want["score"].view(np.uint64)))
    lines = [f"{len(bad)} of {got.size} picks differ"]
    for idx in bad[:limit]:
        i = tuple(idx)
        lines.append(f"  {i}: got {got[i]} want {want[i]}")
    return "\n".join(lines)


class OrderedLrus:
    """hashicorp/golang-lru, the plainest way: one ordered dict per endpoint (lru[e], oldest first) with its own
    capacity (cap[e], C until resized), and the index as the set of (endpoint, hash) pairs"""

    def __init__(self, E, cap):
        self.C = cap
        self.cap = [cap] * E
        self.lru = [OrderedDict() for _ in range(E)]
        self.pairs = set()

    def apply(self, ops):
        """direct SET / CLEAR ops [(hash, endpoint, op)]: the pair set only"""
        for h, e, o in ops:
            (self.pairs.add if o == abi.FI_OP_SET else self.pairs.discard)((int(e), int(h)))

    def add_chain(self, e, keys):
        """upstream indexer.Add: a hit becomes the most recent, a miss is inserted and SET, evicting (and CLEARing)
        the oldest key past the capacity"""
        e, d = int(e), self.lru[int(e)]
        for k in (int(x) for x in keys):
            if k in d:
                d.move_to_end(k)
                continue
            d[k] = True
            self.pairs.add((e, k))
            if len(d) > self.cap[e]:
                old, _ = d.popitem(last=False)
                self.pairs.discard((e, old))

    def resize(self, e, c):
        """capacity c (0: C) -> the keys evicted, oldest first"""
        self.cap[e] = c or self.C
        d, gone = self.lru[e], []
        while len(d) > self.cap[e]:
            old, _ = d.popitem(last=False)
            self.pairs.discard((e, old))
            gone.append(old)
        return gone

    def remove(self, eps):
        """upstream indexer.RemovePod: every pair of the endpoints leaves and their LRUs empty -> pairs dropped"""
        drop = {int(e) for e in eps}
        gone = {p for p in self.pairs if p[0] in drop}
        self.pairs -= gone
        for e in drop:
            self.lru[e].clear()
        return len(gone)


def small_workload(**kw):
    base = dict(R=128, E=40, T=512, seed=synth.SEEDS[1], max_blocks=32, lru_capacity=400)
    base.update(kw)
    return synth.Workload(**base)


def config_for(wl, profiles=None, pd=None, match_mode=abi.FI_MATCH_UPSTREAM, **kw):
    profiles = profiles or [{"name": "default", "scorers": [(P, 100)]}]
    slots = 4096
    while slots < 4 * wl.E * max(wl.lru_capacity, wl.groups_per_endpoint * wl.n_blocks):
        slots *= 2
    args = dict(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=0,
                max_batch=max(wl.R, 1), profiles=profiles, pd=pd, match_mode=match_mode, index_slots=slots)
    args.update(kw)
    return make_config(**args)
