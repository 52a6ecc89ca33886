"""Helpers for handles over part of the pool (docs/SPEC.md S.2e), shared by tests/test_shard_view_cpu.py and
tests/test_gpu_shard_handle.py (test helper, not collected).

A shard's picks compose into the unsharded pool's when the shards' walks agree with the pool's walk (LPM, or
UPSTREAM on a prefix-closed index) and no PD rule runs per shard: each shard's best is the best of its part, and the
best of the parts is taken by (score desc, rotation asc), the rule of the sharded mode's merge."""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.dist import shard_range
from tests import restate
from tests.test_dist_cpu import merge_picks_numpy

NO = abi.FI_NO_ENDPOINT


def splits(E: int):
    """partitions of a pool of E endpoints into [(begin, count)]: even ones from shard_range, and adversarial ones
    (a shard of one endpoint, word-straddling cuts)"""
    out = [[shard_range(E, r, w) for r in range(w)] for w in (2, 3, 5) if w <= E]
    if E > 34:
        out.append([(0, 1), (1, 32), (33, E - 33)])
    if E > 64:
        out.append([(0, 31), (31, 2), (33, E - 34), (E - 1, 1)])
    return out


def starts(chains, nblocks, h0, E: int):
    """every request's tie-rotation start (fi_epp.h "Ties", restated)"""
    h0 = np.broadcast_to(np.asarray(h0, dtype=np.uint64), (len(nblocks),))
    return [restate.tie_start(int(nblocks[r]), int(chains[r, 0]), int(h0[r]), r, E) for r in range(len(nblocks))]


def merge_single(parts, st, E: int):
    """[R, P] picks of each shard -> the pool's [R, P] picks"""
    return merge_picks_numpy([np.ascontiguousarray(p) for p in parts], st, E)


def merge_ranked(parts, st, E: int):
    """[R, P, k] ranked lists of each shard -> the pool's top k per request and profile"""
    out = parts[0].copy()
    R, Pn, k = out.shape
    for r in range(R):
        for p in range(Pn):
            ents = [x for part in parts for x in part[r, p] if x["endpoint"] != NO]
            ents.sort(key=lambda x: (-float(x["score"]), (int(x["endpoint"]) - st[r]) % E))
            n = out[r, p, 0]["n_blocks"]
            for j in range(k):
                out[r, p, j] = ents[j] if j < len(ents) else (NO, 0, n, 0.0)
    return out


def tie_states(E: int, rng, dead: float = 0.15, roles: bool = True):
    """endpoint states with few distinct kv / queue values, so that many endpoints share a zero-match total"""
    st = np.zeros(E, dtype=abi.np_dtypes()[2])
    st["endpoint"] = np.arange(E)
    st["kv_util"] = rng.integers(0, 2, E) * 0.5
    st["queue_depth"] = rng.integers(0, 3, E)
    st["role_mask"] = rng.integers(1, 8, E) if roles else abi.FI_ROLE_WORKER
    st["flags"] = np.where(rng.random(E) < dead, 0, abi.FI_ENDPOINT_ALIVE)
    return st
