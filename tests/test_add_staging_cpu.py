"""CPU: how fi_epp_index_add_chains stages the host LRU's ops (plan_staging, lru_batch.h).

The GPU applies an op group as all its SETs, then all its CLEARs.  The batched host Add copies its ops into the open
group segment by segment and flushes when a buffer is full or a segment ends; its tail stays staged for the next call.
Checked through libfi_hostcheck.so: the plan against a model of that walk, and the groups of consecutive calls,
applied SETs-then-CLEARs, against sequential Adds.
"""
import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H

LIB = os.path.join(abi.LIB_DIR, "libfi_hostcheck.so")


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(LIB)
    V, U32, U64 = C.c_void_p, C.c_uint32, C.c_uint64
    lib.fihc_plan_staging.restype = U64
    lib.fihc_plan_staging.argtypes = [U32, U32, V, V, U64, U64, U64, V, U64, V, U64, V]
    lib.fihc_lrupool_new.restype = V
    lib.fihc_lrupool_new.argtypes = [U32, U32, U32]
    lib.fihc_lrupool_free.argtypes = [V]
    lib.fihc_lrupool_stage.restype = U64
    lib.fihc_lrupool_stage.argtypes = [V, V, V, U32, V, U32, U64, U64, U64, V, V, U64, V]
    return lib


def _walk_model(counts, wseg, ns0, nc0, chunk):
    """the staging loop fi_epp_index_add_chains ran before plan_staging, plus a leading flush when CLEARs are staged:
    groups of (pieces, n_sets, n_clears), a piece = (worker, seg, clear, src, n, dst)"""
    W, nseg = counts.shape[0], counts.shape[1]
    groups, cur, fill = [], [], [ns0, nc0]

    def flush():
        nonlocal cur
        groups.append((cur, fill[0], fill[1]))
        cur = []
        fill[0] = fill[1] = 0

    if nc0:
        flush()
    for seg in range(nseg):
        for kind in range(2):
            for w in range(W):
                if wseg[w] <= seg:
                    continue
                n, done = int(counts[w, seg, kind]), 0
                while done < n:
                    take = min(chunk - fill[kind], n - done)
                    cur.append((w, seg, kind, done, take, fill[kind]))
                    fill[kind] += take
                    done += take
                    if fill[kind] == chunk:
                        flush()
        if seg + 1 < nseg and (fill[0] or fill[1]):
            flush()
    groups.append((cur, fill[0], fill[1]))
    return groups


def _plan(hc, counts, wseg, ns0, nc0, chunk):
    W, nseg = counts.shape[0], counts.shape[1]
    cap = int(counts.sum()) + 16
    pieces = np.zeros((cap, 7), np.uint64)
    fills = np.zeros((cap, 2), np.uint64)
    npieces = C.c_uint64(0)
    c = np.ascontiguousarray(counts, dtype=np.uint64)
    ws = np.ascontiguousarray(wseg, dtype=np.uint32)
    ng = hc.fihc_plan_staging(W, nseg, ws.ctypes.data, c.ctypes.data, ns0, nc0, chunk, pieces.ctypes.data, cap,
                              fills.ctypes.data, cap, C.byref(npieces))
    assert ng <= cap and npieces.value <= cap
    groups = [([], int(fills[g, 0]), int(fills[g, 1])) for g in range(ng)]
    for row in pieces[: npieces.value]:
        groups[int(row[0])][0].append(tuple(int(x) for x in row[1:]))
    return groups


@pytest.mark.parametrize("seed", range(6))
def test_plan_matches_walk_model(hc, seed):
    """random op counts over several workers and segments, nonzero starting fills, a small chunk: the same flushes,
    group contents and tail as the walk the planner replaced"""
    rng = np.random.default_rng(seed)
    chunk = int(rng.choice([3, 7, 16]))
    for _ in range(60):
        W, nseg = int(rng.integers(1, 5)), int(rng.integers(0, 5))
        wseg = rng.integers(0, nseg + 1, size=W)
        counts = rng.integers(0, 3 * chunk, size=(W, max(nseg, 1), 2))[:, :nseg]
        counts[rng.random(counts.shape) < 0.3] = 0
        ns0, nc0 = int(rng.integers(0, chunk)), int(rng.choice([0, int(rng.integers(0, chunk))]))
        got = _plan(hc, counts, wseg, ns0, nc0, chunk)
        assert got == _walk_model(counts, wseg, ns0, nc0, chunk)
        if nc0:
            assert got[0] == ([], ns0, nc0)  # the leading flush


class _Index:
    """the GPU index as op groups reach it (a group: its SETs, then its CLEARs), with the open group of the engine"""

    def __init__(self):
        self.pairs = set()
        self.sets, self.clears = [], []

    def stage(self, ops, group, n_groups):
        for g in range(n_groups):
            for h, e, o in ops[group == g]:
                (self.sets if o == abi.FI_OP_SET else self.clears).append((int(e), int(h)))
            if g + 1 < n_groups:
                self.flush()

    def flush(self):
        self.pairs |= set(self.sets)
        self.pairs -= set(self.clears)
        self.sets, self.clears = [], []

    def view(self):
        """what a pick sees: the pick flushes the open group first"""
        return (self.pairs | set(self.sets)) - set(self.clears)


class _Lrus:
    def __init__(self, E, cap):
        self.cap, self.lru, self.pairs = cap, [OrderedDict() for _ in range(E)], set()

    def add_chain(self, e, keys):
        d = self.lru[e]
        for k in (int(x) for x in keys):
            if k in d:
                d.move_to_end(k)
                continue
            d[k] = True
            self.pairs.add((e, k))
            if len(d) > self.cap:
                self.pairs.discard((e, d.popitem(last=False)[0]))


def _add_chains(hc, pool, index, eps, chains, nb, chunk, leading_flush=True):
    """one fi_epp_index_add_chains: its groups go to `index` (leading_flush=False: the old rule, which staged the
    call's ops behind the open group's CLEARs without a flush)"""
    R, pitch = chains.shape
    cap = 2 * R * pitch + 16
    ops = np.zeros(cap, dtype=H.OP_DTYPE)
    group = np.zeros(cap, np.uint32)
    ng = C.c_uint64(0)
    nc0 = len(index.clears) if leading_flush else 0
    n = hc.fihc_lrupool_stage(pool, eps.ctypes.data, chains.ctypes.data, pitch, nb.ctypes.data, R, len(index.sets), nc0,
                              chunk, ops.ctypes.data, group.ctypes.data, cap, C.byref(ng))
    assert n <= cap
    index.stage(ops[:n], group[:n], ng.value)


def _one(e, keys, pitch):
    chains = np.zeros((1, pitch), np.uint64)
    chains[0, : len(keys)] = keys
    return np.array([e], np.uint32), chains, np.array([len(keys)], np.uint32)


@pytest.mark.parametrize("leading_flush", [True, False])
def test_clear_in_tail_then_re_set(hc, leading_flush):
    """a call evicts (1, e) and leaves the CLEAR in its tail; the next call adds key 1 again: only the leading flush
    keeps the pair in the index"""
    pool = hc.fihc_lrupool_new(1, 2, 1)
    index, model = _Index(), _Lrus(1, 2)
    for keys in ([1, 2, 3], [1]):
        _add_chains(hc, pool, index, *_one(0, keys, 3), chunk=1 << 16, leading_flush=leading_flush)
        model.add_chain(0, keys)
    hc.fihc_lrupool_free(pool)
    assert model.pairs == {(0, 3), (0, 1)}
    if leading_flush:
        assert index.view() == model.pairs
    else:
        assert index.view() == {(0, 3)}  # the CLEAR staged before the SET wins in the shared group


@pytest.mark.parametrize("workers", [1, 4])
def test_consecutive_calls_match_sequential_adds(hc, workers):
    """several calls in a row with nothing flushed between them (hot endpoints, re-added evictions, small chunk): after
    every call the index holds exactly the pairs of sequential Adds"""
    E, cap, mb, R, chunk = 6, 8, 6, 12, 16
    rng = np.random.default_rng(workers)
    pool = hc.fihc_lrupool_new(E, cap, workers)
    index, model = _Index(), _Lrus(E, cap)
    for step in range(40):
        hot = int(rng.integers(0, E))
        eps = np.where(rng.random(R) < 0.5, hot, rng.integers(0, E, size=R)).astype(np.uint32)
        eps[rng.random(R) < 0.05] = abi.FI_NO_ENDPOINT
        chains = rng.integers(1, 16, size=(R, mb), dtype=np.uint64)
        nb = rng.integers(0, mb + 1, size=R).astype(np.uint32)
        _add_chains(hc, pool, index, eps, chains, nb, chunk)
        for r in range(R):
            if eps[r] != abi.FI_NO_ENDPOINT:
                model.add_chain(int(eps[r]), chains[r, : nb[r]])
        assert index.view() == model.pairs, step
    hc.fihc_lrupool_free(pool)
