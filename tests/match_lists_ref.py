"""The reference of fi_epp_match_lists (docs/SPEC.md S.3b): the match-count matrix of fi_epp_match_counts made sparse,
shared by tests/test_match_lists_cpu.py and tests/test_gpu_match_lists.py (test helper, not collected)."""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi

ENTRY = abi.match_entry_dtype()


def sparsify(counts: np.ndarray, begin: int = 0):
    """[R, c] uint16 counts -> (list_offsets uint64 [R + 1], entries ENTRY [nnz]): request r's non-zero columns j in
    ascending order as (begin + j, counts[r, j])"""
    counts = np.asarray(counts)
    r, j = np.nonzero(counts)  # row-major: rows ascending, columns ascending within a row
    off = np.zeros(counts.shape[0] + 1, dtype=np.uint64)
    np.cumsum(np.count_nonzero(counts, axis=1), out=off[1:])
    ent = np.zeros(len(r), dtype=ENTRY)
    ent["endpoint"] = j + begin
    ent["match_blocks"] = counts[r, j]
    return off, ent


def oracle_lists(o, prompts, offsets, h0):
    """ExtOracle o's lists: (list_offsets, entries, nblocks)"""
    counts, nb = o.match_counts(prompts, offsets, h0)
    off, ent = sparsify(counts, 0 if o.shard is None else o.shard[0])
    return off, ent, nb


def densify(off: np.ndarray, ent: np.ndarray, begin: int, cols: int) -> np.ndarray:
    """the inverse of sparsify"""
    out = np.zeros((len(off) - 1, cols), dtype=np.uint16)
    for r in range(len(off) - 1):
        e = ent[int(off[r]):int(off[r + 1])]
        out[r, e["endpoint"].astype(np.int64) - begin] = e["match_blocks"]
    return out
