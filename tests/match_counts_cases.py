"""Index states and prompts for the match-count tests (docs/SPEC.md S.3a), shared by tests/test_match_counts_cpu.py
and tests/test_gpu_match_counts.py (test helper, not collected).

A case is a pool of E endpoints and R prompts drawn from a few prefix families, so that many prompts share cached
prefixes of different lengths, some prompts are shorter than one block and some run to max_blocks.  Its index is
built from the families' chains in any of three ways, each applied to every handle and oracle the same way:
  * direct SET / CLEAR ops with holes: endpoint e holds blocks [0, k) of a family chain minus a few, then some of its
    pairs are cleared again;
  * Adds through an LRU whose capacity is below what the Adds touch, so that chain fronts are evicted;
  * removals of a few endpoints after either."""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi
from tests import helpers as H


def prompts(R: int, B: int, M: int, rng, families: int = 6):
    """-> (prompt bytes, offsets [R + 1]) of R prompts: a family prefix of 0 .. M blocks, then request-own bytes; the
    first requests are shorter than one block"""
    base = rng.integers(0, 256, size=(families, (M + 2) * B), dtype=np.uint8)
    blobs = []
    for r in range(R):
        if r < 3:
            blobs.append(bytes(rng.integers(0, 256, size=int(rng.integers(0, B)), dtype=np.uint8)))
            continue
        f = int(rng.integers(0, families))
        shared = int(rng.integers(0, M + 1)) * B + int(rng.integers(0, B))
        total = shared + int(rng.integers(0, 3 * B))
        if r % 7 == 0:
            total = (M + 1) * B + 3  # longer than max_blocks blocks
        own = rng.integers(0, 256, size=max(total - shared, 0), dtype=np.uint8)
        blobs.append(bytes(base[f, :min(shared, total)]) + bytes(own))
    return H.pack_prompts(blobs)


def family_ops(chains, nb, E: int, rng, holes: float = 0.1, per_endpoint: int = 3):
    """SET ops: every endpoint holds a random leading part of a few requests' chains, with holes, then a few CLEARs;
    -> a list of OP_DTYPE arrays to apply in order"""
    sets, clears = [], []
    rows = [r for r in range(len(nb)) if nb[r] > 0]
    for e in range(E):
        for r in rng.choice(rows, size=min(per_endpoint, len(rows)), replace=False):
            k = int(rng.integers(1, int(nb[r]) + 1))
            for i in range(k):
                if rng.random() >= holes:
                    sets.append((int(chains[r, i]), e, abi.FI_OP_SET))
            if rng.random() < 0.3:
                i = int(rng.integers(0, k))
                clears.append((int(chains[r, i]), e, abi.FI_OP_CLEAR))
    return [H.ops_array(sets), H.ops_array(clears)]


def add_batches(chains, nb, E: int, rng, batches: int = 3):
    """[(endpoints [R], chains, nblocks)] of Adds aimed across the pool, some FI_NO_ENDPOINT"""
    out = []
    for _ in range(batches):
        dest = rng.integers(0, E, len(nb)).astype(np.uint32)
        dest[rng.random(len(nb)) < 0.1] = abi.FI_NO_ENDPOINT
        out.append((dest, chains, nb))
    return out


def unique_counts(counts: np.ndarray) -> int:
    """how many distinct non-zero counts a matrix holds (a case should exercise many)"""
    return len(np.unique(counts[counts > 0]))
