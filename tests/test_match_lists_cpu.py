"""CPU: the reference of fi_epp_match_lists (docs/SPEC.md S.3b), the yardstick of tests/test_gpu_match_lists.py.

  * fi_match_entry is 8 bytes: endpoint at 0, match_blocks at 4, reserved at 6, and match_entry_dtype agrees.
  * The sparsified ExtOracle.match_counts (tests/match_lists_ref.py) equals lists built from the independent
    restatement's match (tests/restate.py) in both match modes, on the whole pool and on shard views.
  * In LPM mode, the per-request lists of a partition's shard views, concatenated in shard order, are the pool's lists.
"""
import ctypes as C

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from tests import helpers as H
from tests import match_counts_cases as MC
from tests import match_lists_ref as ML
from tests import restate
from tests import shard_view as SV
from tests.ext_oracle import ExtOracle

MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]


def _cfg(E, B, M, R, mode, lru=0):
    return H.make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=lru, max_batch=R, index_slots=1 << 14,
                         match_mode=mode, profiles=[{"name": "d", "scorers": [(H.P, 100)]}])


def test_entry_layout():
    assert C.sizeof(abi.fi_match_entry) == 8
    assert abi.fi_match_entry.endpoint.offset == 0
    assert abi.fi_match_entry.match_blocks.offset == 4 and abi.fi_match_entry.reserved.offset == 6
    dt = abi.match_entry_dtype()
    assert dt.itemsize == 8 and dt.fields["endpoint"][1] == 0 and dt.fields["match_blocks"][1] == 4
    assert dt.fields["reserved"][1] == 6 and dt["match_blocks"] == np.dtype("<u2")


def test_sparsify_round_trip_and_order():
    counts = np.array([[0, 3, 0, 1], [0, 0, 0, 0], [7, 0, 0, 2]], dtype=np.uint16)
    off, ent = ML.sparsify(counts, begin=10)
    assert off.tolist() == [0, 2, 2, 4]
    assert ent["endpoint"].tolist() == [11, 13, 10, 13] and ent["match_blocks"].tolist() == [3, 1, 7, 2]
    assert (ent["reserved"] == 0).all()
    assert np.array_equal(ML.densify(off, ent, 10, 4), counts)
    off0, ent0 = ML.sparsify(np.zeros((0, 4), np.uint16))
    assert off0.tolist() == [0] and len(ent0) == 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B", [5, 64])
@pytest.mark.parametrize("shard", [None, (3, 33)])
def test_lists_equal_restatement(mode, B, shard):
    E, R, M = 37, 96, 24
    rng = np.random.default_rng(11 + B)
    tok, offs = MC.prompts(R, B, M, rng)
    cfg = _cfg(E, B, M, R, mode)
    o = ExtOracle(cfg, shard=shard)
    py = restate.from_config(cfg, shard=shard)
    chains, nb = o.hash_batch(tok, offs, 0x77)
    for ops in MC.family_ops(chains, nb, E, rng):
        o.index_apply(ops)
        py.apply(ops)
    off, ent, n = ML.oracle_lists(o, tok, offs, 0x77)
    assert (n == nb).all()
    want_off, want = [0], []
    for r in range(R):
        m = py.match([int(h) for h in chains[r, : nb[r]]])
        row = sorted((e, c) for e, c in m.items() if c > 0 and e in py.own)
        want += row
        want_off.append(want_off[-1] + len(row))
    assert off.tolist() == want_off
    assert list(zip(ent["endpoint"].tolist(), ent["match_blocks"].tolist())) == want
    assert len(want) > R // 4 and (np.diff(off) == 0).any()
    o.close()


def test_shard_lists_concatenate_into_the_pool():
    """LPM, holes included: request r's lists of a partition's views, concatenated in shard order, are its pool list"""
    E, R, M, B = 70, 64, 24, 64
    rng = np.random.default_rng(23)
    tok, offs = MC.prompts(R, B, M, rng)
    cfg = _cfg(E, B, M, R, abi.FI_MATCH_LPM)
    full = ExtOracle(cfg)
    chains, nb = full.hash_batch(tok, offs, 5)
    ops = MC.family_ops(chains, nb, E, rng, holes=0.1)
    for a in ops:
        full.index_apply(a)
    woff, went, _ = ML.oracle_lists(full, tok, offs, 5)
    for parts in SV.splits(E):
        lists = []
        for bc in parts:
            v = ExtOracle(cfg, shard=bc)
            for a in ops:
                v.index_apply(a)
            lists.append(ML.oracle_lists(v, tok, offs, 5)[:2])
            v.close()
        for r in range(R):
            got = np.concatenate([e[int(o[r]):int(o[r + 1])] for o, e in lists])
            assert got.tobytes() == went[int(woff[r]):int(woff[r + 1])].tobytes(), (parts, r)
    full.close()
