"""CPU: the subset pick of the oracle extension (tests/ext_oracle.cpp) on hand-worked cases (docs/SPEC.md S.5a), its
bitset helper and its C binding.

Each case is small enough to work out by hand: four endpoints, one four-block prompt, and the index rows set
explicitly from the prompt's own chain.
"""
import os
import re

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import make_config, subset_bitsets, synth
from tests import helpers as H
from tests.ext_oracle import ExtOracle

P, K, Q = H.P, H.K, H.Q
NO = abi.FI_NO_ENDPOINT
B = 64  # block bytes
H0 = 0x1234


def _oracle(profiles, E=4, pd=None, mode=abi.FI_MATCH_UPSTREAM, queue=None, roles=None, alive=None):
    cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=8, max_batch=16, match_mode=mode, profiles=profiles,
                      pd=pd)
    o = ExtOracle(cfg)
    o.update_endpoints(H.states_array(E, queue=queue, roles=roles, alive=alive))
    return o


def _prompt(nblocks=4, seed=1):
    blob = np.random.default_rng(seed).integers(0, 256, nblocks * B, dtype=np.uint8).tobytes()
    return H.pack_prompts([blob])


def _hold(o, tok, offs, holders):
    """holders: {endpoint: [block indices]} -> SET ops of those blocks of the prompt's chain"""
    chain = o.hash_batch(tok, offs, H0)[0][0]
    o.index_apply(H.ops_array([(int(chain[i]), e, abi.FI_OP_SET) for e, bl in holders.items() for i in bl]))


def _row(o, *endpoints):
    return subset_bitsets([list(endpoints)], o.E)


def _entries(picks, r=0, p=0):
    return [(int(x["endpoint"]), int(x["match_blocks"]), float(x["score"])) for x in picks[r, p]]


def test_queue_scores_are_normalised_over_the_subset():
    """queues [0, 10, 5, 20], subset {1, 3}: endpoint 1 scores (20-10)/(20-10) = 1.0, not the pool's 0.5"""
    o = _oracle([{"name": "default", "scorers": [(Q, 1)]}], queue=np.array([0, 10, 5, 20]))
    tok, offs = _prompt()
    got = o.pick_batch_subset(tok, offs, H0, _row(o, 1, 3), k=2)
    assert _entries(got) == [(1, 0, 1.0), (3, 0, 0.0)]
    whole = o.pick_batch_subset(tok, offs, H0, None, k=4)
    assert _entries(whole) == [(0, 0, 1.0), (2, 0, 0.75), (1, 0, 0.5), (3, 0, 0.0)]
    o.close()


def test_a_subset_without_the_best_matching_pod():
    o = _oracle([{"name": "default", "scorers": [(P, 100)]}])
    tok, offs = _prompt()
    _hold(o, tok, offs, {2: [0, 1, 2, 3], 0: [0, 1]})
    assert _entries(o.pick_batch_subset(tok, offs, H0, None)) == [(2, 4, 100.0)]
    assert _entries(o.pick_batch_subset(tok, offs, H0, _row(o, 0, 1))) == [(0, 2, 50.0)]
    o.close()


def test_an_empty_subset_gives_no_endpoint():
    o = _oracle([{"name": "default", "scorers": [(P, 100), (K, 1)]}])
    tok, offs = _prompt()
    _hold(o, tok, offs, {1: [0, 1]})
    got = o.pick_batch_subset(tok, offs, H0, _row(o), k=3)
    assert _entries(got) == [(NO, 0, 0.0)] * 3
    assert (got["n_blocks"] == 4).all()
    o.close()


def test_a_subset_of_dead_or_filtered_pods_gives_no_endpoint():
    """endpoint 0 is dead, endpoint 1 lacks the profile's label: a subset of the two has no eligible pod"""
    o = _oracle([{"name": "a", "role_mask": 2, "scorers": [(P, 100)]}], roles=np.array([2, 1, 2, 2], dtype=np.uint32),
                alive=np.array([0, 1, 1, 1]))
    tok, offs = _prompt()
    _hold(o, tok, offs, {0: [0, 1, 2, 3], 1: [0, 1, 2, 3]})
    assert _entries(o.pick_batch_subset(tok, offs, H0, _row(o, 0, 1))) == [(NO, 0, 0.0)]
    assert _entries(o.pick_batch_subset(tok, offs, H0, _row(o, 0, 1, 3))) == [(3, 0, 0.0)]
    o.close()


def test_the_walk_stays_pool_wide():
    """upstream mode: block 1 is held only by endpoint 3, outside the subset {0}; the walk still passes it, so
    endpoint 0's block 2 counts (match 2 of 4)"""
    o = _oracle([{"name": "default", "scorers": [(P, 100)]}])
    tok, offs = _prompt()
    _hold(o, tok, offs, {0: [0, 2], 3: [1]})
    assert _entries(o.pick_batch_subset(tok, offs, H0, _row(o, 0))) == [(0, 2, 50.0)]
    o.close()


PD = [{"name": "prefill", "role_mask": 1, "scorers": [(P, 50), (K, 5)]},
      {"name": "decode", "role_mask": 2, "scorers": [(P, 50), (Q, 5)]}]


def test_pd_with_a_subset_that_holds_no_decode_pod():
    """decode pod 2 holds the whole prompt, so the whole pool skips prefill (0 miss bytes < 100); a subset of the
    prefill pods has no decode pick, every byte misses and prefill runs"""
    o = _oracle(PD, pd={"prefill": 0, "decode": 1, "threshold": 100.0}, roles=np.array([1, 1, 2, 2], dtype=np.uint32))
    tok, offs = _prompt()
    _hold(o, tok, offs, {2: [0, 1, 2, 3], 1: [0]})
    whole = o.pick_batch_subset(tok, offs, H0, None)
    assert _entries(whole, p=1) == [(2, 4, 55.0)] and _entries(whole, p=0) == [(NO, 0, 0.0)]
    got = o.pick_batch_subset(tok, offs, H0, _row(o, 0, 1), k=2)
    assert _entries(got, p=1) == [(NO, 0, 0.0)] * 2
    assert _entries(got, p=0) == [(1, 1, 17.5), (0, 0, 5.0)]
    o.close()


def test_k_beyond_the_subset_is_padded():
    o = _oracle([{"name": "default", "scorers": [(P, 100)]}])
    tok, offs = _prompt()
    _hold(o, tok, offs, {2: [0, 1], 1: [0]})
    assert _entries(o.pick_batch_subset(tok, offs, H0, _row(o, 1, 2), k=4)) == \
        [(2, 2, 50.0), (1, 1, 25.0), (NO, 0, 0.0), (NO, 0, 0.0)]
    o.close()


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_no_subset_and_all_ones_equal_the_ranked_oracle(mode):
    """No subset is the ranked pick itself (one function, which test_ranked_cpu.py's
    test_ranked_oracle_matches_numpy_ranking checks against tests/restate.py).  All-ones rows must equal it: the queue
    range over a full row is the pool's.  Entry 0 of both is the oracle's single pick (epo_pick_batch, code the ranked
    pick does not share).  A subset never adds an endpoint."""
    rng = np.random.default_rng(9 + mode)
    E = 40
    wl = synth.Workload(R=24, E=E, T=160, seed=synth.SEEDS[1], max_blocks=8, lru_capacity=64, holes=True)
    profiles = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]},
                {"name": "a", "role_mask": 3, "scorers": [(P, 10), (Q, 3)]}]
    cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=wl.R,
                      match_mode=mode, profiles=profiles)
    o = ExtOracle(cfg)
    o.update_endpoints(H.states_array(E, kv=rng.integers(0, 8, E) / 8.0, queue=rng.integers(0, 6, E),
                                      roles=rng.integers(1, 8, E).astype(np.uint32),
                                      alive=np.where(rng.random(E) < 0.2, 0, 1)))
    for ops in wl.index_ops():
        o.index_apply(ops)
    tok, offs = wl.prompts()
    single = o.pick_batch(tok, offs, wl.h0)
    for k in (1, 5):
        want = o.pick_batch_ranked(tok, offs, wl.h0, k)
        assert H.picks_equal(np.ascontiguousarray(want[:, :, 0]), single)
        assert H.picks_equal(o.pick_batch_subset(tok, offs, wl.h0, subset_bitsets([None] * wl.R, E), k), want)
    # a subset never adds an endpoint: every listed pick is a candidate of its request
    lists = [sorted(rng.choice(E, 6, replace=False).tolist()) for _ in range(wl.R)]
    got = o.pick_batch_subset(tok, offs, wl.h0, subset_bitsets(lists, E), 3)
    for r in range(wl.R):
        real = got["endpoint"][r][got["endpoint"][r] != NO]
        assert set(real.tolist()) <= set(lists[r])
    o.close()


def test_subset_bitsets():
    rows = subset_bitsets([None, [], [0, 31, 32, 69], [5, 5, 70, -1, 1000]], 70)
    assert rows.shape == (4, 3) and rows.dtype == np.uint32
    assert (rows[0] == 0xFFFFFFFF).all()
    assert (rows[1] == 0).all()
    assert rows[2].tolist() == [(1 << 0) | (1 << 31), 1, 1 << 5]
    assert rows[3].tolist() == [1 << 5, 0, 0]  # duplicates once, addresses outside the pool dropped


def test_header_declares_the_subset_calls_as_bound():
    src = open(os.path.join(os.path.dirname(os.path.dirname(abi.__file__)), "include", "fi_epp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    bound = {name: args for name, _, args in abi.SYMBOLS}
    for name in ("fi_epp_pick_batch_subset", "fi_epp_pick_batch_device_subset"):
        decl = re.search(name + r"\s*\(([^)]*)\)", src)
        assert decl, name
        assert len(decl.group(1).split(",")) == len(bound[name]), name
    lib = abi.load()
    assert hasattr(lib, "fi_epp_pick_batch_subset") and hasattr(lib, "fi_epp_pick_batch_device_subset")
