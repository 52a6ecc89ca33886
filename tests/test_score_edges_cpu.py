"""CPU: the scoring edge cases of tests/score_edges.py through the three CPU restatements of docs/SPEC.md — the
oracle, tests/restate.py and the exact Fraction reference spec_total — which must agree bit for bit; the ranked and
subset oracles against the single pick and the subset-aware reference; and proof that every modelled kernel mistake
changes an expected output of the cases, so the bit-exact GPU comparisons of test_gpu_score_edges.py can see it."""
import functools

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import restate
from tests import score_edges as S
from tests.helpers import describe_diff
from tests.ranked_oracle import RankedOracle
from tests.subset_oracle import SubsetOracle

MODES = [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM]
POOLS = [3, 40, 100]


@functools.lru_cache(maxsize=None)
def _case(kind, E, mode, R=96):
    return S.make_case(kind, E, mode, seed=1000 * E + 10 * mode + S.ALL_KINDS.index(kind), R=R)


def _eq(got, want, what):
    assert got.tobytes() == want.tobytes(), what + "\n" + describe_diff(got, want)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("E", POOLS)
@pytest.mark.parametrize("kind", S.ALL_KINDS)
def test_oracle_restatement_and_exact_reference_agree(kind, E, mode):
    c = _case(kind, E, mode)
    cfg = c.config()
    o = eo.Oracle(cfg)
    c.load(o)
    want = S.spec_picks(c)
    _eq(o.pick_batch(c.tok, c.offs, c.h0, adapters=c.adapters), want, "oracle vs spec_total")
    rs = restate.from_config(cfg)
    rs.update_endpoints(c.states)
    if c.lora is not None:
        rs.update_lora(c.lora)
    rs.apply(c.ops)
    _eq(rs.pick(c.tok, c.offs, c.h0, adapters=c.adapters), want, "tests/restate.py vs spec_total")
    o.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("E", POOLS)
@pytest.mark.parametrize("kind", S.ALL_KINDS)
def test_ranked_and_subset_oracles_on_the_edges(kind, E, mode):
    c = _case(kind, E, mode)
    cfg = c.config()
    ro, so = RankedOracle(cfg), SubsetOracle(cfg)
    c.load(ro)
    c.load(so)
    spec = S.Spec(c)
    single = spec.picks()
    for k in (1, 5, 16):
        ranked = ro.pick_batch_ranked(c.tok, c.offs, c.h0, k, adapters=c.adapters)
        _eq(np.ascontiguousarray(ranked[:, :, 0]), single, f"ranked k={k} entry 0 vs the single pick")
        _eq(ranked, spec.ranked(k), f"ranked k={k} vs spec")
        full = np.full((c.R, (E + 31) // 32), 0xFFFFFFFF, dtype=np.uint32)
        _eq(so.pick_batch_subset(c.tok, c.offs, c.h0, full, k, adapters=c.adapters), ranked, f"full subset k={k} vs ranked")
    sub = S.subset_rows(c, seed=E + mode)
    for k in (1, 5):
        _eq(so.pick_batch_subset(c.tok, c.offs, c.h0, sub, k, adapters=c.adapters), spec.ranked(k, sub),
            f"proper subsets k={k} vs the subset-aware spec")
    ro.close()
    so.close()


def test_queue_extremes_inside_and_outside_the_subsets():
    """the edge cases put INT32_MIN and INT32_MAX on endpoints 0 and E - 1; the subset rows hold both, and neither"""
    c = _case("edges", 40, abi.FI_MATCH_UPSTREAM)
    assert c.states["queue_depth"][0] == S.I32_MIN and c.states["queue_depth"][-1] == S.I32_MAX
    sub = S.subset_rows(c, seed=1)
    bits = np.unpackbits(sub.view(np.uint8), axis=1, bitorder="little")[:, : c.E].astype(bool)
    both = bits[:, 0] & bits[:, -1]
    neither = ~bits[:, 0] & ~bits[:, -1] & bits.any(axis=1)
    assert both.any() and neither.any()


GPU_CPU_CASES = [(kind, E) for kind, E in S.GPU_CASES if E <= 1024]  # the GPU suite's cases, E > 1024 too slow here


def test_every_variant_changes_an_expected_output_of_the_gpu_cases():
    """each modelled kernel mistake moves at least one single pick of the GPU suite's cases to another endpoint, and
    every one of those cases is kept by the seeded search (some variant changes it), so a kernel making one of these
    mistakes cannot pass the bit-exact GPU comparisons"""
    cands = [S.gpu_case(kind, E) for kind, E in GPU_CPU_CASES]
    kept = S.discriminating(cands)
    assert sorted(c.name + str(c.E) for c, _ in kept) == sorted(c.name + str(c.E) for c in cands), "cases without power"
    total = {v: [0, 0] for v in S.VARIANTS}
    for _, d in kept:
        for v, (ep, anyd) in d.items():
            total[v][0] += ep
            total[v][1] += anyd
    missing = [v for v, (ep, _) in total.items() if ep == 0]
    assert not missing, f"variants the cases cannot tell from the spec by endpoint: {missing} ({total})"


def test_every_variant_changes_a_ranked_or_subset_output_of_the_gpu_cases():
    """the same for the ranked lists (k = 5) and for the subset picks with the GPU suite's subset rows, whose queue
    range is normalised per request (INT32_MIN / INT32_MAX inside and outside the subset)"""
    ranked = {v: 0 for v in S.VARIANTS if v != "zero_tie"}  # zero_tie models the single pick's shortcut only
    subset = {v: 0 for v in ranked}
    for kind, E in GPU_CPU_CASES:
        if E > 100:
            continue
        c = S.gpu_case(kind, E)
        sub = S.subset_rows(c, seed=E)  # the rows test_gpu_score_edges.py uses
        want, want_sub = S.Spec(c).ranked(5), S.Spec(c).ranked(5, sub)
        for v in ranked:
            sp = S.Spec(c, v)
            ranked[v] += S.differs(sp.ranked(5), want)[0]
            subset[v] += S.differs(sp.ranked(5, sub), want_sub)[0]
    assert all(ranked.values()), ranked
    assert all(subset.values()), subset


def test_rounding_order_alone_decides_some_picks():
    """the order cases hold pairs of endpoints whose exact rational totals tie and whose fp64 totals differ; the pick
    of such a request goes to one of the pair, and which one flips with the accumulation order"""
    c = _case("order", 40, abi.FI_MATCH_UPSTREAM)
    spec = S.spec_picks(c)
    rev = S.spec_picks(c, "reverse")
    flipped = 0
    for r in range(c.R):
        for pi in range(len(c.profiles)):
            a, b = int(spec[r, pi]["endpoint"]), int(rev[r, pi]["endpoint"])
            if a != b and a // 2 == b // 2 and a < 32:  # the two endpoints of one pair
                flipped += 1
    assert flipped > 0
    assert S._order_pairs(S.MAX_BLOCKS)


def test_spec_total_rounds_every_operation():
    """spec_total is the rounded sequence of S.4: it equals IEEE double arithmetic in profile order, the clamp maps
    every out-of-range kv to a score of 0 or 1, and a queue range of INT32_MIN .. INT32_MAX needs 64-bit differences"""
    sc = ((S.K, 1), (S.K, 1))
    assert S.spec_total(sc, 0, 0, 0.9, 0, 0, 0) == (1.0 - 0.9) * 2
    assert S.spec_total(((S.K, 1), (S.Q, 1)), 0, 0, 0.9, 0, 0, 0) == (1.0 - 0.9) + 1.0
    for kv, want in ((-1e308, 1.0), (1e308, 0.0), (-0.0, 1.0), (5e-324, 1.0), (1.5, 0.0), (-0.5, 1.0)):
        assert S.spec_total(((S.K, S.W_MAX),), 0, 0, kv, 0, 0, 0) == want * S.W_MAX
    # INT32 extremes: (max - q) / (max - min) in 64-bit integers, 2^32 - 1 in the denominator
    assert S.spec_total(((S.Q, 1),), 0, 0, 0.0, 0, S.I32_MIN, S.I32_MAX) == S.I32_MAX / (2**32 - 1)
    assert S.spec_total(((S.Q, 1),), 0, 0, 0.0, 0, S.I32_MIN, S.I32_MAX, variant="q_int32") == 0.0
