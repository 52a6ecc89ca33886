"""CPU: the constructions of tests/craft.py, checked against the C++ oracle's hashing and against the python
restatement (tests/restate.py, the `xxhash` wheel), and the picks of the two references on crafted chains.

Both references treat the hashes 0 and ~0 as ordinary keys (docs/SPEC.md S.1, S.2a): a chain block that hashes to a
marker is held, counted and removed like any other.  The GPU tests of tests/test_gpu_craft.py compare the kernels with
these references on the same constructions.
"""
import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import make_config
from oracle import epp_oracle as eo
from tests import craft as K
from tests import helpers as H
from tests import restate as RS

BLOCK_BYTES = [8, 16, 32, 40, 48, 64, 96, 128, 1024]


def _oracle(B, M, E=8, mode=abi.FI_MATCH_UPSTREAM, profiles=None):
    cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=0, max_batch=256, match_mode=mode,
                      profiles=profiles or [{"name": "default", "scorers": [(H.P, 100), (H.K, 13), (H.Q, 7)]}])
    return cfg, eo.Oracle(cfg)


@pytest.mark.parametrize("B", BLOCK_BYTES)
def test_crafted_value_lands_at_its_block(B):
    M = 72
    cfg, ref = _oracle(B, M)
    rng = np.random.default_rng(B)
    targets = [0, K.MASK64, int(rng.integers(1, 1 << 63))]
    specs = [(M, p, t) for p in (0, 1, 7, 8, 63, 64, M - 1) for t in targets]
    s = K.scene(specs, B, rng, tail=5)
    chains, nb = ref.hash_batch(s.tok, s.offs, s.h0)
    assert (nb == M).all()
    for r, (n, p, t) in enumerate(specs):
        assert int(chains[r, p]) == t, (B, p, t)
        assert s.chain(r, p) == t
        if r % 3 == 0:  # the python restatement (xxhash wheel), on fewer rows: it is slow
            assert RS.chain(s.blobs[r], B, M, int(s.h0[r]))[p] == t
        # the other blocks are ordinary: no accidental marker
        others = np.delete(chains[r, :n], p)
        assert not np.isin(others, np.array(K.MARKERS, dtype=np.uint64)).any()
    ref.close()


@pytest.mark.parametrize("B", [4, 12, 20, 24, 56, 88, 100])
def test_block_sizes_that_cannot_be_crafted_are_refused(B):
    with pytest.raises(ValueError):
        K.check_block_bytes(B)
    with pytest.raises(ValueError):
        K.scene([(3, 1, 0)], B, np.random.default_rng(0))


def test_the_rejected_stripe_case_really_breaks_the_inversion():
    """At 24-byte blocks h_prev sits in the message's only stripe: the one-step inverse misses its target"""
    rng = np.random.default_rng(24)
    block = rng.integers(0, 256, 24, dtype=np.uint8).tobytes()
    h = eo.xxh64(block + b"\0" * 8)
    pre = K._rotr((K.avalanche_inv(h) - K.P4) * K.P1_INV & K.MASK64, 27)
    prev = K.unlink(pre, 0)
    assert eo.xxh64(block + prev.to_bytes(8, "little")) != 0


def test_inverses_are_inverses():
    rng = np.random.default_rng(5)
    for x in [0, 1, K.MASK64, 1 << 63] + [int(v) for v in rng.integers(0, 1 << 63, 200)]:
        assert K.round0_inv(K.round0(x)) == x
        assert K.avalanche_inv(K.avalanche(x)) == x
        assert K.tie_mix_inv(K.tie_mix(x)) == x
        p = int(rng.integers(0, 1 << 63))
        assert K.unlink(p, K.link(p, x)) == x


@pytest.mark.parametrize("E", [1, 2, 3, 31, 32, 33, 40, 64, 100, 1024, 2048, 4096])
def test_every_start_is_reached(E):
    starts = range(E) if E <= 1024 else sorted({0, 1, E - 2, E - 1} | {32 * k + d for k in range(1, E // 32)
                                                                      for d in (-1, 0, 1)})
    for s in starts:
        h1 = K.h1_for_start(s, E)
        assert RS.tie_start(1, h1, 0, 0, E) == s == K.tie_start(h1, E)
        low = (s * 0x9E3779B1 + 12345) & 0xFFFFFFFF
        assert RS.tie_start(1, K.h1_for_start(s, E, low), 0, 0, E) == s
        assert RS.tie_start(1, K.h1_for_start(s, E, 0xFFFFFFFF), 0, 0, E) == s
        for r in (0, 7):
            h0 = K.h0_for_start(s, E, r)
            assert RS.tie_start(0, 0, h0, r, E) == s


@pytest.mark.parametrize("E", [1, 3, 40, 100])
def test_oracle_picks_follow_the_crafted_starts(E):
    """Cold requests (an empty index, equal endpoint states): every endpoint ties and the oracle's pick is the start
    itself, for requests with blocks (seed h_1) and without (seed h0 ^ (r + 1)·GOLDEN)"""
    B = 64
    cfg, ref = _oracle(B, 8, E=E, profiles=[{"name": "p", "scorers": [(H.P, 100)]}])
    ref.update_endpoints(H.states_array(E))
    rng = np.random.default_rng(E)
    blobs, h0, want = [], [], []
    for r in range(2 * E):
        s = r % E
        if r < E:
            raw = rng.integers(0, 256, 3 * B, dtype=np.uint8).tobytes()
            blocks = [raw[j * B:(j + 1) * B] for j in range(3)]
        else:
            raw, blocks = b"\x01" * (r % B), []
        blobs.append(raw)
        h0.append(K.h0_for_start(s, E, r, blocks))
        want.append(s)
    tok, offs = H.pack_prompts(blobs)
    picks = ref.pick_batch(tok, offs, np.array(h0, dtype=np.uint64))
    assert picks[:, 0]["endpoint"].tolist() == want
    ref.close()


def _both(cfg, ops):
    ref = eo.Oracle(cfg)
    rs = RS.from_config(cfg)
    st = H.states_array(cfg.num_endpoints, kv=np.linspace(0, 0.5, cfg.num_endpoints),
                        queue=np.arange(cfg.num_endpoints) % 5)
    ref.update_endpoints(st)
    rs.update_endpoints(st)
    ref.index_apply(ops)
    rs.apply(ops)
    return ref, rs


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM], ids=["upstream", "lpm"])
@pytest.mark.parametrize("B", [64, 40])
def test_oracle_and_restatement_agree_on_marker_chains(B, mode):
    """Small scenes with the marker at the first, an interior and the last block, held by one endpoint, several or
    none, and the blocks around it held: a marker is an ordinary key to both references"""
    E, M = 6, 24
    cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=M, lru_capacity=0, max_batch=64, match_mode=mode,
                      profiles=[{"name": "default", "scorers": [(H.P, 100), (H.K, 13), (H.Q, 7)]}])
    rng = np.random.default_rng(B + mode)
    specs = [(n, p, t) for t in K.MARKERS for n, p in ((12, 0), (12, 5), (12, 11), (20, 8), (3, 2))]
    s = K.scene(specs, B, rng)
    probe = eo.Oracle(cfg)
    chains, nb = probe.hash_batch(s.tok, s.offs, s.h0)
    probe.close()
    for held in ("one", "many", "none"):
        triples = []
        for r, (n, p, t) in enumerate(specs):
            assert int(chains[r, p]) == t
            holders = {"one": [r % E], "many": [r % E, (r + 2) % E, (r + 3) % E], "none": []}[held]
            for e in range(E):  # everyone holds the first half; the holders hold everything but the marker too
                upto = n if e in holders else n // 2
                triples += [(int(chains[r, j]), e, abi.FI_OP_SET) for j in range(upto) if j != p]
            triples += [(t, e, abi.FI_OP_SET) for e in holders]
        # the markers are shared keys: a scene holds 0 and ~0 at once, for every request that crafted them
        ref, rs = _both(cfg, H.ops_array(triples))
        want = ref.pick_batch(s.tok, s.offs, s.h0)
        got = rs.pick(s.tok, s.offs, s.h0)
        for f in ("endpoint", "match_blocks", "n_blocks"):
            assert np.array_equal(want[f], got[f]), (held, f, want[f].ravel(), got[f].ravel())
        assert np.array_equal(want["score"].view(np.uint64), got["score"].view(np.uint64)), held
        if held != "none" and mode == abi.FI_MATCH_UPSTREAM:
            # the holders' count includes the marker: the full chain
            assert any(int(want[r, 0]["match_blocks"]) == n for r, (n, _, _) in enumerate(specs))
        ref.close()
