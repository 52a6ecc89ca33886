"""CPU: chains of up to FI_EPP_MAX_BLOCKS = 4095 blocks.

- the EndpointPickerConfig loader takes maxPrefixBlocksToMatch up to 4095 and refuses 4096;
- the 12-plane bit counters of the windowed match kernel (bitslice.cuh BitCounter<12>, through libfi_hostcheck.so)
  count, merge and unpack up to 4095 like numpy;
- the oracle agrees with the independent restatement (tests/restate.py) on prompts of 1024, 2500 and 4095 blocks in
  both match modes, on indexes whose cached prefixes have holes past block 1023.
"""
import ctypes as C
import os

import numpy as np
import pytest

from fusioninfer_b200 import FiEppError, config_from_yaml, make_config
from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import helpers as H
from tests import restate

P, K, Q = H.P, H.K, H.Q

YAML = """apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
- type: prefix-cache-scorer
  parameters:
    blockSize: 64
    maxPrefixBlocksToMatch: {m}
    lruCapacityPerServer: 31250
- type: max-score-picker
schedulingProfiles:
- name: default
  plugins:
  - pluginRef: max-score-picker
  - pluginRef: prefix-cache-scorer
    weight: 100
"""


# ---- the loader -------------------------------------------------------------------------------------------------
def test_max_blocks_bound():
    assert abi.FI_EPP_MAX_BLOCKS == 4095


@pytest.mark.parametrize("m", [1024, 2047, 4095])
def test_loader_accepts_long_prefixes(m):
    assert config_from_yaml(YAML.format(m=m)).max_blocks == m


@pytest.mark.parametrize("m", [4096, 65535])
def test_loader_refuses_past_4095(m):
    with pytest.raises(FiEppError) as ei:
        config_from_yaml(YAML.format(m=m))
    assert ei.value.status == abi.FI_ERR_CONFIG and "maxPrefixBlocksToMatch" in str(ei.value)


# ---- 12 bit-planes ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    lib.fihc_bitcount12.restype = None
    lib.fihc_bitcount12.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.fihc_bitcount_merge12.restype = None
    lib.fihc_bitcount_merge12.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.fihc_bc_unpack12.restype = C.c_int
    lib.fihc_bc_unpack12.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    return lib


def _bits(words):
    """numpy count of each of the 32 bits over the words"""
    return ((words[:, None] >> np.arange(32, dtype=np.uint32)) & 1).sum(axis=0)


def _words(rng, n, density):
    w = np.zeros(n, dtype=np.uint32)
    for b in range(32):
        w |= (rng.random(n) < density[b]).astype(np.uint32) << np.uint32(b)
    return w


@pytest.mark.parametrize("K", [1, 2, 4, 8, 16])
def test_bitcount12_counts_to_4095(hc, K):
    """Every bit set in all 4095 words (all 12 planes), bits that cross 1023, 1024, 2047 and 2048, random ones."""
    rng = np.random.default_rng(K)
    for n in (1, 1023, 1024, 1025, 2047, 2048, 3000, 4095):
        dens = rng.random(32)
        dens[:4] = [1.0, 0.0, 0.5, 0.999]
        w = np.ascontiguousarray(_words(rng, n, dens))
        got = np.zeros(32, dtype=np.uint32)
        hc.fihc_bitcount12(w.ctypes.data, n, K, got.ctypes.data)
        assert got.tolist() == _bits(w).tolist(), (n, K)
    w = np.full(4095, 0xFFFFFFFF, dtype=np.uint32)
    got = np.zeros(32, dtype=np.uint32)
    hc.fihc_bitcount12(w.ctypes.data, 4095, K, got.ctypes.data)
    assert (got == 4095).all()


def test_bitcount12_merge(hc):
    """Two counters merged as the lane groups of one match window merge theirs: sums up to 4095."""
    rng = np.random.default_rng(7)
    for na, nb in ((2047, 2048), (4095, 0), (1024, 1024), (3000, 1095), (1, 4094)):
        a = np.ascontiguousarray(_words(rng, na, rng.random(32)))
        b = np.ascontiguousarray(_words(rng, nb, rng.random(32)))
        a[: min(na, 16)] = 0xFFFFFFFF
        b[: min(nb, 16)] = 0xFFFFFFFF
        got = np.zeros(32, dtype=np.uint32)
        nz = np.zeros(1, dtype=np.uint32)
        hc.fihc_bitcount_merge12(a.ctypes.data, na, b.ctypes.data, nb, got.ctypes.data, nz.ctypes.data)
        want = _bits(np.concatenate([a, b]))
        assert got.tolist() == want.tolist(), (na, nb)
        assert int(nz[0]) == int(sum(1 << i for i in range(32) if want[i]))


def test_bc_unpack12_equals_bc_get(hc):
    rng = np.random.default_rng(3)
    for trial in range(200):
        planes = rng.integers(0, 2**32, size=12, dtype=np.uint64).astype(np.uint32)
        if trial % 4 == 0:
            planes[rng.random(12) < 0.5] = 0
        if trial % 4 == 1:
            planes[:] = 0xFFFFFFFF  # every count 4095
        planes = np.ascontiguousarray(planes)
        for nbits in (1, 2, 4, 8, 16, 32):
            for bit0 in range(0, 33 - nbits, nbits):
                a = np.zeros(nbits, dtype=np.uint16)
                b = np.zeros(nbits, dtype=np.uint16)
                assert hc.fihc_bc_unpack12(planes.ctypes.data, bit0, nbits, a.ctypes.data, b.ctypes.data) == 0
                assert np.array_equal(a, b), (trial, nbits, bit0)
                want = [sum(((int(planes[pl]) >> (bit0 + j)) & 1) << pl for pl in range(12)) for j in range(nbits)]
                assert a.tolist() == want
    z = np.zeros(12, dtype=np.uint32)
    a = np.zeros(32, dtype=np.uint16)
    assert hc.fihc_bc_unpack12(z.ctypes.data, 16, 32, a.ctypes.data, a.ctypes.data) == -1


# ---- oracle against the restatement ------------------------------------------------------------------------------
def _long_case(M, E=8, R=6, B=16, seed=0):
    """R prompts of M + 1 blocks of B bytes (capped at M), pairs of requests sharing a prefix of about M / 2 blocks.
    Endpoint r % E caches request r's chain up to a cut drawn past block 1023, with a hole (one block left out)
    past block 1023 for every third request; request 0's whole chain is cached by endpoint E - 1."""
    rng = np.random.default_rng(seed)
    T = (M + 1) * B
    tok = rng.integers(0, 256, size=(R, T), dtype=np.uint8)
    for r in range(1, R, 2):
        tok[r, : (M // 2) * B] = tok[r - 1, : (M // 2) * B]
    offs = np.arange(R + 1, dtype=np.uint64) * T
    h0 = rng.integers(0, 2**63, size=R, dtype=np.uint64)
    return tok, offs, h0


def _case_ops(o, tok, offs, h0, E, M):
    chains, nb = o.hash_batch(tok.reshape(-1), offs, h0)
    assert (nb == M).all()
    rng = np.random.default_rng(M)
    trip = []
    for r in range(len(nb)):
        cut = int(rng.integers(min(1024, M - 1), M + 1))
        hole = int(rng.integers(1024, cut)) if r % 3 == 0 and cut > 1024 else -1
        trip += [(int(chains[r, i]), r % E, abi.FI_OP_SET) for i in range(cut) if i != hole]
    trip += [(int(h), E - 1, abi.FI_OP_SET) for h in chains[0, :M]]
    return H.ops_array(trip), chains


@pytest.mark.parametrize("M", [1024, 2500, 4095])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_oracle_equals_restatement_long(M, mode):
    E = 8
    tok, offs, h0 = _long_case(M, E=E)
    cfg = make_config(num_endpoints=E, block_bytes=16, max_blocks=M, max_batch=len(h0), max_prompt_bytes=int(offs[-1]),
                      index_slots=1 << 17, match_mode=mode,
                      profiles=[{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}])
    o = eo.Oracle(cfg)
    r = restate.from_config(cfg)
    st = H.states_array(E, kv=np.linspace(0.8, 0.1, E), queue=np.arange(E)[::-1] % 5)  # endpoint E - 1 least loaded
    o.update_endpoints(st)
    r.update_endpoints(st)
    ops, chains = _case_ops(o, tok, offs, h0, E, M)
    o.index_apply(ops)
    r.apply(ops)
    assert restate.chain(tok[0].tobytes(), 16, M, int(h0[0])) == [int(h) for h in chains[0, :M]]
    want = r.pick(tok.reshape(-1), offs, h0)
    got = o.pick_batch(tok.reshape(-1), offs, h0)
    o.close()
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    mb = want[:, 0]["match_blocks"]
    assert mb[0] == M  # the whole chain: a count past 1023 (4095: 12 planes)
    assert (mb >= 1023).sum() >= 3
