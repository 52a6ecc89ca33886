"""CPU: the index snapshot format (docs/SPEC.md S.2d) and the sufficiency of the state it stores.

fi_epp_snapshot_info needs no device: it is held to blobs written by the independent writer of tests/snapshot_ref.py,
which it must accept and read, and to malformed ones (truncations, flipped bytes, a wrong magic or version, rows and
LRUs that break the structural rules), which it must refuse with FI_ERR_INVALID.  The format's checksum and structural
check (snapshot_format.h) are driven through libfi_hostcheck.so.  Last, S.2d claims that the pair set, the LRU lists and
the capacities are all the state later calls depend on: an oracle aged by a churn history is copied into a fresh one
through those three parts alone, and both stay equal under a further history.
"""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import snapshot_info
from tests import helpers as H
from tests import resize_ref as RR
from tests import snapshot_ref as SR
from tests.ext_oracle import ExtOracle

U64_MAX = 0xFFFFFFFFFFFFFFFF


def _aged(seed, E=40, lru_capacity=48, n=16):
    """an ExtOracle after a churn history: Adds with evictions, direct SETs / CLEARs (markers 0 and ~0 included),
    capacity changes and a removal; -> (oracle, call stream, the state calls fed to it)"""
    cfg = RR.config(E, lru_capacity=lru_capacity)
    cs = RR.CallStream(seed, RR.config(E))
    ora = ExtOracle(cfg, track_removal=True)
    states = []
    for i, entry in enumerate(cs.calls(E, n=n) if lru_capacity else _no_lru_calls(cs, E, n)):
        RR.apply(ora, entry)
        if entry[0] in ("states", "lora"):
            states.append(entry)
        if i == n // 2 and lru_capacity:
            ora.remove_endpoints([int(cs.rng.integers(0, E))])
    ops = H.ops_array([(0, 1, abi.FI_OP_SET), (U64_MAX, 2, abi.FI_OP_SET), (U64_MAX, 3, abi.FI_OP_SET)])
    ora.index_apply(ops)
    return ora, cs, states


def _no_lru_calls(cs, E, n):
    return [c for c in cs.calls(E, n=3 * n) if c[0] in ("states", "lora", "ops")][:n]


def _info(blob):
    out = abi.fi_epp_snapshot_info()
    buf = np.frombuffer(bytes(blob), dtype=np.uint8) if len(blob) else np.zeros(1, np.uint8)
    rc = abi.load().fi_epp_snapshot_info(buf.ctypes.data_as(C.c_void_p), len(blob), C.byref(out))
    return rc, out


@pytest.mark.parametrize("lru_capacity", [48, 0])
@pytest.mark.parametrize("shuffle", [False, True])
def test_info_reads_reference_blobs(lru_capacity, shuffle):
    ora, cs, _ = _aged(3 + lru_capacity, lru_capacity=lru_capacity)
    blob = SR.from_oracle(ora, np.random.default_rng(5) if shuffle else None)
    pairs, lrus, caps = ora.state()
    info = snapshot_info(blob)
    cfg = ora.cfg
    assert (info.block_bytes, info.max_blocks, info.lru_capacity, info.num_endpoints) == \
        (cfg.block_bytes, cfg.max_blocks, lru_capacity, cfg.num_endpoints)
    assert info.n_nodes == len({h for _, h in pairs}) and info.pairs == len(pairs) and info.bytes == len(blob)
    assert info.n_lru == sum(len(x) for x in lrus)
    assert {(1, 0), (2, U64_MAX), (3, U64_MAX)} <= pairs
    back = SR.read(blob)
    assert back.pairs() == pairs and back.caps.tolist() == caps
    assert all(np.array_equal(a, b) for a, b in zip(back.lrus, lrus))
    ora.close()


def test_info_reads_an_empty_blob():
    cfg = RR.config(5)
    ora = ExtOracle(cfg)
    blob = SR.from_oracle(ora)
    info = snapshot_info(blob)
    assert (info.n_nodes, info.n_lru, info.pairs, info.bytes) == (0, 0, 0, 64 + 8 * 5)
    ora.close()


def _blob_and_layout():
    ora, _, _ = _aged(11, E=37)  # 37: the last row word has bits at and above E
    blob = SR.from_oracle(ora)
    s = SR.read(blob)
    lay = SR.layout(s.num_endpoints, len(s.node_keys), sum(len(x) for x in s.lrus))
    ora.close()
    return blob, s, lay


def test_info_refuses_truncations_and_flipped_bytes():
    blob, s, lay = _blob_and_layout()
    assert _info(blob)[0] == abi.FI_OK
    cuts = {0, 8, 63, 64}
    for k in ("lru_len", "lru_keys", "node_keys", "node_rows"):
        cuts |= {lay[k], lay[k] + 4, lay[k] - 4}
    cuts |= {lay["end"] - 1, lay["end"] - 4}
    for cut in sorted(cuts):
        assert _info(blob[:cut])[0] == abi.FI_ERR_INVALID, cut
    assert _info(blob + b"\0\0\0\0")[0] == abi.FI_ERR_INVALID
    at = [0, 9, 13, 17, 21, 25, 29, 33, 41, 49, 57]  # every header field
    at += [lay[k] + 1 for k in ("caps", "lru_len", "lru_keys", "node_keys", "node_rows")] + [lay["end"] - 1]
    for i in at:
        bad = bytearray(blob)
        bad[i] ^= 0x10
        assert _info(bytes(bad))[0] == abi.FI_ERR_INVALID, i


def _patched(blob, off, fmt, value):
    bad = bytearray(blob)
    struct.pack_into(fmt, bad, off, value)
    return SR.resealed(bytes(bad))


def test_info_refuses_what_the_checksum_does_not_catch():
    blob, s, lay = _blob_and_layout()
    E = s.num_endpoints
    assert _info(_patched(blob, 0, "<8s", b"FIEPPSNQ"))[0] == abi.FI_ERR_INVALID
    for v in (0, 2):
        assert _info(_patched(blob, 8, "<I", v))[0] == abi.FI_ERR_INVALID, v
    assert _info(_patched(blob, 12, "<I", 32))[0] == abi.FI_ERR_INVALID
    W = SR.row_words(E)
    # an empty row; a bit at E (the first bit past the pool in the last word)
    assert _info(_row(blob, lay, W, 3, [0] * W))[0] == abi.FI_ERR_INVALID
    row = s.node_rows[5].copy()
    row[W - 1] |= np.uint32(1 << (E % 32))
    assert _info(_row(blob, lay, W, 5, row.tolist()))[0] == abi.FI_ERR_INVALID
    # capacities out of [max_blocks, lru_capacity]; an LRU longer than its capacity
    for cap in (s.max_blocks - 1, s.lru_capacity + 1, 0):
        assert _info(_patched(blob, lay["caps"] + 4 * 2, "<I", cap))[0] == abi.FI_ERR_INVALID, cap
    e = int(np.argmax([len(x) for x in s.lrus]))
    n = len(s.lrus[e])
    assert n > s.max_blocks
    long = SR.Snapshot(**{**s.__dict__, "caps": s.caps.copy()})
    long.caps[e] = n - 1
    assert _info(SR.write(long))[0] == abi.FI_ERR_INVALID
    # lru_capacity 0: every capacity must be 0
    zero = SR.Snapshot(**{**s.__dict__, "lru_capacity": 0, "lrus": [np.zeros(0, np.uint64)] * E,
                          "caps": np.zeros(E, np.uint32)})
    assert _info(SR.write(zero))[0] == abi.FI_OK
    zero.caps[1] = s.max_blocks
    assert _info(SR.write(zero))[0] == abi.FI_ERR_INVALID
    # a version this library does not read, written whole with its own checksum
    assert _info(SR.write(s, version=2))[0] == abi.FI_ERR_INVALID


def _row(blob, lay, W, i, words):
    bad = bytearray(blob)
    struct.pack_into("<" + "I" * W, bad, lay["node_rows"] + 4 * W * i, *[int(w) for w in words])
    return SR.resealed(bytes(bad))


# ---- the format rule through libfi_hostcheck.so (snapshot_format.h) ----------------------------------------------
@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(os.path.join(abi.LIB_DIR, "libfi_hostcheck.so"))
    lib.fihc_snap_xxh64.restype = C.c_uint64
    lib.fihc_snap_xxh64.argtypes = [C.c_char_p, C.c_uint64]
    lib.fihc_snap_checksum.restype = C.c_uint64
    lib.fihc_snap_checksum.argtypes = [C.c_char_p, C.c_uint64, C.c_uint]
    lib.fihc_snap_check.restype = C.c_int
    lib.fihc_snap_check.argtypes = [C.c_char_p, C.c_uint64, C.c_uint, C.POINTER(C.c_uint64)]
    lib.fihc_snap_markers.restype = C.c_int
    lib.fihc_snap_markers.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    return lib


def test_word_xxh64_matches_the_oracle(hc):
    rng = np.random.default_rng(1)
    for n in list(range(0, 80)) + [1 << 20, (1 << 20) + 13, 3 * (1 << 20) + 4]:
        data = rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
        assert hc.fihc_snap_xxh64(data, n) == SR.xxh64(data), n


def test_checksum_over_chunks(hc):
    rng = np.random.default_rng(2)
    head = rng.integers(0, 256, size=64, dtype=np.uint8).tobytes()
    for n in (0, 4, 1 << 20, (1 << 20) + 4, 5 * (1 << 20) + 12):
        payload = rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
        want = SR.checksum(head[:56], payload)
        for threads in (1, 3, 8):
            assert hc.fihc_snap_checksum(head + payload, 64 + n, threads) == want, (n, threads)


def test_structural_check(hc):
    blob, s, lay = _blob_and_layout()
    pairs = C.c_uint64(0)
    for threads in (1, 4):
        assert hc.fihc_snap_check(blob, len(blob), threads, C.byref(pairs)) == 0
        assert pairs.value == len(s.pairs())
    assert hc.fihc_snap_check(blob[:-4], len(blob) - 4, 4, C.byref(pairs)) != 0
    W = SR.row_words(s.num_endpoints)
    bad = _row(blob, lay, W, len(s.node_keys) - 1, [0] * W)  # the last row: the last thread's range
    assert hc.fihc_snap_check(bad, len(bad), 4, C.byref(pairs)) != 0


def test_marker_positions(hc):
    pos = (C.c_uint64 * 2)()
    keys = np.array([5, U64_MAX, 7, 0, 9], dtype=np.uint64).tobytes()
    assert hc.fihc_snap_markers(keys, 5, pos) == 0 and list(pos) == [3, 1]
    keys = np.array([5, 7], dtype=np.uint64).tobytes()
    assert hc.fihc_snap_markers(keys, 2, pos) == 0 and list(pos) == [U64_MAX, U64_MAX]
    keys = np.array([0, 7, 0], dtype=np.uint64).tobytes()
    assert hc.fihc_snap_markers(keys, 3, pos) != 0


# ---- S.2d's state is sufficient (oracle only) ---------------------------------------------------------------------
def _same(a, b, cs, E, what):
    tok, offs, h0 = cs.tok, cs.offs, cs.h0
    ad = cs.adapters()
    got, want = a.pick_batch(tok, offs, h0, adapters=ad), b.pick_batch(tok, offs, h0, adapters=ad)
    assert H.picks_equal(got, want), what + " (single)\n" + H.describe_diff(got, want)
    got, want = a.pick_batch_ranked(tok, offs, h0, 4, adapters=ad), b.pick_batch_ranked(tok, offs, h0, 4, adapters=ad)
    assert H.picks_equal(got, want), what + " (ranked)\n" + H.describe_diff(got, want)
    sub = cs.subsets(E)
    got, want = a.pick_batch_subset(tok, offs, h0, sub, 4), b.pick_batch_subset(tok, offs, h0, sub, 4)
    assert H.picks_equal(got, want), what + " (subset)\n" + H.describe_diff(got, want)
    sa, sb = a.state(), b.state()
    assert sa[0] == sb[0], what + " (pairs)"
    assert all(np.array_equal(x, y) for x, y in zip(sa[1], sb[1])), what + " (LRUs)"
    assert sa[2] == sb[2], what + " (capacities)"


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_the_three_parts_carry_every_later_call(seed):
    E = 40
    src, cs, states = _aged(seed, E=E, n=24)
    dst = ExtOracle(src.cfg, track_removal=True)
    for entry in states:  # endpoint states and adapters are not part of the state: the caller re-sends them
        RR.apply(dst, entry)
    dst.load_state(*src.state())
    _same(src, dst, cs, E, "after the copy")
    for step in range(4):
        calls = cs.calls(E, n=6) + [("chains", cs.rng.integers(0, E, size=32).astype(np.uint32), cs.chains[:32].copy(),
                                     cs.nb[:32].copy())]
        for entry in calls:
            RR.apply(src, entry)
            RR.apply(dst, entry)
            if entry[0] in ("states", "lora"):
                states.append(entry)
        victim = [int(cs.rng.integers(0, E))]
        src.remove_endpoints(victim)
        dst.remove_endpoints(victim)
        _same(src, dst, cs, E, f"after step {step}")
    # and the copy through a blob, in shuffled node order, too
    again = ExtOracle(src.cfg, track_removal=True)
    for entry in states:
        RR.apply(again, entry)
    s = SR.read(SR.from_oracle(src, np.random.default_rng(seed)))
    again.load_state(s.pairs(), s.lrus, s.caps)
    _same(src, again, cs, E, "through a blob")
    for o in (src, dst, again):
        o.close()
