"""An independent reader and writer of the index snapshot format (docs/SPEC.md S.2d, version 1), test infrastructure
only.  The checksum's XXH64 is the CPU oracle's (epo_xxh64), not the library's.

A blob is a 64-byte little-endian header (magic FIEPPSNP, version, header size, block_bytes, max_blocks, lru_capacity,
num_endpoints E, n_nodes, n_lru, payload bytes, checksum), then caps[E] u32, lru_len[E] u32, lru_keys[n_lru] u64,
node_keys[n_nodes] u64 and node_rows[n_nodes][ceil(E / 32)] u32.  The checksum is XXH64 of header[0:56] followed by the
LE64 XXH64 of each 1 MiB chunk of the payload."""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

from oracle import epp_oracle

HEADER = struct.Struct("<8sIIIIIIQQQQ")
MAGIC = b"FIEPPSNP"
CHUNK = 1 << 20
assert HEADER.size == 64


def xxh64(data: bytes) -> int:
    return int(epp_oracle.load().epo_xxh64(data, len(data), 0))


def checksum(header56: bytes, payload: bytes) -> int:
    inner = b"".join(struct.pack("<Q", xxh64(payload[o:o + CHUNK])) for o in range(0, len(payload), CHUNK))
    return xxh64(bytes(header56) + inner)


@dataclass
class Snapshot:
    block_bytes: int
    max_blocks: int
    lru_capacity: int
    num_endpoints: int
    caps: np.ndarray       # [E] u32
    lrus: list             # E arrays of u64 keys, least recently used first
    node_keys: np.ndarray  # [n] u64
    node_rows: np.ndarray  # [n, ceil(E / 32)] u32

    def pairs(self) -> set:
        """{(endpoint, hash)}"""
        out = set()
        for key, row in zip(self.node_keys.tolist(), self.node_rows):
            bits = np.unpackbits(row.view(np.uint8), bitorder="little")
            out.update((int(e), key) for e in np.flatnonzero(bits))
        return out


def row_words(E: int) -> int:
    return (E + 31) // 32


def rows_of(pairs, keys, E: int) -> np.ndarray:
    """membership rows of `keys` (in that order) from {(endpoint, hash)}"""
    at = {int(k): i for i, k in enumerate(keys)}
    rows = np.zeros((len(keys), row_words(E)), dtype=np.uint32)
    for e, h in pairs:
        rows[at[int(h)], e // 32] |= np.uint32(1 << (e % 32))
    return rows


def write(s: Snapshot, version: int = 1) -> bytes:
    E = s.num_endpoints
    lens = np.array([len(x) for x in s.lrus], dtype=np.uint32)
    lru_keys = np.concatenate([np.asarray(x, dtype=np.uint64) for x in s.lrus] + [np.zeros(0, np.uint64)])
    rows = np.ascontiguousarray(s.node_rows, dtype=np.uint32).reshape(len(s.node_keys), row_words(E))
    payload = (np.asarray(s.caps, dtype=np.uint32).tobytes() + lens.tobytes() + lru_keys.tobytes() +
               np.asarray(s.node_keys, dtype=np.uint64).tobytes() + rows.tobytes())
    head = HEADER.pack(MAGIC, version, 64, s.block_bytes, s.max_blocks, s.lru_capacity, E, len(s.node_keys),
                       len(lru_keys), len(payload), 0)
    return head[:56] + struct.pack("<Q", checksum(head[:56], payload)) + payload


def read(blob) -> Snapshot:
    blob = bytes(blob)
    magic, ver, hb, bb, mb, lc, E, nn, nl, pb, ck = HEADER.unpack_from(blob)
    assert magic == MAGIC and ver == 1 and hb == 64 and pb == len(blob) - 64, "malformed header"
    assert checksum(blob[:56], blob[64:]) == ck, "checksum mismatch"
    W = row_words(E)
    o = 64
    caps = np.frombuffer(blob, np.uint32, E, o)
    lens = np.frombuffer(blob, np.uint32, E, o + 4 * E)
    o += 8 * E
    keys = np.frombuffer(blob, np.uint64, nl, o)
    o += 8 * nl
    starts = np.concatenate([[0], np.cumsum(lens, dtype=np.int64)])
    lrus = [keys[starts[e]:starts[e + 1]].copy() for e in range(E)]
    node_keys = np.frombuffer(blob, np.uint64, nn, o).copy()
    o += 8 * nn
    node_rows = np.frombuffer(blob, np.uint32, nn * W, o).reshape(nn, W).copy()
    assert o + 4 * nn * W == len(blob)
    return Snapshot(bb, mb, lc, E, caps.copy(), lrus, node_keys, node_rows)


def layout(E: int, n_nodes: int, n_lru: int) -> dict:
    """absolute byte offsets of the sections and the end of the blob"""
    o = {"caps": 64, "lru_len": 64 + 4 * E, "lru_keys": 64 + 8 * E}
    o["node_keys"] = o["lru_keys"] + 8 * n_lru
    o["node_rows"] = o["node_keys"] + 8 * n_nodes
    o["end"] = o["node_rows"] + 4 * row_words(E) * n_nodes
    return o


def resealed(blob: bytes) -> bytes:
    """the blob with its checksum recomputed (to test the checks behind the checksum)"""
    return blob[:56] + struct.pack("<Q", checksum(blob[:56], blob[64:])) + blob[64:]


def from_oracle(ora, rng=None) -> bytes:
    """a blob of an ExtOracle's state; rng: the node order shuffled"""
    cfg = ora.cfg
    pairs, lrus, caps = ora.state()
    keys = np.array(sorted({h for _, h in pairs}), dtype=np.uint64)
    if rng is not None:
        keys = keys[rng.permutation(len(keys))]
    return write(Snapshot(cfg.block_bytes, cfg.max_blocks, cfg.lru_capacity, cfg.num_endpoints,
                          np.asarray(caps, dtype=np.uint32), lrus, keys, rows_of(pairs, keys, cfg.num_endpoints)))
