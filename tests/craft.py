"""Prompts whose block-hash chains hold a chosen value at a chosen block, and requests whose tie rotation starts at a
chosen endpoint (test helper, not collected).

The chain is h_i = XXH64(block_i ‖ LE64(h_{i-1})), h_0 = the request's seed (docs/SPEC.md S.1).  Every caller passes
h0 per request, and each link can be run backwards once the block's bytes are known.  When the message's last 8-byte
step is LE64(h_{i-1}), XXH64 ends in

    h_i = avalanche(rotl(pre_i ^ round(0, h_{i-1}), 27)·P1 + P4)

where pre_i (the state before that step) depends on the block's bytes only.  avalanche, rotl, ·P1 and round(0, ·) are
all bijections of 64-bit words, so every target t has exactly one h_{i-1}, and i + 1 such steps give the h0 that puts t
at block i of a prompt.  The message block ‖ LE64(h_prev) is block_bytes + 8 bytes long: its 32-byte stripes come
first, then its 8-byte steps.  So LE64(h_prev) is the last 8-byte step only when block_bytes % 8 == 0 and
block_bytes % 32 != 24.  At block_bytes ≡ 24 (mod 32) the message is a whole number of stripes, h_prev enters a
stripe accumulator and then the merge twice, and no closed-form inverse exists.  Those block sizes are rejected.

The tie rotation of a request starts at ((mix(seed) >> 32)·E) >> 32 (tiebreak.cuh), with seed = h_1 when the
request has blocks and h0 ^ (r + 1)·0x9E3779B97F4A7C15 when it has none.  mix is the SplitMix64 finaliser, also a
bijection, so any start s in [0, E) is reached by seed = mix⁻¹(ceil(s·2^32 / E) << 32).

The targets that matter are the hashes 0 and ~0: the index table's EMPTY / TOMB markers, which own the fixed nodes
C and C + 1 instead of a table slot.  Random prompts produce them with probability 2^-63 per block.
"""
from __future__ import annotations

import numpy as np

from oracle import epp_oracle as eo

MASK64 = (1 << 64) - 1
P1 = 0x9E3779B185EBCA87
P2 = 0xC2B2AE3D27D4EB4F
P3 = 0x165667B19E3779F9
P4 = 0x85EBCA77C2B2AE63
P1_INV, P2_INV, P3_INV = (pow(p, -1, 1 << 64) for p in (P1, P2, P3))
M1, M2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB  # tie_mix's multipliers
M1_INV, M2_INV = pow(M1, -1, 1 << 64), pow(M2, -1, 1 << 64)
GOLDEN = 0x9E3779B97F4A7C15  # the seed of a request without blocks: h0 ^ (r + 1)·GOLDEN
MARKERS = (0, MASK64)


def _rotl(x: int, r: int) -> int:
    return ((x << r) | (x >> (64 - r))) & MASK64


def _rotr(x: int, r: int) -> int:
    return _rotl(x, 64 - r)


def _unxorshift(y: int, s: int) -> int:
    """x with x ^ (x >> s) == y"""
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x


# ---- XXH64 pieces and their inverses ---------------------------------------------------------------------------
def round0(v: int) -> int:
    """round(0, v) = rotl(v·P2, 31)·P1"""
    return _rotl(v * P2 & MASK64, 31) * P1 & MASK64


def round0_inv(x: int) -> int:
    return _rotr(x * P1_INV & MASK64, 31) * P2_INV & MASK64


def avalanche(h: int) -> int:
    h ^= h >> 33
    h = h * P2 & MASK64
    h ^= h >> 29
    h = h * P3 & MASK64
    return h ^ (h >> 32)


def avalanche_inv(h: int) -> int:
    h ^= h >> 32
    h = _unxorshift(h * P3_INV & MASK64, 29)
    h = h * P2_INV & MASK64
    return h ^ (h >> 33)


def tie_mix(x: int) -> int:
    x ^= x >> 30
    x = x * M1 & MASK64
    x ^= x >> 27
    x = x * M2 & MASK64
    return x ^ (x >> 31)


def tie_mix_inv(y: int) -> int:
    y = _unxorshift(y, 31) * M2_INV & MASK64
    y = _unxorshift(y, 27) * M1_INV & MASK64
    return _unxorshift(y, 30)


def tie_start(seed: int, E: int) -> int:
    return ((tie_mix(seed) >> 32) * E) >> 32


def check_block_bytes(block_bytes: int):
    if block_bytes % 8 or block_bytes % 32 == 24:
        raise ValueError(f"block_bytes = {block_bytes}: LE64(h_prev) is not the last 8-byte step of XXH64 "
                         "(block_bytes % 8 != 0 or block_bytes % 32 == 24), the chain cannot be run backwards")


def pre(block: bytes) -> int:
    """the XXH64 state of block ‖ LE64(h_prev) right before the h_prev step, read back from XXH64(block ‖ 0^8):
    round(0, 0) = 0, so that hash is avalanche(rotl(pre, 27)·P1 + P4)"""
    check_block_bytes(len(block))
    h = eo.xxh64(bytes(block) + b"\0" * 8)
    return _rotr((avalanche_inv(h) - P4) * P1_INV & MASK64, 27)


def link(pre_i: int, prev: int) -> int:
    """one chain step from the block's pre-state: h_i from h_{i-1}"""
    return avalanche((_rotl(pre_i ^ round0(prev), 27) * P1 + P4) & MASK64)


def unlink(pre_i: int, h: int) -> int:
    """h_{i-1} from h_i"""
    return round0_inv(_rotr((avalanche_inv(h) - P4) * P1_INV & MASK64, 27) ^ pre_i)


def h0_for(blocks, i: int, target: int) -> int:
    """the seed h0 that makes chain[i] (0-based: the hash of blocks[i]) equal `target`"""
    h = int(target) & MASK64
    for j in range(i, -1, -1):
        h = unlink(pre(blocks[j]), h)
    return h


def h1_for_start(s: int, E: int, low: int = 0) -> int:
    """a first block hash (tie seed) whose rotation over E endpoints starts at s.  The start reads only the high 32
    bits of mix(seed): `low` sets the other 32, so that requests with one start need not share their first block."""
    assert 0 <= s < E and 0 <= low < 1 << 32
    x = -(-(s << 32) // E)  # ceil(s·2^32 / E) < 2^32
    return tie_mix_inv(x << 32 | low)


def h0_for_start(s: int, E: int, r: int, blocks=(), low: int = 0) -> int:
    """h0 of request r (its index in the batch) whose tie rotation starts at s: through h_1 when the prompt has
    blocks, through the seed h0 ^ (r + 1)·GOLDEN when it has none"""
    seed = h1_for_start(s, E, low)
    if len(blocks):
        return h0_for(blocks, 0, seed)
    return seed ^ ((r + 1) * GOLDEN & MASK64)


# ---- scenes ----------------------------------------------------------------------------------------------------
class Scene:
    """A batch of crafted requests: tok / offs (H.pack_prompts layout), h0 [R] uint64, and per request the block
    count n, the crafted position (None: not crafted) and its target.  blocks[r] are request r's whole blocks."""

    def __init__(self, blobs, blocks, h0, n, pos, target, block_bytes):
        from tests import helpers as H

        self.blobs, self.blocks = blobs, blocks
        self.tok, self.offs = H.pack_prompts(blobs)
        self.h0 = np.asarray(h0, dtype=np.uint64)
        self.n = np.asarray(n, dtype=np.int64)
        self.pos, self.target, self.B = list(pos), list(target), block_bytes
        self.R = len(blobs)

    def tiled(self, copies: int) -> "Scene":
        """the same requests repeated `copies` times (seeds of requests with blocks do not depend on r)"""
        assert (self.n > 0).all(), "a request without blocks takes its seed from its index"
        return Scene(self.blobs * copies, self.blocks * copies, np.tile(self.h0, copies), np.tile(self.n, copies),
                     self.pos * copies, self.target * copies, self.B)

    def chain(self, r: int, j: int) -> int:
        """the hash at block j of request r, by the forward links"""
        h = int(self.h0[r])
        for b in self.blocks[r][: j + 1]:
            h = link(pre(b), h)
        return h


def scene(specs, block_bytes: int, rng, tail=0) -> Scene:
    """specs: [(n_blocks, position, target)] -> a Scene.  position None: the request is left as drawn (random h0).
    Block bytes come from the seeded numpy Generator rng; tail > 0 appends 1 .. tail junk bytes (fewer than a block)
    after each prompt.  Crafting position i costs i + 1 XXH64 calls."""
    check_block_bytes(block_bytes)
    blobs, blocks, h0s, ns, ps, ts = [], [], [], [], [], []
    for r, (n, p, t) in enumerate(specs):
        raw = rng.integers(0, 256, size=n * block_bytes, dtype=np.uint8).tobytes()
        bl = [raw[j * block_bytes:(j + 1) * block_bytes] for j in range(n)]
        if p is None:
            h0 = int(rng.integers(0, 1 << 63)) << 1 | 1
        else:
            assert 0 <= p < n, (n, p)
            h0 = h0_for(bl, p, t)
        if tail:
            raw += b"\x5a" * (1 + r % min(tail, block_bytes - 1))
        blobs.append(raw)
        blocks.append(bl)
        h0s.append(h0)
        ns.append(n)
        ps.append(p)
        ts.append(t)
    return Scene(blobs, blocks, h0s, ns, ps, ts, block_bytes)
