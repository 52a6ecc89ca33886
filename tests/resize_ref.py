"""The tests' reference for fi_epp_resize_pool (docs/SPEC.md S.2c), and a random call stream to drive it with.

S.2c defines a resize by a history: after a resize to E', the handle behaves like one created at E' and fed the same
calls, with everything ever addressed to an endpoint a shrink dropped left out.  History keeps those calls and replays
them, so filtered, into a fresh ResizeOracle: what tests/test_resize_cpu.py holds ResizeOracle.resize to.  CallStream makes
the calls: endpoint states with label bits, adapters, direct SETs and CLEARs (the index markers 0 and ~0 included),
batched Adds and per-endpoint LRU capacities, over prompts that share prefixes so that picks match across endpoints.
"""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import make_config, subset_bitsets
from tests import helpers as H
from tests.resize_oracle import ResizeOracle

P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
U64_MAX = 0xFFFFFFFFFFFFFFFF
LABEL = abi.FI_ROLE_FIRST_FREE  # a by-label filter's bit
# profile 0: prefill (prefix + load, by-label filter), profile 1: decode (adds the lora-affinity-scorer)
PROFILES = [{"name": "prefill", "role_mask": abi.FI_ROLE_PREFILLER | abi.FI_ROLE_WORKER, "more_filters": [LABEL],
             "scorers": [(P, 100), (K, 13), (Q, 7)]},
            {"name": "decode", "scorers": [(P, 100), (Q, 5), (L, 11)]}]
PD = {"prefill": 0, "decode": 1, "threshold": 96.0}
LORA_DTYPE = abi.lora_dtype()


def config(E, match_mode=abi.FI_MATCH_UPSTREAM, lru_capacity=48, max_blocks=16, max_batch=96, index_slots=0):
    return make_config(num_endpoints=E, block_bytes=32, max_blocks=max_blocks, lru_capacity=lru_capacity,
                       max_batch=max_batch, index_slots=index_slots, match_mode=match_mode, profiles=PROFILES, pd=PD)


class History:
    """the calls fed to a handle since create, with everything aimed at a dropped endpoint left out"""

    def __init__(self, cfg):
        self.cfg = abi.fi_epp_config.from_buffer_copy(cfg)
        self.log = []

    def record(self, entry):
        self.log.append(entry)

    def shrink(self, En):
        log = []
        for kind, *a in self.log:
            if kind in ("states", "lora", "ops"):
                rows = a[0][a[0]["endpoint"] < En]
                if len(rows):
                    log.append((kind, rows))
            elif kind == "chains":
                eps = a[0].copy()
                eps[(eps != abi.FI_NO_ENDPOINT) & (eps >= En)] = abi.FI_NO_ENDPOINT
                log.append((kind, eps, a[1], a[2]))
            else:  # caps
                keep = a[0] < En
                if keep.any():
                    log.append((kind, a[0][keep], a[1][keep]))
        self.log = log

    def replay(self, E) -> ResizeOracle:
        cfg = abi.fi_epp_config.from_buffer_copy(self.cfg)
        cfg.num_endpoints = cfg.endpoint_count = E
        ora = ResizeOracle(cfg, track_removal=True)
        for entry in self.log:
            apply(ora, entry)
        return ora


def apply(target, entry):
    """one call on an EndpointPicker or a ResizeOracle"""
    kind, *a = entry
    if kind == "states":
        target.update_endpoints(a[0])
    elif kind == "lora":
        target.update_endpoints_lora(a[0])
    elif kind == "ops":
        target.index_apply(a[0])
    elif kind == "chains":
        target.index_add_chains(a[0], a[1], a[2])
    else:
        target.set_lru_capacities(a[0], a[1])


class CallStream:
    """random calls over a fixed set of prompts: G prefix groups of 4..10 blocks, each prompt a group's prefix and a
    tail of its own"""

    def __init__(self, seed, cfg, R=64, G=10):
        self.rng = np.random.default_rng(seed)
        self.cfg = cfg
        B, M = cfg.block_bytes, cfg.max_blocks
        heads = [self.rng.integers(0, 256, size=B * int(self.rng.integers(4, 11)), dtype=np.uint8) for _ in range(G)]
        blobs = []
        for r in range(R):
            tail = self.rng.integers(0, 256, size=int(self.rng.integers(0, (M - 4) * B)), dtype=np.uint8)
            blobs.append(bytes(heads[r % G]) + bytes(tail))
        self.tok, self.offs = H.pack_prompts(blobs)
        self.h0 = 0x5EED
        self.R = R
        ora = ResizeOracle(cfg)
        self.chains, self.nb = ora.hash_batch(self.tok, self.offs, self.h0)
        ora.close()
        self.hashes = np.unique(np.concatenate([self.chains[r, : self.nb[r]] for r in range(R)] +
                                               [np.array([0, U64_MAX], dtype=np.uint64)]))

    def calls(self, E, n=6):
        """n random calls addressed to endpoints [0, E)"""
        out = []
        rng = self.rng
        for _ in range(n):
            kind = rng.choice(["states", "lora", "ops", "ops", "chains", "chains", "caps"])
            if kind == "states":
                eps = rng.choice(E, size=min(E, int(rng.integers(1, 40))), replace=False)
                s = H.states_array(len(eps), kv=rng.random(len(eps)), queue=rng.integers(0, 50, size=len(eps)),
                                   roles=rng.choice([abi.FI_ROLE_WORKER | LABEL, abi.FI_ROLE_PREFILLER | LABEL,
                                                     abi.FI_ROLE_DECODER, abi.FI_ROLE_PREFILLER], size=len(eps)),
                                   alive=rng.choice([abi.FI_ENDPOINT_ALIVE] * 5 + [0], size=len(eps)))
                s["endpoint"] = eps
                out.append(("states", s))
            elif kind == "lora":
                eps = rng.choice(E, size=min(E, int(rng.integers(1, 6))), replace=False)
                s = np.zeros(len(eps), dtype=LORA_DTYPE)
                s["endpoint"] = eps
                s["max_active"] = rng.integers(0, 3, size=len(eps))
                s["n_active"] = rng.integers(0, 3, size=len(eps))
                s["active"][:, :2] = rng.integers(1, 4, size=(len(eps), 2))
                out.append(("lora", s))
            elif kind == "ops":
                m = int(rng.integers(1, 120))
                ops = np.zeros(m, dtype=H.OP_DTYPE)
                ops["hash"] = rng.choice(self.hashes, size=m)
                ops["endpoint"] = rng.integers(0, E, size=m)
                ops["op"] = rng.choice([abi.FI_OP_SET] * 4 + [abi.FI_OP_CLEAR], size=m)
                out.append(("ops", ops))
            elif kind == "chains":
                rows = rng.integers(0, self.R, size=int(rng.integers(1, 48)))
                eps = rng.integers(0, E, size=len(rows)).astype(np.uint32)
                eps[rng.random(len(rows)) < 0.1] = abi.FI_NO_ENDPOINT
                out.append(("chains", eps, self.chains[rows].copy(), self.nb[rows].copy()))
            else:
                eps = rng.choice(E, size=min(E, int(rng.integers(1, 4))), replace=False).astype(np.uint32)
                caps = rng.integers(self.cfg.max_blocks, self.cfg.lru_capacity + 1, size=len(eps)).astype(np.uint32)
                caps[rng.random(len(eps)) < 0.2] = 0
                out.append(("caps", eps, caps))
        return out

    def subsets(self, E):
        rng = self.rng
        rows = []
        for r in range(self.R):
            x = rng.random()
            rows.append(None if x < 0.2 else [] if x < 0.25 else rng.choice(E, size=min(E, int(rng.integers(1, 9))),
                                                                           replace=False))
        return subset_bitsets(rows, E)

    def adapters(self):
        return self.rng.integers(0, 4, size=self.R).astype(np.uint64)
