"""The CPU oracle with upstream indexer.RemovePod on top, for the tests of fi_epp_index_remove_endpoints.

The oracle has no removal of its own, and none is needed.  Its index is a set of (endpoint, hash) pairs.  A direct
SET / CLEAR changes one pair, and an Add to endpoint e changes only pairs of e (through e's own LRU).  So the state
after removing a set D of endpoints is the state the same calls produce with everything aimed at D left out: D's
pairs are gone, D's LRUs are empty, and every other endpoint's pairs and LRU are what they were.  RemovalOracle keeps
the calls it forwarded and, on a removal, rebuilds a fresh oracle by replaying them without D.  The pairs removed are
counted by probing the old oracle for every hash ever aimed at a removed endpoint.
"""
from __future__ import annotations

import numpy as np

from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo


class RemovalOracle:
    def __init__(self, cfg: abi.fi_epp_config):
        self.cfg = abi.fi_epp_config.from_buffer_copy(cfg)
        self.E = cfg.num_endpoints
        self._log = []    # ("states" | "lora", array) | ("ops", array) | ("chain", e, keys) | ("chains", eps, chains, nb)
        self._seen = {}   # endpoint -> hashes ever aimed at it since its last removal
        self._cpu = eo.Oracle(self.cfg)

    def close(self):
        self._cpu.close()

    # -- forwarded calls, logged -----------------------------------------------------
    def _replay(self, cpu, entry):
        kind = entry[0]
        if kind == "states":
            cpu.update_endpoints(entry[1])
        elif kind == "lora":
            cpu.update_endpoints_lora(entry[1])
        elif kind == "ops":
            cpu.index_apply(entry[1])
        elif kind == "chain":
            cpu.index_add_chain(entry[1], entry[2])
        else:
            cpu.index_add_chains(entry[1], entry[2], entry[3])

    def _do(self, entry):
        self._log.append(entry)
        self._replay(self._cpu, entry)

    def _see(self, e, hashes):
        self._seen.setdefault(int(e), set()).update(int(h) for h in hashes)

    def update_endpoints(self, states):
        self._do(("states", np.array(states, copy=True)))

    def update_endpoints_lora(self, states):
        self._do(("lora", np.array(states, copy=True)))

    def index_apply(self, ops):
        ops = np.array(ops, dtype=eo.OP_DTYPE, copy=True)
        for e in np.unique(ops["endpoint"]):
            self._see(e, ops["hash"][ops["endpoint"] == e])
        self._do(("ops", ops))

    def index_add_chain(self, endpoint: int, hashes):
        hashes = np.array(hashes, dtype=np.uint64, copy=True)
        self._see(endpoint, hashes)
        self._do(("chain", int(endpoint), hashes))

    def index_add_chains(self, endpoints, chains, nblocks):
        endpoints = np.array(endpoints, dtype=np.uint32, copy=True)
        chains = np.array(chains, dtype=np.uint64, copy=True)
        nblocks = np.array(nblocks, dtype=np.uint32, copy=True)
        for r, e in enumerate(endpoints):
            if e != abi.FI_NO_ENDPOINT:
                self._see(e, chains[r, : nblocks[r]])
        self._do(("chains", endpoints, chains, nblocks))

    def index_contains(self, endpoint: int, h: int) -> bool:
        return self._cpu.index_contains(endpoint, h)

    def hash_batch(self, *a, **kw):
        return self._cpu.hash_batch(*a, **kw)

    def pick_batch(self, *a, **kw):
        return self._cpu.pick_batch(*a, **kw)

    # -- indexer.RemovePod -----------------------------------------------------------
    def remove_endpoints(self, endpoints) -> int:
        """-> the (endpoint, hash) pairs removed.  ValueError (and nothing changes) for an endpoint out of range."""
        drop = {int(e) for e in np.atleast_1d(np.asarray(endpoints, dtype=np.int64))}
        if any(e < 0 or e >= self.E for e in drop):
            raise ValueError("endpoint out of range")
        removed = sum(self._cpu.index_contains(e, h) for e in drop for h in self._seen.get(e, ()))
        log = []
        for entry in self._log:
            kind = entry[0]
            if kind == "ops":
                ops = entry[1][~np.isin(entry[1]["endpoint"], list(drop))]
                if len(ops):
                    log.append(("ops", ops))
            elif kind == "chain":
                if entry[1] not in drop:
                    log.append(entry)
            elif kind == "chains":
                eps = entry[1].copy()
                eps[np.isin(eps, list(drop))] = abi.FI_NO_ENDPOINT
                log.append(("chains", eps, entry[2], entry[3]))
            else:
                log.append(entry)
        cpu = eo.Oracle(self.cfg)
        for entry in log:
            self._replay(cpu, entry)
        self._cpu.close()
        self._cpu, self._log = cpu, log
        for e in drop:
            self._seen.pop(e, None)
        return int(removed)
