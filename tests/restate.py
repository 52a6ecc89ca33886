"""A SECOND, independent restatement of SURVEY.md Appendix A.1-A.6 (+ the tie rule of include/fi_epp.h) in plain
Python / numpy — test infrastructure.

Purpose (VERDICT r1, "parity is partial"): the C++ oracle and the CUDA kernels were written by the same hand from
the same appendix; this module shares NO code with either (no import from oracle/, nothing from the package
beyond the numpy record layouts of the C ABI) and uses different data structures (python dicts of sets, python
floats, the `xxhash` wheel for XXH64), so a misreading of the appendix would have to be made three times in
three different shapes to go unnoticed.  It is slow: use it on small workloads only.

Semantics restated:
  A.1 chain        h_i = XXH64(block_i ‖ LE64(h_{i-1})), h_0 = seed; partial trailing block dropped; cap M
  A.2 index        dict hash -> set(endpoints); SET adds, CLEAR discards; LRU add with hashicorp semantics
  A.3 match        upstream: stop at the first block with an empty set, count membership per endpoint before it
                   lpm: per-endpoint longest contiguous prefix
  A.4 score        prefix m/n (0 if n = 0); kv 1 - util; queue (max-q)/(max-min) over the FILTERED set (1.0 if
                   equal); lora 1.0 / 0.8 / 0.6 / 0; total = sum clamp01(s)·w in profile order (IEEE double)
  A.5 pick         max total over alive endpoints passing the profile's role filter; ties by the request's
                   rotation (fi_epp.h "Ties")
  A.6 PD           decode first; prefill stands iff (1 - m_dec/n)·len >= threshold
  shard view       (docs/SPEC.md S.2e) a handle over endpoints [b, b + c): ops and Adds for other endpoints are
                   dropped, only its own endpoints are candidates; queue min/max and the rotation stay pool-wide
"""
from __future__ import annotations

import struct
from collections import OrderedDict

import numpy as np

NO_ENDPOINT = 0xFFFFFFFF
MASK64 = (1 << 64) - 1
KIND_PREFIX, KIND_KV, KIND_QUEUE, KIND_LORA = 1, 2, 3, 4
ALIVE = 1


def chain(prompt: bytes, block_bytes: int, max_blocks: int, h0: int):
    import xxhash

    n = min(len(prompt) // block_bytes, max_blocks)
    out, prev = [], h0
    for i in range(n):
        prev = xxhash.xxh64_intdigest(prompt[i * block_bytes:(i + 1) * block_bytes] + struct.pack("<Q", prev))
        out.append(prev)
    return out


def tie_start(n_blocks: int, first_hash: int, h0: int, r: int, E: int) -> int:
    x = first_hash if n_blocks else (h0 ^ (((r + 1) * 0x9E3779B97F4A7C15) & MASK64))
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    x = x ^ (x >> 31)
    return ((x >> 32) * E) >> 32


class Restatement:
    def __init__(self, num_endpoints, block_bytes, max_blocks, profiles, pd=None, lpm=False, lru_capacity=0, shard=None):
        """profiles: [{"filters": [label-bit masks, ANDed], "scorers": [(kind, weight), ...]}]; pd: {"decode", "prefill", "threshold"};
        shard: (b, c) for the view of a handle over endpoints [b, b + c)"""
        self.E, self.B, self.M = num_endpoints, block_bytes, max_blocks
        self.own = range(num_endpoints) if shard is None else range(shard[0], shard[0] + shard[1])
        self.profiles, self.pd, self.lpm = profiles, pd, lpm
        self.index = {}  # hash -> set of endpoints
        self.state = {}  # endpoint -> dict(role_mask, kv_util, queue, flags)
        self.lora = {}   # endpoint -> (max_active, [active], [waiting])
        self.cap = lru_capacity
        self.lru = {}    # endpoint -> OrderedDict (last = most recent)

    # ---- A.2
    def apply(self, ops):
        for h, e, op in zip(ops["hash"].tolist(), ops["endpoint"].tolist(), ops["op"].tolist()):
            if e not in self.own:
                continue
            if op == 1:
                self.index.setdefault(h, set()).add(e)
            else:
                s = self.index.get(h)
                if s is not None:
                    s.discard(e)

    def add_chain(self, endpoint, hashes):
        if endpoint not in self.own:
            return
        d = self.lru.setdefault(endpoint, OrderedDict())
        for h in hashes:
            h = int(h)
            if h in d:
                d.move_to_end(h)
                continue
            d[h] = True
            self.index.setdefault(h, set()).add(endpoint)
            if len(d) > self.cap:
                old, _ = d.popitem(last=False)
                self.index[old].discard(endpoint)

    def update_endpoints(self, states):
        for s in states:
            self.state[int(s["endpoint"])] = dict(role_mask=int(s["role_mask"]), kv_util=float(s["kv_util"]),
                                                  queue=int(s["queue_depth"]), flags=int(s["flags"]))

    def update_lora(self, states):
        for s in states:
            self.lora[int(s["endpoint"])] = (int(s["max_active"]), [int(x) for x in s["active"][: int(s["n_active"])]],
                                             [int(x) for x in s["waiting"][: int(s["n_waiting"])]])

    # ---- A.3
    def match(self, ch):
        counts = {}
        if not self.lpm:
            for h in ch:
                s = self.index.get(h)
                if not s:
                    break
                for e in s:
                    counts[e] = counts.get(e, 0) + 1
        else:
            alive = None
            for h in ch:
                s = self.index.get(h)
                if not s:
                    break
                alive = set(s) if alive is None else (alive & s)
                if not alive:
                    break
                for e in alive:
                    counts[e] = counts.get(e, 0) + 1
        return counts

    # ---- A.4
    def _eligible(self, e, prof):
        st = self.state.get(e)
        if st is None or not (st["flags"] & ALIVE):
            return False
        return all(st["role_mask"] & f for f in prof.get("filters", []))

    def _lora_score(self, e, adapter):
        mx, act, wai = self.lora.get(e, (0, [], []))
        if adapter in act:
            return 1.0
        if len(act) + len(wai) < mx:
            return 0.8
        return 0.6 if adapter in wai else 0.0

    def pick(self, prompts, offsets, h0, adapters=None):
        R = len(offsets) - 1
        P = len(self.profiles)
        out = np.zeros((R, P), dtype=[("endpoint", "<u4"), ("match_blocks", "<u2"), ("n_blocks", "<u2"), ("score", "<f8")])
        raw = bytes(np.ascontiguousarray(prompts).view(np.uint8))
        h0 = np.broadcast_to(np.asarray(h0, dtype=np.uint64), (R,))
        qctx = []
        for prof in self.profiles:
            qs = [self.state[e]["queue"] for e in range(self.E) if self._eligible(e, prof)]
            qctx.append((min(qs), max(qs)) if qs else (0, 0))
        for r in range(R):
            p = raw[int(offsets[r]):int(offsets[r + 1])]
            ch = chain(p, self.B, self.M, int(h0[r]))
            n = len(ch)
            counts = self.match(ch)
            start = tie_start(n, ch[0] if n else 0, int(h0[r]), r, self.E)
            ad = int(adapters[r]) if adapters is not None else 0
            for pi, prof in enumerate(self.profiles):
                best = None
                mn, mx = qctx[pi]
                for e in self.own:
                    if not self._eligible(e, prof):
                        continue
                    st = self.state[e]
                    m = counts.get(e, 0)
                    total = 0.0
                    for kind, w in prof["scorers"]:
                        if kind == KIND_PREFIX:
                            s = (m / n) if n else 0.0
                        elif kind == KIND_KV:
                            s = 1.0 - st["kv_util"]
                        elif kind == KIND_QUEUE:
                            s = 1.0 if mx == mn else (mx - st["queue"]) / (mx - mn)
                        else:
                            s = self._lora_score(e, ad)
                        s = 0.0 if s < 0.0 else (1.0 if s > 1.0 else s)
                        total = total + s * float(w)
                    key = (-total, (e - start) % self.E)
                    if best is None or key < best[0]:
                        best = (key, e, m, total)
                if best is None:
                    out[r, pi] = (NO_ENDPOINT, 0, n, 0.0)
                else:
                    out[r, pi] = (best[1], best[2], n, best[3])
            if self.pd:
                d = out[r, self.pd["decode"]]
                hit = (int(d["match_blocks"]) / n) if (d["endpoint"] != NO_ENDPOINT and n) else 0.0
                if not ((1.0 - hit) * float(len(p)) >= float(self.pd.get("threshold", 0.0))):
                    out[r, self.pd["prefill"]] = (NO_ENDPOINT, 0, n, 0.0)
        return out


def from_config(cfg, lpm=None, shard=None):
    """Build a Restatement from an abi.fi_epp_config (ctypes struct: layout only, no library call)."""
    profiles = []
    for i in range(cfg.n_profiles):
        p = cfg.profiles[i]
        filters = ([int(p.role_mask)] if p.role_mask else []) + [int(p.more_filters[f]) for f in range(p.n_more_filters)]
        profiles.append({"filters": filters,
                         "scorers": [(int(p.scorers[j].kind), int(p.scorers[j].weight)) for j in range(p.n_scorers)]})
    pd = None
    if cfg.pd_enabled:
        pd = {"decode": int(cfg.pd_decode_profile), "prefill": int(cfg.pd_prefill_profile), "threshold": float(cfg.pd_threshold)}
    return Restatement(cfg.num_endpoints, cfg.block_bytes, cfg.max_blocks, profiles, pd,
                       lpm=bool(cfg.match_mode) if lpm is None else lpm, lru_capacity=int(cfg.lru_capacity), shard=shard)
