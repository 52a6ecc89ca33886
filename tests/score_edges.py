"""Edge cases of the fp64 scoring of docs/SPEC.md S.4, S.6, S.6a and S.7, and an exact reference of it (helper module
of test_score_edges_cpu.py and test_gpu_score_edges.py; not collected).

The picks are one exact sequence of fp64 operations.  Ordinary workloads keep kv_util in [0, 1) on a dyadic grid,
queue depths small and weights at most 100, where most of that sequence cannot go wrong.  The cases here set:
  - kv_util below 0 and above 1 (the clamp), +-1e308, -0.0, subnormals, non-dyadic values, nextafter around 0 and 1;
  - queue depths INT32_MIN and INT32_MAX in one eligible set, negative depths, all depths equal, one eligible endpoint;
  - weights 0, 1, 2^31 - 1 and mixed magnitudes, FI_EPP_MAX_SCORERS scorers with a kind repeated;
  - PD thresholds equal to fl(fl(1 - fl(m/n)) * len) and the doubles on each side of it, +-inf, a negative one;
  - ties between matched and zero-match endpoints (prefix weight 0, many endpoints in one identical state), so the
    tie rotation alone decides them;
  - pools in which two endpoints' exact rational totals tie but their fp64 totals do not, so the rounding order of
    S.4 alone decides the pick.
Match counts are set per request and endpoint: every prompt has a chosen number of whole blocks (0 included) and
the index holds, per endpoint, a chosen prefix of the request's own chain (with holes for LPM), through direct SETs.

spec_total() evaluates S.4 with fractions.Fraction, rounding to the nearest double after every operation;
Spec.picks() and Spec.ranked() apply S.5a, S.6, S.6a and S.7 on top.  None of it shares code with the oracle or
tests/restate.py.  A `variant` models one plausible wrong kernel (VARIANTS); the CPU suite checks that every variant
changes some expected output of the cases, so the bit-exact comparisons on the GPU can see each of them.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass
from fractions import Fraction
from typing import Optional

import numpy as np

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import make_config, synth

PICK_DTYPE, OP_DTYPE, ENDPOINT_DTYPE = abi.np_dtypes()
LORA_DTYPE = abi.lora_dtype()
NO = abi.FI_NO_ENDPOINT
P, K, Q, L = abi.FI_SCORER_PREFIX, abi.FI_SCORER_KV_UTIL, abi.FI_SCORER_QUEUE, abi.FI_SCORER_LORA
I32_MIN, I32_MAX = -(2**31), 2**31 - 1
W_MAX = 2**31 - 1
BLOCK_BYTES = 64
MAX_BLOCKS = 24
ROLE_FEW = abi.FI_ROLE_FIRST_FREE  # a label only a handful of endpoints carry
MASK64 = (1 << 64) - 1

KV_EDGES = [-1e308, 1e308, -0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 0.1, 1 / 3, 0.7, 2 / 3, 0.3, 1.0,
            -0.5, 1.5, 2.0, math.nextafter(0.0, 1.0), math.nextafter(0.0, -1.0), math.nextafter(1.0, 0.0),
            math.nextafter(1.0, 2.0), 0.25, 0.9]
Q_EDGES = [I32_MIN, I32_MAX, I32_MIN + 1, I32_MAX - 1, -1, 0, 1, -7, 5, 1000, -(2**30)]

# one plausible wrong kernel each
VARIANTS = (
    "prefix_last",  # per-endpoint precomputed base of the other scorers, plus m/n * w added last
    "fma",          # total = fl(v * w + total) (a fused multiply-add)
    "rcp",          # prefix score m * fl(1 / n)
    "q_int32",      # queue score from int32 (wrapping) differences
    "no_clamp",     # scores not clamped to [0, 1]
    "reverse",      # scorers accumulated in reverse profile order
    "pd_gt",        # PD: the prefill pick stands iff miss > threshold
    "zero_tie",     # single pick: a matched endpoint wins a tie with a zero-match endpoint whatever the rotation
)


# ---- fp64 operations, each rounded once (exact rational arithmetic, then the nearest double) ----------------
def _rnd(q: Fraction) -> float:
    try:
        return float(q)  # int / int true division: correctly rounded
    except OverflowError:
        return math.inf if q > 0 else -math.inf


def _op(a: float, b: float, f) -> float:
    if math.isfinite(a) and math.isfinite(b):
        return _rnd(f(Fraction(a), Fraction(b)))
    return float(f(a, b))  # an infinity (only the no_clamp variant gets here): IEEE


def fadd(a, b):
    return _op(a, b, lambda x, y: x + y)


def fsub(a, b):
    return _op(a, b, lambda x, y: x - y)


def fmul(a, b):
    return _op(a, b, lambda x, y: x * y)


def fdiv(a, b):
    return _op(a, b, lambda x, y: x / y)


def ffma(a, b, c):
    if math.isfinite(a) and math.isfinite(b) and math.isfinite(c):
        return _rnd(Fraction(a) * Fraction(b) + Fraction(c))
    return a * b + c


def _wrap32(x: int) -> int:
    return ((x + 2**31) % 2**32) - 2**31


def lora_value(lora_row, adapter: int) -> float:
    """S.4 lora-affinity: active 1.0, room for another adapter 0.8, queued 0.6, else 0"""
    if lora_row is None:
        return 0.0
    mx, act, wai = lora_row
    if adapter in act:
        return 1.0
    if len(act) + len(wai) < mx:
        return 0.8
    return 0.6 if adapter in wai else 0.0


@functools.lru_cache(maxsize=None)
def spec_total(scorers: tuple, m: int, n: int, kv: float, q: int, qmin: int, qmax: int, lora_v: float = 0.0,
               variant: Optional[str] = None) -> float:
    """S.4: total = 0; for each (kind, weight) in profile order: total = fl(total + fl(clamp01(score) * weight)).
    qmin / qmax: the queue depths' min and max over the eligible set the pick is taken over."""
    def value(kind):
        if kind == P:
            if not n:
                return 0.0
            return fmul(float(m), fdiv(1.0, float(n))) if variant == "rcp" else fdiv(float(m), float(n))
        if kind == K:
            return fsub(1.0, kv)
        if kind == Q:
            if qmax == qmin:
                return 1.0
            num, den = qmax - q, qmax - qmin
            if variant == "q_int32":
                num, den = _wrap32(num), _wrap32(den)
            return fdiv(float(num), float(den))
        return lora_v

    order = list(scorers)
    if variant == "reverse":
        order.reverse()
    elif variant == "prefix_last":
        order = [s for s in order if s[0] != P] + [s for s in order if s[0] == P]
    total = 0.0
    for kind, w in order:
        v = value(kind)
        if variant != "no_clamp":
            v = 0.0 if v < 0.0 else (1.0 if v > 1.0 else v)
        total = ffma(v, float(w), total) if variant == "fma" else fadd(total, fmul(v, float(w)))
    return total


def tie_start(n: int, first_hash: int, h0: int, r: int, E: int) -> int:
    """S.6: the request's rotation start"""
    x = first_hash if n else (h0 ^ (((r + 1) * 0x9E3779B97F4A7C15) & MASK64))
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    x ^= x >> 31
    return ((x >> 32) * E) >> 32


def pd_runs(dec_e: int, dec_m: int, n: int, length: int, threshold: float, variant: Optional[str] = None) -> bool:
    """S.7: the prefill pick stands iff fl(fl(1 - hit) * len) >= threshold"""
    hit = fdiv(float(dec_m), float(n)) if (dec_e != NO and n) else 0.0
    miss = fmul(fsub(1.0, hit), float(length))
    return miss > threshold if variant == "pd_gt" else miss >= threshold


# ---- cases -------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    E: int
    mode: int
    profiles: list           # [{"name", "role_mask", "scorers": [(kind, weight)]}]
    pd: Optional[dict]
    states: np.ndarray       # ENDPOINT_DTYPE [E]
    lora: Optional[np.ndarray]
    ops: np.ndarray          # OP_DTYPE SETs
    tok: np.ndarray          # uint8 prompt bytes
    offs: np.ndarray         # uint64 [R + 1]
    adapters: Optional[np.ndarray]
    h0: int = synth.xxh64_py(synth.MODEL_NAME)
    max_blocks: int = MAX_BLOCKS

    @property
    def R(self) -> int:
        return len(self.offs) - 1

    def config(self, **kw):
        args = dict(num_endpoints=self.E, block_bytes=BLOCK_BYTES, max_blocks=self.max_blocks, lru_capacity=0,
                    max_batch=self.R, profiles=self.profiles, pd=self.pd, match_mode=self.mode, index_slots=1 << 16,
                    max_prompt_bytes=int(self.offs[-1]) + 64)
        args.update(kw)
        return make_config(**args)

    def load(self, g):
        """the case's endpoint state and index into a picker or an oracle"""
        g.update_endpoints(self.states)
        if self.lora is not None:
            g.update_endpoints_lora(self.lora)
        g.index_apply(self.ops)


def _prompt(rng, nblocks: int, tail: int) -> bytes:
    return rng.integers(0, 256, nblocks * BLOCK_BYTES + tail, dtype=np.uint8).tobytes()


def _chain(prompt: bytes, max_blocks: int, h0: int) -> np.ndarray:
    return synth.chain_py(prompt, BLOCK_BYTES, max_blocks, h0)


class _Builder:
    def __init__(self, E, mode, seed, max_blocks=MAX_BLOCKS):
        self.E, self.mode, self.max_blocks = E, mode, max_blocks
        self.rng = np.random.default_rng(seed)
        self.h0 = synth.xxh64_py(synth.MODEL_NAME)
        self.prompts, self.ops = [], []

    def request(self, nblocks: int, tail: Optional[int] = None, matches=()):
        """one prompt of `nblocks` whole blocks; matches: [(endpoint, m)] -> SETs of the first m blocks of its chain
        (in LPM mode a third of them leave a hole in the middle)"""
        tail = int(self.rng.integers(0, BLOCK_BYTES)) if tail is None else tail
        p = _prompt(self.rng, nblocks, tail)
        ch = _chain(p, self.max_blocks, self.h0)
        for e, m in matches:
            blocks = list(range(min(m, len(ch))))
            if self.mode == abi.FI_MATCH_LPM and len(blocks) > 2 and self.rng.random() < 0.33:
                blocks.pop(int(self.rng.integers(1, len(blocks) - 1)))
            self.ops += [(int(ch[i]), int(e), abi.FI_OP_SET) for i in blocks]
        self.prompts.append(p)

    def random_request(self, pool, n_max_matched=6):
        n = int(self.rng.choice([0, 1, 2, 3, 5, 8, 13, self.max_blocks, self.max_blocks + 3]))
        k = int(self.rng.integers(0, min(len(pool), n_max_matched) + 1)) if n else 0
        eps = self.rng.choice(pool, k, replace=False) if k else []
        self.request(n, matches=[(int(e), int(self.rng.integers(1, min(n, self.max_blocks) + 1))) for e in eps])

    def finish(self, name, profiles, pd, states, lora=None, adapters=None):
        ops = np.zeros(len(self.ops), dtype=OP_DTYPE)
        for i, t in enumerate(self.ops):
            ops[i] = t
        offs = np.zeros(len(self.prompts) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(p) for p in self.prompts])
        tok = np.frombuffer(b"".join(self.prompts) + b"\0" * 16, dtype=np.uint8).copy()
        return Case(name, self.E, self.mode, profiles, pd, states, lora, ops, tok, offs, adapters, self.h0, self.max_blocks)


def _states(E):
    s = np.zeros(E, dtype=ENDPOINT_DTYPE)
    s["endpoint"] = np.arange(E)
    s["role_mask"] = abi.FI_ROLE_WORKER
    s["flags"] = abi.FI_ENDPOINT_ALIVE
    return s


def case_edges(E, mode, seed, R=256):
    """clamp / integer-range edges: every kv and queue edge value, extreme weights, a kind repeated, a profile whose
    filter admits a handful of endpoints (ranked k above its eligible count)"""
    b = _Builder(E, mode, seed)
    rng = b.rng
    st = _states(E)
    st["kv_util"] = rng.choice(KV_EDGES + [0.5, 0.75, 0.125], E)
    st["queue_depth"] = rng.choice(Q_EDGES, E)
    st["queue_depth"][0], st["queue_depth"][E - 1] = I32_MIN, I32_MAX
    few = rng.choice(E, min(E, 5), replace=False)
    st["role_mask"][few] |= ROLE_FEW
    st["role_mask"][[0, E - 1]] |= ROLE_FEW
    dead = rng.random(E) < 0.1
    dead[[0, E - 1]] = False
    st["flags"][dead] = 0
    profiles = [{"name": "mixed", "scorers": [(K, W_MAX), (P, 3), (Q, 1), (K, 0)]},
                {"name": "few", "role_mask": ROLE_FEW, "scorers": [(Q, W_MAX), (P, 1), (Q, 2)]},
                {"name": "prefix", "scorers": [(P, 100), (K, 1), (Q, 65536)]}]
    for _ in range(R):
        b.random_request(np.arange(E))
    return b.finish("edges", profiles, None, st)


def case_zero_tie(E, mode, seed, R=256):
    """most endpoints in one best state (kv below 0, -1e308 or exactly 0 clamp to the same score; queue INT32_MIN):
    the zero-match tie set holds most of the pool, matched endpoints among them, and with prefix weight 0 the tie
    rotation alone picks"""
    b = _Builder(E, mode, seed)
    rng = b.rng
    st = _states(E)
    tied = rng.random(E) < 0.6
    tied[0] = True
    st["kv_util"] = np.where(tied, rng.choice([-0.5, -1e308, 0.0, -0.0, -5e-324], E), rng.choice([0.1, 0.7, 1 / 3, 0.9], E))
    st["queue_depth"] = np.where(tied, I32_MIN, rng.choice([I32_MIN + 1, 0, I32_MAX, 12], E))
    if E > 2:
        st["queue_depth"][E - 1] = I32_MAX
    profiles = [{"name": "kvq", "scorers": [(P, 0), (K, 3), (Q, 5)]},
                {"name": "qbig", "scorers": [(K, 1), (P, 0), (Q, W_MAX)]},
                {"name": "none", "scorers": [(P, 0)]}]
    pool_tied = np.flatnonzero(tied)
    for r in range(R):
        pool = pool_tied if r % 3 else np.arange(E)
        b.random_request(pool, n_max_matched=12)
    return b.finish("zero_tie", profiles, None, st)


PD_THRESHOLDS = ("exact", "exact_full", "below", "above", "+inf", "-inf", "neg")
PD_N0, PD_M0, PD_TAIL = 10, 3, 37  # hit fl(3/10), len 677: fl(fl(1 - 0.3) * 677) is not (7/10) * 677


def pd_threshold(which: str) -> float:
    n0, m0, len0 = PD_N0, PD_M0, PD_N0 * BLOCK_BYTES + PD_TAIL
    t0 = fmul(fsub(1.0, fdiv(float(m0), float(n0))), float(len0))
    return {"exact": t0, "exact_full": 0.0, "below": math.nextafter(t0, -math.inf),
            "above": math.nextafter(t0, math.inf), "+inf": math.inf, "-inf": -math.inf, "neg": -1.0}[which]


def case_pd(E, mode, seed, threshold="exact", R=256):
    """PD with the decode pick's match set so that (1 - hit) * len lands exactly on the threshold and next to it"""
    b = _Builder(E, mode, seed)
    rng = b.rng
    st = _states(E)
    dec = np.arange(E) % 2 == 1 if E > 1 else np.zeros(E, bool)
    st["role_mask"] = np.where(dec, abi.FI_ROLE_DECODER, abi.FI_ROLE_PREFILLER)
    st["kv_util"] = rng.choice(KV_EDGES, E)
    st["queue_depth"] = rng.choice(Q_EDGES, E)
    profiles = [{"name": "prefill", "role_mask": abi.FI_ROLE_PREFILLER, "scorers": [(P, 50), (K, 5)]},
                {"name": "decode", "role_mask": abi.FI_ROLE_DECODER, "scorers": [(P, 1000), (Q, 1)]}]
    decoders, prefillers = np.flatnonzero(dec), np.flatnonzero(~dec)
    for r in range(R):
        if r % 4 == 3 or not len(decoders):
            b.random_request(np.arange(E))
            continue
        # the class of (n0, len0): the one matched decoder is the decode pick (prefix weight 1000 beats queue 1)
        full = threshold == "exact_full" and r % 2
        m = PD_N0 if full else int(np.clip(PD_M0 + rng.integers(-1, 2), 0, PD_N0))
        mt = [(int(rng.choice(decoders)), m)] if m else []
        if len(prefillers):
            mt.append((int(rng.choice(prefillers)), int(rng.integers(1, PD_N0 + 1))))
        b.request(PD_N0, PD_TAIL, mt)
    return b.finish(f"pd_{threshold}", profiles, {"decode": 1, "prefill": 0, "threshold": pd_threshold(threshold)}, st)


def case_lora(E, mode, seed, R=256):
    """the score-everything kernel: LoRA affinity 1.0 / 0.8 / 0.6 / 0 under weights up to 2^31 - 1"""
    b = _Builder(E, mode, seed)
    rng = b.rng
    st = _states(E)
    st["kv_util"] = rng.choice(KV_EDGES, E)
    st["queue_depth"] = rng.choice(Q_EDGES, E)
    lo = np.zeros(E, dtype=LORA_DTYPE)
    lo["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 4)), int(rng.integers(0, 3))
        ids = rng.permutation(6)[: na + nw] + 1000
        lo[e]["n_active"], lo[e]["n_waiting"] = na, nw
        lo[e]["active"][:na] = ids[:na]
        lo[e]["waiting"][:nw] = ids[na:]
        lo[e]["max_active"] = int(rng.integers(0, 6))
    profiles = [{"name": "lora", "scorers": [(L, W_MAX), (P, 7), (K, W_MAX), (Q, 1)]},
                {"name": "mix", "scorers": [(P, 1), (L, 3), (L, 0)]}]
    for _ in range(R):
        b.random_request(np.arange(E))
    adapters = (rng.integers(0, 8, R) + 1000).astype(np.uint64)
    return b.finish("lora", profiles, None, st, lo, adapters)


def _order_pairs(max_blocks):
    """(n, mA, mB) with x = fl(mB/n), z = fl(mA/n) in [1/2, 1): fl(fl(x + 1) + z) != fl(fl(z + 1) + x) although the
    exact sums are equal"""
    out = []
    for n in range(2, max_blocks + 1):
        for ma in range((n + 1) // 2, n):
            for mb in range((n + 1) // 2, n):
                x, z = fdiv(float(mb), float(n)), fdiv(float(ma), float(n))
                if x != z and fadd(fadd(x, 1.0), z) != fadd(fadd(z, 1.0), x):
                    out.append((n, ma, mb))
    return out


def case_order(E, mode, seed, R=256):
    """pairs of endpoints A, B whose three score terms are (x, 1, z) and (z, 1, x): their exact totals tie, their
    fp64 totals do not, and which one wins depends on the profile order alone"""
    b = _Builder(E, mode, seed)
    rng = b.rng
    st = _states(E)
    st["kv_util"] = 1.0  # everyone else: kv score 0
    st["queue_depth"] = 7  # all equal: queue score 1.0
    pairs = _order_pairs(MAX_BLOCKS)
    npairs = min(E // 2, 16)
    chosen = [pairs[i] for i in rng.choice(len(pairs), npairs, replace=False)] if npairs else []
    for j, (n, ma, mb) in enumerate(chosen):
        a, bb = 2 * j, 2 * j + 1
        st["kv_util"][a] = fsub(1.0, fdiv(float(mb), float(n)))  # exact (Sterbenz): 1 - kv_A == fl(mB / n)
        st["kv_util"][bb] = fsub(1.0, fdiv(float(ma), float(n)))
    profiles = [{"name": "kqp", "scorers": [(K, 1), (Q, 1), (P, 1)]},
                {"name": "pqk", "scorers": [(P, 1), (Q, 1), (K, 1)]},
                {"name": "kqp_w", "scorers": [(K, 3), (Q, 5), (P, 3)]},
                {"name": "pqk_w", "scorers": [(P, 7), (Q, 1), (K, 7)]}]
    for r in range(R):
        if not npairs or r % 5 == 4:
            b.random_request(np.arange(E))
            continue
        j = r % npairs
        n, ma, mb = chosen[j]
        b.request(n, matches=[(2 * j, ma), (2 * j + 1, mb)])
    return b.finish("order", profiles, None, st)


KINDS = {"edges": case_edges, "zero_tie": case_zero_tie, "lora": case_lora, "order": case_order}


def make_case(kind: str, E: int, mode: int, seed: int, R: int = 256) -> Case:
    if kind.startswith("pd_"):
        return case_pd(E, mode, seed, threshold=kind[3:], R=R)
    return KINDS[kind](E, mode, seed, R=R)


ALL_KINDS = tuple(KINDS) + tuple("pd_" + t for t in PD_THRESHOLDS)


# ---- the exact reference of the picks ----------------------------------------------------------------------
class Spec:
    """S.3 match, S.4 totals (spec_total), S.5 / S.5a eligibility, S.6 / S.6a selection and S.7 of one case"""

    def __init__(self, case: Case, variant: Optional[str] = None):
        self.c, self.variant = case, variant
        E = case.E
        index = {}
        for h, e in zip(case.ops["hash"].tolist(), case.ops["endpoint"].tolist()):
            index.setdefault(h, set()).add(e)
        self.index = index
        st = case.states
        self.kv = [float(x) for x in st["kv_util"]]
        self.q = [int(x) for x in st["queue_depth"]]
        self.elig = []
        for pr in case.profiles:
            filt = pr.get("role_mask", 0)
            self.elig.append(np.array([(int(st["flags"][e]) & abi.FI_ENDPOINT_ALIVE) != 0
                                       and (not filt or (int(st["role_mask"][e]) & filt) != 0) for e in range(E)]))
        self.lora = [None] * E
        if case.lora is not None:
            for row in case.lora:
                self.lora[int(row["endpoint"])] = (int(row["max_active"]), [int(x) for x in row["active"][: int(row["n_active"])]],
                                                   [int(x) for x in row["waiting"][: int(row["n_waiting"])]])
        self.has_lora = any(k == L for pr in case.profiles for k, _ in pr["scorers"])
        self.requests = []
        raw = case.tok.tobytes()
        for r in range(case.R):
            p = raw[int(case.offs[r]):int(case.offs[r + 1])]
            ch = _chain(p, case.max_blocks, case.h0)
            n = len(ch)
            start = tie_start(n, int(ch[0]) if n else 0, case.h0, r, E)
            self.requests.append((n, len(p), self._match(ch), start))
        self._zero = {}

    def _match(self, ch):
        """S.3: {endpoint: match} over the blocks before the first one no endpoint holds"""
        counts, run = {}, None
        for h in ch.tolist():
            s = self.index.get(h)
            if not s:
                break
            if self.c.mode == abi.FI_MATCH_LPM:
                run = set(s) if run is None else (run & s)
                held = run
            else:
                held = s
            for e in held:
                counts[e] = counts.get(e, 0) + 1
        return counts

    def _total(self, pi, e, m, n, qmin, qmax, lora_v):
        sc = tuple(self.c.profiles[pi]["scorers"])
        return spec_total(sc, m, n, self.kv[e], self.q[e], qmin, qmax, lora_v, self.variant)

    def _lora_v(self, e, adapter):
        return lora_value(self.lora[e], adapter) if self.has_lora else 0.0

    def _totals(self, pi, members, qmin, qmax, matches, n, adapter):
        """fp64 totals of `members` (sorted endpoint array); zero-match totals of the pool-wide queue range cached"""
        out = np.empty(len(members), dtype=np.float64)
        key = (pi, qmin, qmax)
        for i, e in enumerate(members.tolist()):
            m = matches.get(e, 0)
            lv = self._lora_v(e, adapter)
            if m == 0:
                z = self._zero.get(key + (e, lv))
                if z is None:
                    z = self._zero[key + (e, lv)] = self._total(pi, e, 0, n, qmin, qmax, lv)
                out[i] = z
            else:
                out[i] = self._total(pi, e, m, n, qmin, qmax, lv)
        return out

    def _ranked_one(self, pi, r, k, sub_mask=None, adapter=0, single=False):
        E = self.c.E
        n, _, matches, start = self.requests[r]
        elig = self.elig[pi] if sub_mask is None else (self.elig[pi] & sub_mask)
        members = np.flatnonzero(elig)
        out = np.zeros(k, dtype=PICK_DTYPE)
        out["endpoint"], out["n_blocks"] = NO, n
        if not len(members):
            return out
        qs = [self.q[e] for e in members.tolist()]
        tot = self._totals(pi, members, min(qs), max(qs), matches, n, adapter)
        keys = (members - start) % E
        if single and self.variant == "zero_tie" and not self.has_lora:
            # the matched side wins a tie with the zero-match side, rotation only within each side
            matched = np.array([matches.get(e, 0) > 0 for e in members.tolist()])
            top = tot == tot.max()
            if (top & matched).any():
                keys = np.where(matched, keys, keys + E)
        order = np.lexsort((keys, -tot))[:k]
        for j, i in enumerate(order.tolist()):
            e = int(members[i])
            out[j] = (e, matches.get(e, 0), n, tot[i])
        return out

    def ranked(self, k: int, subsets: Optional[np.ndarray] = None, single: bool = False) -> np.ndarray:
        """[R, n_profiles, k] (S.6a; with subsets [R, ceil(E / 32)] uint32 rows, S.5a)"""
        c = self.c
        Pn = len(c.profiles)
        out = np.zeros((c.R, Pn, k), dtype=PICK_DTYPE)
        bits = None
        if subsets is not None:
            bits = np.unpackbits(np.ascontiguousarray(subsets, dtype="<u4").view(np.uint8), axis=1, bitorder="little")[:, : c.E]
        for r in range(c.R):
            ad = int(c.adapters[r]) if c.adapters is not None else 0
            sub = None if bits is None else bits[r].astype(bool)
            for pi in range(Pn):
                out[r, pi] = self._ranked_one(pi, r, k, sub, ad, single)
            if c.pd:
                n, length, _, _ = self.requests[r]
                d = out[r, c.pd["decode"], 0]
                if not pd_runs(int(d["endpoint"]), int(d["match_blocks"]), n, length, c.pd["threshold"], self.variant):
                    out[r, c.pd["prefill"]] = (NO, 0, n, 0.0)
        return out

    def picks(self) -> np.ndarray:
        """[R, n_profiles] (S.6, S.7)"""
        return np.ascontiguousarray(self.ranked(1, single=True)[:, :, 0])


    def total_of(self, pi: int, r: int, e: int) -> float:
        """endpoint e's fp64 total for request r in profile pi (queue range over the profile's whole eligible set)"""
        n, _, matches, _ = self.requests[r]
        qs = [self.q[x] for x in np.flatnonzero(self.elig[pi]).tolist()]
        ad = int(self.c.adapters[r]) if self.c.adapters is not None else 0
        return float(self._totals(pi, np.array([e]), min(qs), max(qs), matches, n, ad)[0])


def spec_picks(case: Case, variant: Optional[str] = None) -> np.ndarray:
    return Spec(case, variant).picks()


def subset_rows(case: Case, seed: int) -> np.ndarray:
    """per-request candidate subsets: random, singleton, empty and full rows, and rows with the INT32_MIN / INT32_MAX
    queue endpoints (0 and E - 1 in the edge cases) inside and outside"""
    rng = np.random.default_rng(seed)
    E, W = case.E, (case.E + 31) // 32
    out = np.zeros((case.R, W), dtype=np.uint32)
    for r in range(case.R):
        kind = r % 6
        if kind == 0:
            s = rng.choice(E, int(rng.integers(1, min(E, 48) + 1)), replace=False)
        elif kind == 1:
            s = [int(rng.integers(0, E))]
        elif kind == 2:
            s = []
        elif kind == 3:
            s = list(range(E))
        elif kind == 4:
            s = list({0, E - 1} | set(rng.choice(E, min(E, 8), replace=False).tolist()))
        else:
            s = [e for e in rng.choice(E, min(E, 16), replace=False).tolist() if e not in (0, E - 1)]
        for e in s:
            out[r, e >> 5] |= np.uint32(1 << (e & 31))
    return out


def differs(a: np.ndarray, b: np.ndarray):
    """(picks whose endpoint differs, picks whose endpoint, match, n or score bits differ)"""
    ep = a["endpoint"] != b["endpoint"]
    anyd = ep | (a["match_blocks"] != b["match_blocks"]) | (a["n_blocks"] != b["n_blocks"]) | (
        a["score"].view(np.uint64) != b["score"].view(np.uint64))
    return int(ep.sum()), int(anyd.sum())


def discriminating(candidates):
    """The seeded search: of the candidate cases keep those in which some variant changes the spec's picks, most
    changed endpoints first.  -> [(case, {variant: (endpoint differences, any differences)})]"""
    kept = []
    for c in candidates:
        want = spec_picks(c)
        d = {v: differs(spec_picks(c, v), want) for v in VARIANTS}
        if any(x[1] for x in d.values()):
            kept.append((c, d))
    kept.sort(key=lambda cd: -sum(x[0] for x in cd[1].values()))
    return kept


# The cases of the GPU suite (test_gpu_score_edges.py).  Pool sizes 3 .. 4096 give membership rows of 1, 2, 4, 32, 64
# and 128 words: every match_pick_kernel row shape.  The CPU suite checks that they discriminate every variant.
GPU_POOLS = (3, 40, 100, 1024, 2048, 4096)
GPU_R = 256
GPU_CASES = [(kind, E) for kind in ("edges", "zero_tie", "lora", "order") for E in GPU_POOLS] + [
    ("pd_" + t, E) for t in PD_THRESHOLDS for E in (3, 100, 2048)]


@functools.lru_cache(maxsize=None)
def gpu_case(kind: str, E: int) -> Case:
    mode = (GPU_POOLS.index(E) + ALL_KINDS.index(kind)) % 2  # both match modes for every kind across the pools
    return make_case(kind, E, mode, seed=7 * E + ALL_KINDS.index(kind), R=GPU_R)
