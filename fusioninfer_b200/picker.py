"""Host-side mirror of the Endpoint Picker scheduling interface over the C ABI.

`EndpointPicker` plays the role of the upstream EPP's scheduler object for the
ONE path this repo implements: it is configured from the EndpointPickerConfig
YAML that FusionInfer's router role generates
(/root/reference/pkg/router/strategy.go:27-165), receives pod-state refreshes
and prefix-index updates, and schedules batches of requests.  Every call goes
through include/fi_epp.h into the sm_90a kernels; nothing is computed in Python.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _abi as abi

PICK_DTYPE, OP_DTYPE, ENDPOINT_DTYPE = abi.np_dtypes()
LORA_DTYPE = abi.lora_dtype()


class FiEppError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        name = abi.load().fi_epp_status_string(status).decode()
        super().__init__(f"{where}: {name} ({status}){': ' + detail if detail else ''}")


def default_config() -> abi.fi_epp_config:
    cfg = abi.fi_epp_config()
    rc = abi.load().fi_epp_config_default(C.byref(cfg))
    if rc != abi.FI_OK:
        raise FiEppError(rc, "fi_epp_config_default")
    return cfg


def config_from_yaml(yaml_text: str, base: Optional[abi.fi_epp_config] = None) -> abi.fi_epp_config:
    """Apply an EndpointPickerConfig YAML (strategy.go:52-67,126-164) onto `base`."""
    cfg = base if base is not None else default_config()
    raw = yaml_text.encode()
    err = C.create_string_buffer(512)
    rc = abi.load().fi_epp_config_from_yaml(raw, len(raw), C.byref(cfg), err, len(err))
    if rc != abi.FI_OK:
        raise FiEppError(rc, "fi_epp_config_from_yaml", err.value.decode())
    return cfg


def config_picker_endpoints(yaml_text: str) -> list[int]:
    """maxNumOfEndpoints of the max-score-picker each profile of the document references, in profile order (1 when
    absent): how many ranked endpoints (pick_batch_ranked) each profile hands the proxy."""
    raw = yaml_text.encode()
    out = (C.c_uint32 * abi.FI_EPP_MAX_PROFILES)()
    err = C.create_string_buffer(512)
    rc = abi.load().fi_epp_config_picker_endpoints(raw, len(raw), out, err, len(err))
    if rc != abi.FI_OK:
        raise FiEppError(rc, "fi_epp_config_picker_endpoints", err.value.decode())
    return [int(v) for v in out if v]


def subset_bitsets(subsets: Sequence[Optional[Sequence[int]]], num_endpoints: int) -> np.ndarray:
    """Per-request candidate subsets -> the [R, ceil(num_endpoints / 32)] uint32 rows of pick_batch_subset.
    None means no hint (every bit set); an empty list is an all-zero row (no candidate: FI_NO_ENDPOINT).
    Endpoints outside [0, num_endpoints) are dropped, as the data plane's addresses outside the pool are."""
    words = (int(num_endpoints) + 31) // 32
    out = np.zeros((len(subsets), words), dtype=np.uint32)
    for r, s in enumerate(subsets):
        if s is None:
            out[r] = 0xFFFFFFFF
            continue
        e = np.asarray(s, dtype=np.int64).ravel()
        e = e[(e >= 0) & (e < num_endpoints)]
        np.bitwise_or.at(out[r], e >> 5, (np.uint32(1) << (e & 31).astype(np.uint32)))
    return out


def make_config(
    *,
    num_endpoints: int,
    block_bytes: int = 64,
    max_blocks: int = 256,
    lru_capacity: int = 0,
    max_batch: int = 1024,
    max_prompt_bytes: int = 0,
    index_slots: int = 0,
    match_mode: int = abi.FI_MATCH_UPSTREAM,
    device: int = 0,
    endpoint_begin: int = 0,
    endpoint_count: Optional[int] = None,
    profiles: Optional[Sequence[dict]] = None,
    pd: Optional[dict] = None,
    base: Optional[abi.fi_epp_config] = None,
) -> abi.fi_epp_config:
    """Build a config in code.  profiles: [{"name", "role_mask", "more_filters": [...], "scorers": [(kind, weight), ...]}].
    base: a pre-filled struct to start from instead of fi_epp_config_default() (then libfi_epp.so is not touched:
    bench.py's CPU reference arm builds its configuration without mapping the product library)."""
    cfg = base if base is not None else default_config()
    cfg.device = device
    cfg.block_bytes = block_bytes
    cfg.max_blocks = max_blocks
    cfg.lru_capacity = lru_capacity
    cfg.num_endpoints = num_endpoints
    cfg.endpoint_begin = endpoint_begin
    cfg.endpoint_count = num_endpoints - endpoint_begin if endpoint_count is None else endpoint_count
    cfg.match_mode = match_mode
    cfg.max_batch = max_batch
    cfg.max_prompt_bytes = max_prompt_bytes
    cfg.index_slots = index_slots
    if profiles is not None:
        cfg.n_profiles = len(profiles)
        for i, p in enumerate(profiles):
            prof = cfg.profiles[i]
            prof.name = p.get("name", f"p{i}").encode()
            prof.role_mask = p.get("role_mask", 0)
            more = list(p.get("more_filters", []))  # further by-label filters, ANDed with role_mask
            prof.n_more_filters = len(more)
            for j, f in enumerate(more):
                prof.more_filters[j] = f
            sc = p["scorers"]
            prof.n_scorers = len(sc)
            for j, (kind, weight) in enumerate(sc):
                prof.scorers[j].kind = kind
                prof.scorers[j].weight = weight
    if pd is not None:
        cfg.pd_enabled = 1
        cfg.pd_decode_profile = pd["decode"]
        cfg.pd_prefill_profile = pd["prefill"]
        cfg.pd_threshold = float(pd.get("threshold", 0.0))
    return cfg


def model_seed(model: bytes, salt: bytes = b"") -> int:
    out = C.c_uint64(0)
    rc = abi.load().fi_epp_model_seed(model, len(model), salt, len(salt), C.byref(out))
    if rc != abi.FI_OK:
        raise FiEppError(rc, "fi_epp_model_seed")
    return out.value


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def snapshot_info(buf) -> abi.fi_epp_snapshot_info:
    """Check a snapshot blob's structure (everything but key distinctness) and return its header; no handle, no GPU.
    ValueError if the blob is not well-formed."""
    buf = np.ascontiguousarray(np.frombuffer(buf, dtype=np.uint8) if isinstance(buf, (bytes, bytearray)) else buf,
                               dtype=np.uint8)
    out = abi.fi_epp_snapshot_info()
    rc = abi.load().fi_epp_snapshot_info(_ptr(buf), len(buf), C.byref(out))
    if rc != abi.FI_OK:
        raise ValueError("not a well-formed snapshot")
    return out


class SnapshotCapture:
    """A snapshot taken on the device by EndpointPicker.capture_snapshot() (docs/SPEC.md S.2d).  read() gives the
    bytes save_snapshot() would have returned at the capture's point; it never touches the picker, so it may run on
    another thread, and after the picker is resized, loaded or closed.  close() frees the device image."""

    def __init__(self, lib, c: C.c_void_p, nbytes: int):
        self._lib = lib
        self._c = c
        self.nbytes = nbytes

    def read(self) -> np.ndarray:
        """The snapshot blob; blocks until the device image is complete.  Repeatable: the same bytes every time."""
        if not self._c:
            raise ValueError("snapshot capture is closed")
        buf = np.empty(self.nbytes, dtype=np.uint8)
        rc = self._lib.fi_epp_snapshot_read(self._c, _ptr(buf), len(buf))
        if rc != abi.FI_OK:
            raise FiEppError(rc, "fi_epp_snapshot_read")
        return buf

    def close(self):
        if getattr(self, "_c", None):
            self._lib.fi_epp_snapshot_free(self._c)
            self._c = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class EndpointPicker:
    """One handle = one GPU = one endpoint-range shard of the pool."""

    def __init__(self, cfg: abi.fi_epp_config):
        self._lib = abi.load()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self._lib.fi_epp_create(C.byref(cfg), C.byref(h))
        if rc != abi.FI_OK:
            raise FiEppError(rc, "fi_epp_create", "see stderr")
        self._h = h
        self.n_profiles = cfg.n_profiles
        self.max_blocks = cfg.max_blocks

    # -- lifecycle ---------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.fi_epp_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, where: str):
        if rc != abi.FI_OK:
            raise FiEppError(rc, where, self._lib.fi_epp_last_error(self._h).decode())

    # -- pod datastore -------------------------------------------------------
    def update_endpoints(self, states: np.ndarray):
        states = np.ascontiguousarray(states, dtype=ENDPOINT_DTYPE)
        self._check(self._lib.fi_epp_endpoints_update(self._h, _ptr(states), len(states)), "fi_epp_endpoints_update")

    def update_endpoints_lora(self, states: np.ndarray):
        """Adapter residency per endpoint (LORA_DTYPE rows) for the lora-affinity-scorer."""
        states = np.ascontiguousarray(states, dtype=LORA_DTYPE)
        self._check(self._lib.fi_epp_endpoints_lora_update(self._h, _ptr(states), len(states)),
                    "fi_epp_endpoints_lora_update")

    # -- prefix index --------------------------------------------------------
    def index_apply(self, ops: np.ndarray):
        ops = np.ascontiguousarray(ops, dtype=OP_DTYPE)
        self._check(self._lib.fi_epp_index_apply(self._h, _ptr(ops), len(ops)), "fi_epp_index_apply")

    def remove_endpoints(self, endpoints, count: bool = False) -> Optional[int]:
        """upstream indexer.RemovePod: drop every cached prefix of the listed endpoints from the index and empty their
        LRUs (pod gone, restarted, or its index about to be given to a new pod).  Ordered like index_apply.
        count=True blocks until the removal is applied and returns how many (endpoint, hash) pairs it removed."""
        eps = np.ascontiguousarray(np.atleast_1d(np.asarray(endpoints, dtype=np.uint32)))
        out = C.c_uint64(0)
        self._check(self._lib.fi_epp_index_remove_endpoints(self._h, _ptr(eps), len(eps), C.byref(out) if count else None),
                    "fi_epp_index_remove_endpoints")
        return out.value if count else None

    def resize_pool(self, num_endpoints: int, count: bool = False) -> Optional[int]:
        """Grow or shrink the pool to num_endpoints endpoints, keeping the prefixes the kept endpoints [0, min(old,
        new)) have cached: a shrink drops the tail endpoints as remove_endpoints would, a grow appends endpoints that
        are not alive and hold nothing yet.  Blocks until every earlier call is done against the old pool.
        count=True returns how many (endpoint, hash) pairs a shrink removed."""
        out = C.c_uint64(0)
        self._check(self._lib.fi_epp_resize_pool(self._h, int(num_endpoints), C.byref(out) if count else None),
                    "fi_epp_resize_pool")
        # a copy: the caller's config (which created the handle) stays as it was
        self.cfg = abi.fi_epp_config.from_buffer_copy(self.cfg)
        self.cfg.num_endpoints = self.cfg.endpoint_count = int(num_endpoints)
        return out.value if count else None

    def save_snapshot(self) -> np.ndarray:
        """The handle's learned state (docs/SPEC.md S.2d: the index's pairs, every endpoint's LRU and its capacity) as
        a snapshot blob.  Blocks until every earlier call is applied; the handle is not changed."""
        n = C.c_uint64(0)
        self._check(self._lib.fi_epp_snapshot_save(self._h, None, 0, C.byref(n)), "fi_epp_snapshot_save")
        buf = np.empty(n.value, dtype=np.uint8)
        self._check(self._lib.fi_epp_snapshot_save(self._h, _ptr(buf), len(buf), C.byref(n)), "fi_epp_snapshot_save")
        return buf

    def capture_snapshot(self) -> SnapshotCapture:
        """Take a snapshot on the device at this point of the call order, without waiting for picks in flight; copy
        it out with .read() (any thread, the picker not needed) and free it with .close().  The device image (the
        blob's size) is held until then; FiEppError(FI_ERR_NOMEM) when it does not fit, where save_snapshot() still
        works."""
        c = C.c_void_p()
        n = C.c_uint64(0)
        self._check(self._lib.fi_epp_snapshot_capture(self._h, C.byref(c), C.byref(n)), "fi_epp_snapshot_capture")
        return SnapshotCapture(self._lib, c, n.value)

    def load_snapshot(self, buf) -> None:
        """Replace the index, the LRUs and their capacities with a snapshot's: afterwards the handle behaves like the
        one that saved it, except for its own endpoint states and adapters (re-send them).  Blocks like resize_pool;
        a failing load changes nothing."""
        buf = np.ascontiguousarray(np.frombuffer(buf, dtype=np.uint8) if isinstance(buf, (bytes, bytearray)) else buf,
                                   dtype=np.uint8)
        self._check(self._lib.fi_epp_snapshot_load(self._h, _ptr(buf), len(buf)), "fi_epp_snapshot_load")

    def set_lru_capacities(self, endpoints, capacities, want_evicted: bool = False) -> Optional[int]:
        """Per-endpoint LRU capacities (upstream autoTune: a pod's LRU sized from its KV-cache block count).
        capacities[i] is endpoints[i]'s new capacity, 0 meaning lru_capacity; an LRU above its new capacity evicts its
        least recently used keys (and their index pairs) down to it.  Ordered like index_apply.  want_evicted=True
        blocks until the evictions are applied and returns how many LRU entries were evicted."""
        eps = np.ascontiguousarray(np.atleast_1d(np.asarray(endpoints, dtype=np.uint32)))
        caps = np.ascontiguousarray(np.atleast_1d(np.asarray(capacities, dtype=np.uint32)))
        if len(caps) != len(eps):
            raise ValueError("endpoints and capacities differ in length")
        out = C.c_uint64(0)
        self._check(self._lib.fi_epp_set_lru_capacities(self._h, _ptr(eps), _ptr(caps), len(eps),
                                                        C.byref(out) if want_evicted else None),
                    "fi_epp_set_lru_capacities")
        return out.value if want_evicted else None

    def index_add_chain(self, endpoint: int, hashes: np.ndarray):
        hashes = np.ascontiguousarray(hashes, dtype=np.uint64)
        self._check(
            self._lib.fi_epp_index_add_chain(self._h, endpoint, _ptr(hashes), len(hashes)), "fi_epp_index_add_chain"
        )

    def index_add_chains(self, endpoints: np.ndarray, chains: np.ndarray, nblocks: np.ndarray):
        """indexer.Add(chains[r, :nblocks[r]], endpoints[r]) for a whole batch of decisions (upstream PreRequest);
        chains: [R, pitch] u64 as returned by pick_batch(want_chains=True).  Collective on a sharded pool."""
        endpoints = np.ascontiguousarray(endpoints, dtype=np.uint32)
        nblocks = np.ascontiguousarray(nblocks, dtype=np.uint32)
        chains = np.ascontiguousarray(chains, dtype=np.uint64)
        R = len(endpoints)
        pitch = chains.shape[1] if chains.ndim == 2 else (chains.size // max(R, 1))
        self._check(self._lib.fi_epp_index_add_chains(self._h, _ptr(endpoints), _ptr(chains), pitch, _ptr(nblocks), R),
                    "fi_epp_index_add_chains")

    def index_add_chains_device(self, endpoints: np.ndarray, d_chains: int, pitch: int, nblocks: np.ndarray, stream: int = 0):
        """The same with the chains in device memory (pointer; e.g. the chains_out of pick_batch_device, written on
        `stream`): only the two small host arrays cross PCIe.  Needs the device-resident LRU (the default)."""
        endpoints = np.ascontiguousarray(endpoints, dtype=np.uint32)
        nblocks = np.ascontiguousarray(nblocks, dtype=np.uint32)
        self._check(self._lib.fi_epp_index_add_chains_device(self._h, _ptr(endpoints), C.c_void_p(d_chains), pitch, _ptr(nblocks),
                                                             len(endpoints), C.c_void_p(stream)),
                    "fi_epp_index_add_chains_device")

    def lru_dump(self, endpoint: int) -> np.ndarray:
        """Keys of `endpoint` in the device-resident LRU, least recently used first (diagnostics)."""
        cap = max(int(self.cfg.lru_capacity), 1) + 1
        out = np.zeros(cap, dtype=np.uint64)
        n = C.c_uint32(0)
        self._check(self._lib.fi_epp_lru_dump(self._h, endpoint, _ptr(out), cap, C.byref(n)), "fi_epp_lru_dump")
        return out[: n.value].copy()

    def pipeline_info(self) -> dict:
        """How pick_submit runs.  It always runs on the whole GPU with two batches in flight, so this returns
        partitioned False and 0 for walk_sms and main_sms."""
        out = (C.c_int32 * 3)()
        self._check(self._lib.fi_epp_pipeline_info(self._h, out), "fi_epp_pipeline_info")
        return {"partitioned": bool(out[0]), "walk_sms": int(out[1]), "main_sms": int(out[2])}

    def lru_counters(self) -> dict:
        """Totals of the device-resident LRU since create (diagnostics)."""
        out = (C.c_uint64 * 6)()
        self._check(self._lib.fi_epp_lru_counters(self._h, out), "fi_epp_lru_counters")
        return dict(zip(("sets", "clears", "doomed", "maintained", "deferred_requests", "sub_batches"), [int(x) for x in out]))

    def index_sync(self):
        self._check(self._lib.fi_epp_index_sync(self._h), "fi_epp_index_sync")

    def index_contains(self, queries: np.ndarray) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=OP_DTYPE)
        out = np.zeros(len(q), dtype=np.uint8)
        self._check(self._lib.fi_epp_index_contains(self._h, _ptr(q), len(q), _ptr(out)), "fi_epp_index_contains")
        return out

    def index_stats(self) -> abi.fi_index_stats:
        st = abi.fi_index_stats()
        self._check(self._lib.fi_epp_index_stats(self._h, C.byref(st)), "fi_epp_index_stats")
        return st

    # -- hashing / scheduling --------------------------------------------------
    @staticmethod
    def _inputs(prompts, offsets, h0):
        prompts = np.ascontiguousarray(np.frombuffer(prompts, dtype=np.uint8) if isinstance(prompts, (bytes, bytearray)) else prompts)
        if prompts.dtype != np.uint8:
            prompts = prompts.view(np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        R = len(offsets) - 1
        h0 = np.ascontiguousarray(np.broadcast_to(np.asarray(h0, dtype=np.uint64), (R,)))
        return prompts, offsets, h0, R

    def hash_batch(self, prompts, offsets, h0):
        """-> (chains [R, max_blocks] u64, nblocks [R] u32)"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64)
        nb = np.zeros(R, dtype=np.uint32)
        self._check(
            self._lib.fi_epp_hash_batch(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(chains), _ptr(nb)),
            "fi_epp_hash_batch",
        )
        return chains, nb

    def pick_batch(self, prompts, offsets, h0, want_chains: bool = False, adapters=None):
        """Schedule R requests held in host memory.  -> picks [R, n_profiles] (PICK_DTYPE)[, chains]
        adapters: optional [R] uint64 target adapter ids (lora-affinity-scorer)."""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        picks = np.zeros((R, self.n_profiles), dtype=PICK_DTYPE)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64) if want_chains else None
        if adapters is None:
            rc = self._lib.fi_epp_pick_batch(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(picks), _ptr(chains))
        else:
            ad = np.ascontiguousarray(np.broadcast_to(np.asarray(adapters, dtype=np.uint64), (R,)))
            rc = self._lib.fi_epp_pick_batch_lora(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), _ptr(ad), R,
                                                  _ptr(picks), _ptr(chains))
        self._check(rc, "fi_epp_pick_batch")
        return (picks, chains) if want_chains else picks

    def pick_batch_ranked(self, prompts, offsets, h0, k: int, want_chains: bool = False, adapters=None):
        """The best k endpoints of every profile, best first (docs/SPEC.md S.6a).  -> picks [R, n_profiles, k]
        (PICK_DTYPE)[, chains]; entry 0 is pick_batch's pick, a short list ends in FI_NO_ENDPOINT entries."""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        picks = np.zeros((R, self.n_profiles, max(int(k), 1)), dtype=PICK_DTYPE)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64) if want_chains else None
        ad = None if adapters is None else np.ascontiguousarray(np.broadcast_to(np.asarray(adapters, dtype=np.uint64), (R,)))
        rc = self._lib.fi_epp_pick_batch_ranked(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), _ptr(ad), R, int(k),
                                                _ptr(picks), _ptr(chains))
        self._check(rc, "fi_epp_pick_batch_ranked")
        return (picks, chains) if want_chains else picks

    def pick_batch_subset(self, prompts, offsets, h0, subsets, k: int = 1, adapters=None, want_chains: bool = False):
        """The ranked pick restricted to each request's candidate subset (docs/SPEC.md S.5a).  subsets: the
        [R, ceil(E / 32)] uint32 bitsets of subset_bitsets, or None (unrestricted: the same bytes as
        pick_batch_ranked).  -> picks [R, n_profiles, k] (PICK_DTYPE)[, chains]"""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        picks = np.zeros((R, self.n_profiles, max(int(k), 1)), dtype=PICK_DTYPE)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64) if want_chains else None
        ad = None if adapters is None else np.ascontiguousarray(np.broadcast_to(np.asarray(adapters, dtype=np.uint64), (R,)))
        sub = None
        if subsets is not None:
            sub = np.ascontiguousarray(subsets, dtype=np.uint32)
            if sub.shape != (R, (int(self.cfg.num_endpoints) + 31) // 32):
                raise ValueError(f"subsets must be [R, ceil(E / 32)] uint32 words, got {sub.shape}")
        rc = self._lib.fi_epp_pick_batch_subset(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), _ptr(ad), _ptr(sub), R,
                                                int(k), _ptr(picks), _ptr(chains))
        self._check(rc, "fi_epp_pick_batch_subset")
        return (picks, chains) if want_chains else picks

    def match_counts(self, prompts, offsets, h0, want_chains: bool = False):
        """The prefix-cache-scorer alone (docs/SPEC.md S.3a): every local endpoint's prefix match count, for a host
        framework that runs the configuration's other plugins itself.  -> (counts uint16 [R, endpoint_count],
        nblocks uint32 [R][, chains]); counts[r, j] / nblocks[r] is upstream's prefix score of endpoint
        endpoint_begin + j.  After the host's pick, index_add_chains_device(endpoints, 0, 0, nblocks) adds the chains."""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        counts = np.zeros((R, int(self.cfg.endpoint_count)), dtype=np.uint16)
        nb = np.zeros(R, dtype=np.uint32)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64) if want_chains else None
        self._check(self._lib.fi_epp_match_counts(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(counts),
                                                  _ptr(nb), _ptr(chains)),
                    "fi_epp_match_counts")
        return (counts, nb, chains) if want_chains else (counts, nb)

    def match_counts_device(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, d_counts: int,
                            d_nblocks: int = 0, d_chains: int = 0, stream: int = 0):
        """match_counts on device buffers: d_counts holds R * endpoint_count uint16 (2-byte aligned), d_nblocks R uint32
        (optional), d_chains R * max_blocks hashes (optional)."""
        self._check(
            self._lib.fi_epp_match_counts_device(self._h, d_prompts, d_offsets, d_h0, R, total_bytes, d_counts,
                                                 d_nblocks or None, d_chains or None, stream or None),
            "fi_epp_match_counts_device",
        )

    def match_lists(self, prompts, offsets, h0, cap=None, want_chains: bool = False):
        """match_counts as sparse per-request lists (docs/SPEC.md S.3b): only the endpoints that match.
        -> (list_offsets uint64 [R + 1], entries [list_offsets[R]] (match_entry_dtype: global endpoint, match_blocks),
        nblocks uint32 [R][, chains]); request r's entries are entries[list_offsets[r]:list_offsets[r + 1]], in
        ascending endpoint order.  cap (entries): None allows every list (R * endpoint_count); a smaller cap that falls
        short raises FiEppError with status FI_ERR_CAPACITY."""
        prompts, offsets, h0, R = self._inputs(prompts, offsets, h0)
        if cap is None:
            cap = R * int(self.cfg.endpoint_count)
        loff = np.zeros(R + 1, dtype=np.uint64)
        entries = np.zeros(int(cap), dtype=abi.match_entry_dtype())
        nb = np.zeros(R, dtype=np.uint32)
        chains = np.zeros((R, self.max_blocks), dtype=np.uint64) if want_chains else None
        self._check(self._lib.fi_epp_match_lists(self._h, _ptr(prompts), _ptr(offsets), _ptr(h0), R, _ptr(loff),
                                                 _ptr(entries) if cap else None, int(cap), _ptr(nb), _ptr(chains)),
                    "fi_epp_match_lists")
        out = (loff, entries[: int(loff[R])].copy(), nb)
        return out + (chains,) if want_chains else out

    def match_lists_device(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int,
                           d_list_offsets: int, d_entries: int, cap: int, d_nblocks: int = 0, d_chains: int = 0,
                           stream: int = 0):
        """match_lists on device buffers: d_list_offsets holds R + 1 uint64, d_entries cap fi_match_entry (4-byte
        aligned), d_nblocks R uint32 (optional), d_chains R * max_blocks hashes (optional).  A cap that falls short is
        not an error here: compare list_offsets[R] with cap once the stream has run."""
        self._check(
            self._lib.fi_epp_match_lists_device(self._h, d_prompts, d_offsets, d_h0, R, total_bytes, d_list_offsets,
                                                d_entries or None, int(cap), d_nblocks or None, d_chains or None,
                                                stream or None),
            "fi_epp_match_lists_device",
        )

    def pick_batch_raw(self, prompts_ptr: int, offsets_ptr: int, h0_ptr: int, R: int, out_ptr: int, chains_ptr: int = 0):
        """Host-pointer variant without numpy marshalling (pinned buffers from pinned_alloc)."""
        self._check(
            self._lib.fi_epp_pick_batch(self._h, prompts_ptr, offsets_ptr, h0_ptr, R, out_ptr, chains_ptr or None),
            "fi_epp_pick_batch",
        )

    def pick_batch_device(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, d_out: int,
                          d_chains: int = 0, stream: int = 0):
        """Every buffer already resident in this handle's device memory (raw device pointers)."""
        self._check(
            self._lib.fi_epp_pick_batch_device(
                self._h, d_prompts, d_offsets, d_h0, R, total_bytes, d_out, d_chains or None, stream or None
            ),
            "fi_epp_pick_batch_device",
        )

    def pick_batch_device_ranked(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, k: int,
                                 d_out: int, d_chains: int = 0, stream: int = 0, d_adapters: int = 0):
        """pick_batch_ranked on device buffers: d_out holds R * n_profiles * k picks."""
        self._check(
            self._lib.fi_epp_pick_batch_device_ranked(
                self._h, d_prompts, d_offsets, d_h0, d_adapters or None, R, total_bytes, int(k), d_out, d_chains or None,
                stream or None
            ),
            "fi_epp_pick_batch_device_ranked",
        )

    def pick_batch_device_subset(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, k: int,
                                 d_out: int, d_subsets: int = 0, d_chains: int = 0, stream: int = 0, d_adapters: int = 0):
        """pick_batch_subset on device buffers: d_subsets holds R rows of ceil(E / 32) uint32 words (0: unrestricted),
        d_out R * n_profiles * k picks."""
        self._check(
            self._lib.fi_epp_pick_batch_device_subset(
                self._h, d_prompts, d_offsets, d_h0, d_adapters or None, d_subsets or None, R, total_bytes, int(k), d_out,
                d_chains or None, stream or None
            ),
            "fi_epp_pick_batch_device_subset",
        )

    def pick_submit(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, d_out: int, stream: int = 0):
        """Pipelined device path: enqueue a batch; its result is valid for `stream` only after pick_wait."""
        self._check(
            self._lib.fi_epp_pick_submit(self._h, d_prompts, d_offsets, d_h0, R, total_bytes, d_out, stream or None),
            "fi_epp_pick_submit",
        )

    def pick_wait(self, stream: int = 0):
        """Make `stream` wait (device-side) for every batch submitted so far."""
        self._check(self._lib.fi_epp_pick_wait(self._h, stream or None), "fi_epp_pick_wait")

    def pick_submit_ex(self, d_prompts: int, d_offsets: int, d_h0: int, R: int, total_bytes: int, d_out: int, k: int = 0,
                       d_adapters: int = 0, d_subsets: int = 0, d_chains: int = 0, stream: int = 0) -> int:
        """Pipelined submit of any pick variant (docs/SPEC.md S.9): k = 0 the single pick ([R, n_profiles] picks, like
        pick_batch_device with adapters), k >= 1 the ranked / subset pick ([R, n_profiles, k]).  d_chains (optional):
        R * max_blocks hashes.  -> the batch's ticket, for pick_wait_batch and index_add_submitted."""
        t = C.c_uint64(0)
        self._check(
            self._lib.fi_epp_pick_submit_ex(self._h, d_prompts, d_offsets, d_h0, d_adapters or None, d_subsets or None, R,
                                            total_bytes, int(k), d_out, d_chains or None, stream or None, C.byref(t)),
            "fi_epp_pick_submit_ex",
        )
        return t.value

    def pick_wait_batch(self, ticket: int, stream: int = 0):
        """Make `stream` wait (device-side) for batch `ticket` and the ones before it, not for later ones."""
        self._check(self._lib.fi_epp_pick_wait_batch(self._h, int(ticket), stream or None), "fi_epp_pick_wait_batch")

    def index_add_submitted(self, ticket: int, endpoints: np.ndarray, nblocks: np.ndarray):
        """upstream PreRequest for a submitted batch: indexer.Add of its chains (kept by the handle) to the picked
        endpoints, without the overflow readback of index_add_chains_device; it waits on the host for the previous
        update's index counters only when the index is too close to its rebuild threshold to let them lag (docs/SPEC.md
        S.9, DESIGN.md §4.0).  Ordered like index_apply."""
        endpoints = np.ascontiguousarray(endpoints, dtype=np.uint32)
        nblocks = np.ascontiguousarray(nblocks, dtype=np.uint32)
        self._check(self._lib.fi_epp_index_add_submitted(self._h, int(ticket), _ptr(endpoints), _ptr(nblocks), len(endpoints)),
                    "fi_epp_index_add_submitted")

    # -- multi-GPU -------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * abi.FI_EPP_UNIQUE_ID_BYTES)()
        rc = abi.load().fi_epp_comm_unique_id(buf)
        if rc != abi.FI_OK:
            raise FiEppError(rc, "fi_epp_comm_unique_id")
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        buf = (C.c_uint8 * abi.FI_EPP_UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        self._check(self._lib.fi_epp_comm_init(self._h, buf, rank, world), "fi_epp_comm_init")

    def comm_exchange(self) -> str:
        """'none' (one rank), 'peer' (in-kernel stores over NVLink peer memory) or 'nccl' (all-gathers)."""
        rc = self._lib.fi_epp_comm_exchange(self._h)
        if rc < 0:
            raise FiEppError(rc, "fi_epp_comm_exchange")
        return {0: "none", 1: "peer", 2: "nccl"}[rc]

    def set_option(self, name: str, value: int):
        """Runtime knobs of include/fi_epp.h (fi_epp_set_option): exchange, shard_hash, feed_slices, lru_threads."""
        self._check(self._lib.fi_epp_set_option(self._h, name.encode(), int(value)), f"fi_epp_set_option({name})")

    # -- stats -----------------------------------------------------------------
    def set_profiling(self, on: bool):
        self._check(self._lib.fi_epp_set_profiling(self._h, 1 if on else 0), "fi_epp_set_profiling")

    def stats(self) -> abi.fi_epp_stats:
        st = abi.fi_epp_stats()
        self._check(self._lib.fi_epp_get_stats(self._h, C.byref(st)), "fi_epp_get_stats")
        return st

    def reset_stats(self):
        self._check(self._lib.fi_epp_reset_stats(self._h), "fi_epp_reset_stats")


class PinnedBuffer:
    """Page-locked host memory from the library (so H2D copies are truly asynchronous)."""

    def __init__(self, nbytes: int):
        self._lib = abi.load()
        self.nbytes = nbytes
        self.ptr = self._lib.fi_epp_pinned_alloc(nbytes)
        if not self.ptr:
            raise MemoryError(f"fi_epp_pinned_alloc({nbytes}) failed")

    def array(self, dtype, count: Optional[int] = None) -> np.ndarray:
        dt = np.dtype(dtype)
        n = self.nbytes // dt.itemsize if count is None else count
        buf = (C.c_uint8 * (n * dt.itemsize)).from_address(self.ptr)
        return np.frombuffer(buf, dtype=dt, count=n)

    def free(self):
        if self.ptr:
            self._lib.fi_epp_pinned_free(self.ptr)
            self.ptr = None
