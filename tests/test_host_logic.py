"""CPU: the product's host-side logic and the arithmetic its kernels share with the host.

libfi_hostcheck.so is a host build of fusioninfer_b200/csrc/{xxh64.cuh,bitslice.cuh,lru.h}
— the same headers the sm_90a kernels compile — so the split pre-state/chain-step
hashing, the bit-plane counters and the LRU are checked here without a GPU.
"""
import ctypes as C
import os
import random

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import config_from_yaml, default_config, model_seed
from fusioninfer_b200.picker import FiEppError
from oracle import epp_oracle as eo
from tests import helpers as H

LIB = os.path.join(abi.LIB_DIR, "libfi_hostcheck.so")


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(LIB)
    lib.fihc_xxh64.restype = C.c_uint64
    lib.fihc_xxh64.argtypes = [C.c_char_p, C.c_uint32]
    for f in (lib.fihc_chain_generic, lib.fihc_chain_split):
        f.restype = C.c_uint32
        f.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.fihc_bitcount.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.fihc_bitcount_merge.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.fihc_lru_new.restype = C.c_void_p
    lib.fihc_lru_new.argtypes = [C.c_uint32]
    lib.fihc_lru_free.argtypes = [C.c_void_p]
    lib.fihc_lru_size.restype = C.c_uint32
    lib.fihc_lru_size.argtypes = [C.c_void_p]
    lib.fihc_lru_contains.argtypes = [C.c_void_p, C.c_uint64]
    lib.fihc_lru_touch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fihc_lru_batch_check.restype = C.c_int
    lib.fihc_lru_batch_check.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                         C.c_uint32, C.c_uint32, C.c_void_p]
    lib.fihc_lru_plan_check.restype = C.c_int
    lib.fihc_lru_plan_check.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                        C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.fihc_tie_start.restype = C.c_uint32
    lib.fihc_tie_start.argtypes = [C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
    lib.fihc_tie_rot.restype = C.c_uint32
    lib.fihc_tie_rot.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    lib.fihc_tie_first_local.restype = C.c_uint32
    lib.fihc_tie_first_local.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    return lib


def test_kernel_header_xxh64_matches_golden(hc):
    g = H.golden()
    for case in g["xxh64"]:
        data = bytes.fromhex(case["hex"])
        assert f"{hc.fihc_xxh64(data, len(data)):016x}" == case["digest"]
    assert model_seed(g["h0_model"].encode()) == int(g["h0"], 16)
    assert model_seed(b"synthetic/", b"model") == int(g["h0"], 16)  # h0 = XXH64(model ‖ salt)


def test_kernel_header_chains_match_golden(hc):
    g = H.golden()
    h0 = int(g["h0"], 16)
    for case in g["chains"]:
        data = bytes.fromhex(case["hex"])
        B, M = case["block_bytes"], case["max_blocks"]
        want = [int(x, 16) for x in case["chain"]]
        out = np.zeros(M, dtype=np.uint64)
        n = hc.fihc_chain_generic(data, len(data), h0, B, M, out.ctypes.data)
        assert n == len(want) and list(out[:n]) == want
        if B % 32 == 0:  # the GPU fast path: stripes + merge hoisted out of the serial chain
            out2 = np.zeros(M, dtype=np.uint64)
            n2 = hc.fihc_chain_split(data, len(data), h0, B, M, out2.ctypes.data)
            assert n2 == len(want) and list(out2[:n2]) == want


@pytest.mark.parametrize("K", [1, 2, 4, 8, 16])
def test_bitplane_counter_counts_exactly(hc, K):
    rng = np.random.default_rng(K)
    for n in (0, 1, 5, 16, 33, 256, 1023):
        words = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
        if n:
            words[rng.integers(0, n, size=n // 3)] = 0xFFFFFFFF  # push some counters towards the maximum
        counts = np.zeros(32, dtype=np.uint32)
        hc.fihc_bitcount(words.ctypes.data, n, K, counts.ctypes.data)
        want = [int(((words >> b) & 1).sum()) for b in range(32)]
        assert list(counts) == want


def test_bitplane_counter_merge(hc):
    rng = np.random.default_rng(3)
    a = rng.integers(0, 2**32, size=300, dtype=np.uint64).astype(np.uint32)
    b = rng.integers(0, 2**32, size=500, dtype=np.uint64).astype(np.uint32)
    counts = np.zeros(32, dtype=np.uint32)
    nz = C.c_uint32(0)
    hc.fihc_bitcount_merge(a.ctypes.data, len(a), b.ctypes.data, len(b), counts.ctypes.data, C.byref(nz))
    want = [int(((a >> i) & 1).sum() + ((b >> i) & 1).sum()) for i in range(32)]
    assert list(counts) == want
    assert nz.value == sum((1 << i) for i in range(32) if want[i])


def _py_lru_trace(cap, keys):
    from collections import OrderedDict

    od = OrderedDict()
    out = []
    for k in keys:
        if k in od:
            od.move_to_end(k)
            out.append((0, 0, 0))
            continue
        ev = (0, 0)
        if len(od) == cap:
            old, _ = od.popitem(last=False)
            ev = (1, old)
        od[k] = None
        out.append((1, ev[0], ev[1]))
    return out, list(od.keys())


@pytest.mark.parametrize("cap", [1, 2, 7, 64, 1000])
def test_host_lru_matches_model(hc, cap):
    rng = random.Random(cap)
    keys = [rng.randrange(1, cap * 3 + 2) for _ in range(cap * 20 + 50)]
    want, final = _py_lru_trace(cap, keys)
    l = hc.fihc_lru_new(cap)
    ka = np.array(keys, dtype=np.uint64)
    ins = np.zeros(len(keys), dtype=np.uint8)
    did = np.zeros(len(keys), dtype=np.uint8)
    ev = np.zeros(len(keys), dtype=np.uint64)
    hc.fihc_lru_touch(l, ka.ctypes.data, len(keys), ins.ctypes.data, did.ctypes.data, ev.ctypes.data)
    got = [(int(i), int(d), int(e) if d else 0) for i, d, e in zip(ins, did, ev)]
    assert got == want
    assert hc.fihc_lru_size(l) == len(final)
    for k in set(keys):
        assert bool(hc.fihc_lru_contains(l, k)) == (k in final)
    hc.fihc_lru_free(l)


def test_host_lru_agrees_with_oracle_lru(hc):
    cap = 16
    cfg = H.make_config(num_endpoints=1, max_batch=1, lru_capacity=cap)
    o = eo.Oracle(cfg)
    l = hc.fihc_lru_new(cap)
    rng = random.Random(5)
    live = set()
    for _ in range(60):
        chain = np.array([rng.randrange(1, 60) for _ in range(rng.randrange(1, 9))], dtype=np.uint64)
        o.index_add_chain(0, chain)
        ins = np.zeros(len(chain), dtype=np.uint8)
        did = np.zeros(len(chain), dtype=np.uint8)
        ev = np.zeros(len(chain), dtype=np.uint64)
        hc.fihc_lru_touch(l, chain.ctypes.data, len(chain), ins.ctypes.data, did.ctypes.data, ev.ctypes.data)
        for k, i, d, e in zip(chain, ins, did, ev):
            if d:
                live.discard(int(e))
            if i:
                live.add(int(k))
        for k in range(1, 60):
            assert o.index_contains(0, k) == (k in live)
    hc.fihc_lru_free(l)


# ---- EndpointPickerConfig loader -----------------------------------------------------
# The documents FusionInfer's router role generates
# (/root/reference/pkg/router/strategy.go:51-68, 70-83, 85-98, 115-165): the drop-in must
# accept them unchanged.  Reproduced here as test inputs (they are the interface contract).
PREFIX_YAML = """apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
- type: prefix-cache-scorer
  parameters:
    blockSize: 5
    maxPrefixBlocksToMatch: 256
    lruCapacityPerServer: 31250
- type: max-score-picker
schedulingProfiles:
- name: default
  plugins:
  - pluginRef: max-score-picker
  - pluginRef: prefix-cache-scorer
    weight: 100
"""

def _single(kind):
    return f"""apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
- type: {kind}
- type: max-score-picker
schedulingProfiles:
- name: default
  plugins:
  - pluginRef: max-score-picker
  - pluginRef: {kind}
    weight: 100
"""

PD_YAML = """apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
- type: pd-profile-handler
  parameters:
    threshold: 0
    hashBlockSize: 5
    primaryPort: 8000
- type: prefill-header-handler
- type: by-label
  name: prefill-pods
  parameters:
    label: "fusioninfer.io/component-type"
    validValues: ["prefiller"]
- type: by-label
  name: decode-pods
  parameters:
    label: "fusioninfer.io/component-type"
    validValues: ["decoder"]
- type: prefix-cache-scorer
  parameters:
    hashBlockSize: 5
    maxPrefixBlocksToMatch: 256
    lruCapacityPerServer: 31250
- type: max-score-picker
schedulingProfiles:
- name: prefill
  plugins:
  - pluginRef: prefill-pods
  - pluginRef: max-score-picker
  - pluginRef: prefix-cache-scorer
    weight: 50
- name: decode
  plugins:
  - pluginRef: decode-pods
  - pluginRef: max-score-picker
  - pluginRef: prefix-cache-scorer
    weight: 50
"""


def test_config_prefix_cache_strategy():
    cfg = config_from_yaml(PREFIX_YAML)
    assert (cfg.block_bytes, cfg.max_blocks, cfg.lru_capacity) == (5, 256, 31250)
    assert cfg.n_profiles == 1 and cfg.pd_enabled == 0
    p = cfg.profiles[0]
    assert p.name == b"default" and p.role_mask == 0 and p.n_scorers == 1
    assert (p.scorers[0].kind, p.scorers[0].weight) == (abi.FI_SCORER_PREFIX, 100)


@pytest.mark.parametrize("kind,enum", [("kv-cache-utilization-scorer", abi.FI_SCORER_KV_UTIL),
                                       ("queue-scorer", abi.FI_SCORER_QUEUE),
                                       ("lora-affinity-scorer", abi.FI_SCORER_LORA)])
def test_config_single_scorer_strategies(kind, enum):
    cfg = config_from_yaml(_single(kind))
    assert cfg.n_profiles == 1
    assert (cfg.profiles[0].scorers[0].kind, cfg.profiles[0].scorers[0].weight) == (enum, 100)
    assert cfg.block_bytes == default_config().block_bytes  # untouched without a prefix scorer


def test_config_pd_disaggregation_strategy():
    cfg = config_from_yaml(PD_YAML)
    assert cfg.pd_enabled == 1 and cfg.pd_threshold == 0.0
    assert cfg.n_profiles == 2
    assert cfg.profiles[cfg.pd_prefill_profile].name == b"prefill"
    assert cfg.profiles[cfg.pd_decode_profile].name == b"decode"
    assert cfg.profiles[cfg.pd_prefill_profile].role_mask == abi.FI_ROLE_PREFILLER
    assert cfg.profiles[cfg.pd_decode_profile].role_mask == abi.FI_ROLE_DECODER
    for i in range(2):
        assert (cfg.profiles[i].scorers[0].kind, cfg.profiles[i].scorers[0].weight) == (abi.FI_SCORER_PREFIX, 50)
    assert (cfg.block_bytes, cfg.max_blocks, cfg.lru_capacity) == (5, 256, 31250)


def test_config_custom_passthrough_multi_scorer_and_comments():
    y = """# custom EndpointPickerConfig (role.EndpointPickerConfig passthrough, strategy.go:29-31)
apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
  - type: prefix-cache-scorer   # indented list style
    name: pfx
    parameters:
      hashBlockSize: 64
      maxPrefixBlocksToMatch: 128
  - type: kv-cache-utilization-scorer
  - type: queue-scorer
  - type: max-score-picker
schedulingProfiles:
  - name: default
    plugins:
      - pluginRef: max-score-picker
      - pluginRef: pfx
        weight: 3
      - pluginRef: queue-scorer
        weight: 2
      - pluginRef: kv-cache-utilization-scorer
"""
    cfg = config_from_yaml(y)
    assert (cfg.block_bytes, cfg.max_blocks) == (64, 128)
    p = cfg.profiles[0]
    got = [(p.scorers[i].kind, p.scorers[i].weight) for i in range(p.n_scorers)]
    assert got == [(abi.FI_SCORER_PREFIX, 3), (abi.FI_SCORER_QUEUE, 2), (abi.FI_SCORER_KV_UTIL, 1)]


@pytest.mark.parametrize("bad,frag", [
    ("kind: Foo\napiVersion: inference.networking.x-k8s.io/v1alpha1\n", "kind"),
    (PREFIX_YAML.replace("max-score-picker\nschedulingProfiles", "random-picker\nschedulingProfiles"), "unsupported plugin"),
    (PREFIX_YAML.replace("  - pluginRef: max-score-picker\n", ""), "picker"),
    (PREFIX_YAML.replace("pluginRef: prefix-cache-scorer", "pluginRef: nope"), "unknown pluginRef"),
    (PREFIX_YAML.replace("256", "100000"), "maxPrefixBlocksToMatch"),
    (PD_YAML.replace("- name: decode", "- name: dec"), "prefill' and 'decode'"),
    ("", "empty"),
])
def test_config_rejects_bad_documents(bad, frag):
    with pytest.raises(FiEppError) as ei:
        config_from_yaml(bad)
    assert ei.value.status == abi.FI_ERR_CONFIG and frag in str(ei.value)


def test_tie_rotation_arithmetic_of_the_kernels(hc):
    """tiebreak.cuh (what the match / merge kernels compile) against the python statement of the rule in
    tests/restate.py: rotation start, rotated distance, and — the part with the bit tricks — the first member
    of a LOCAL tie set in rotation order for shards anywhere in the pool."""
    from tests import restate

    rng = np.random.default_rng(11)
    for _ in range(300):
        E = int(rng.integers(1, 5000))
        n = int(rng.integers(0, 3))
        fh, h0, r = int(rng.integers(0, 2**63)) * 2 + 1, int(rng.integers(0, 2**63)), int(rng.integers(0, 70000))
        start = hc.fihc_tie_start(n, fh, h0, r, E)
        assert start == restate.tie_start(n, fh, h0, r, E) and start < E
        e = int(rng.integers(0, E))
        assert hc.fihc_tie_rot(e, start, E) == (e - start) % E
    for _ in range(400):
        W = int(2 ** rng.integers(0, 8))
        world = int(rng.integers(1, 9))
        ep_count = int(rng.integers(1, W * 32 + 1))
        rank = int(rng.integers(0, world))
        ep_begin = rank * ep_count
        E = world * ep_count
        start = int(rng.integers(0, E))
        dens = rng.choice([0.0, 0.02, 0.5, 1.0])
        members = [e for e in range(ep_count) if rng.random() < dens]
        words = np.zeros(W, dtype=np.uint32)
        for e in members:
            words[e // 32] |= np.uint32(1 << (e % 32))
        got = hc.fihc_tie_first_local(words.ctypes.data, W, start, ep_begin, ep_count)
        want = min(members, key=lambda e: (e + ep_begin - start) % E) if members else 0xFFFFFFFF
        assert got == want, (W, ep_begin, ep_count, start, members[:8], got, want)


LABELS_YAML = """apiVersion: inference.networking.x-k8s.io/v1alpha1
kind: EndpointPickerConfig
plugins:
- type: prefix-cache-scorer
  parameters:
    hashBlockSize: 64
- type: queue-scorer
- type: max-score-picker
- type: by-label
  name: decode-role
  parameters:
    label: "fusioninfer.io/component-type"
    validValues: ["decoder", "worker"]
- type: by-label
  name: zone-filter
  parameters:
    label: "topology.kubernetes.io/zone"
    validValues: ["us-east-1a", "us-east-1b"]
- type: by-label
  name: gpu-filter
  parameters:
    label: "nvidia.com/gpu.product"
    validValues: ["H100"]
schedulingProfiles:
- name: default
  plugins:
  - pluginRef: decode-role
  - pluginRef: zone-filter
  - pluginRef: gpu-filter
  - pluginRef: max-score-picker
  - pluginRef: prefix-cache-scorer
    weight: 70
  - pluginRef: queue-scorer
    weight: 30
"""


def test_config_by_label_with_arbitrary_labels_and_chained_filters():
    """strategy.go:135-144 gives the by-label schema (label + validValues); SURVEY §8(f)3 asks for arbitrary
    label sets.  Component-type values keep their fixed bits, other (label, value) pairs get the next free bit,
    the assignment is reported in cfg.labels, and several filters in one profile are ANDed."""
    cfg = config_from_yaml(LABELS_YAML)
    p = cfg.profiles[0]
    assert p.role_mask == abi.FI_ROLE_DECODER | abi.FI_ROLE_WORKER
    assert p.n_more_filters == 2
    table = {(cfg.labels[i].label.decode(), cfg.labels[i].value.decode()): cfg.labels[i].bit for i in range(cfg.n_labels)}
    assert table[("fusioninfer.io/component-type", "decoder")] == abi.FI_ROLE_DECODER
    assert table[("fusioninfer.io/component-type", "worker")] == abi.FI_ROLE_WORKER
    za, zb = table[("topology.kubernetes.io/zone", "us-east-1a")], table[("topology.kubernetes.io/zone", "us-east-1b")]
    gb = table[("nvidia.com/gpu.product", "H100")]
    assert {za, zb, gb} == {8, 16, 32} and p.more_filters[0] == za | zb and p.more_filters[1] == gb
    # two filters on the same label with disjoint values: ANDed -> nothing passes (round 1 read that as "no filter")
    doc = PD_YAML.replace("  - pluginRef: prefill-pods\n", "  - pluginRef: prefill-pods\n  - pluginRef: decode-pods\n", 1)
    cfg2 = config_from_yaml(doc)
    pf = cfg2.profiles[cfg2.pd_prefill_profile]
    assert pf.role_mask == abi.FI_ROLE_PREFILLER and pf.n_more_filters == 1 and pf.more_filters[0] == abi.FI_ROLE_DECODER


@pytest.mark.parametrize("workers", [1, 3, 8])
def test_batch_lru_walk_equals_sequential_adds(hc, workers):
    """fi_epp_index_add_chains' host phase (lru_batch.h: requests bucketed by endpoint, LRUs walked on a worker
    pool, ops emitted in segments) against the definition — one indexer.Add after the other.  Small capacity and
    recurring chains force evictions and re-adds of evicted hashes INSIDE one batch (the multi-segment path)."""
    rng = np.random.default_rng(17 + workers)
    E, cap, R, pitch, batches = 7, 40, 120, 24, 5
    pool_chains = rng.integers(1, 2**63, size=(30, pitch), dtype=np.uint64)  # 30 recurring chains
    eps = rng.integers(0, E + 2, size=(batches, R)).astype(np.uint32)
    eps[eps == E] = 0xFFFFFFFF      # FI_NO_ENDPOINT: skipped
    eps[eps == E + 1] = E + 100     # another shard: skipped
    pick = rng.integers(0, 30, size=(batches, R))
    chains = pool_chains[pick].copy()
    fresh = rng.random((batches, R)) < 0.3     # some requests end in unique blocks
    chains[fresh, pitch // 2:] = rng.integers(1, 2**63, size=(int(fresh.sum()), pitch - pitch // 2), dtype=np.uint64)
    nb = rng.integers(0, pitch + 1, size=(batches, R)).astype(np.uint32)
    seg = C.c_uint32(0)
    rc = hc.fihc_lru_batch_check(E, cap, eps.ctypes.data, np.ascontiguousarray(chains).ctypes.data, pitch, nb.ctypes.data, R,
                                 batches, workers, C.byref(seg))
    assert rc == 0
    assert seg.value >= 2  # the same-batch re-add path really ran


@pytest.mark.parametrize("plan_cap,cap_touches,cap_requests,min_subs",
                         [(40, 1 << 30, 1 << 30, 2), (0xFFFFFFFF, 1 << 30, 1 << 30, 1), (0xFFFFFFFF, 300, 1 << 30, 2),
                          (40, 1 << 30, 7, 2), (0xFFFFFFFF, 1 << 30, 7, 2)])
def test_device_lru_batch_rule_equals_sequential_adds(hc, plan_cap, cap_touches, cap_requests, min_subs):
    """The rule the device-resident LRU applies (lru_kernels.cu): a sub-batch planned by lru_plan.h is applied at
    once (touched keys move to the back in the order of their LAST touch, then the oldest beyond the capacity go —
    which also removes keys touched early in a sub-batch that brings more than `capacity` distinct ones).  Against
    one indexer.Add after the other: same recency ORDER and content after every batch, with hot endpoints,
    recurring chains, the conservative per-endpoint cap (40 = the capacity) and the optimistic one (none), and
    scratch-size cuts."""
    rng = np.random.default_rng(23)
    E, cap, R, pitch, batches = 5, 40, 150, 24, 6
    pool_chains = rng.integers(1, 2**63, size=(30, pitch), dtype=np.uint64)
    eps = rng.integers(0, E + 2, size=(batches, R)).astype(np.uint32)
    eps[eps == E] = 0xFFFFFFFF
    eps[eps == E + 1] = E + 100
    eps[2, :] = 3                    # one endpoint takes a whole batch
    pick = rng.integers(0, 30, size=(batches, R))
    chains = pool_chains[pick].copy()
    fresh = rng.random((batches, R)) < 0.3
    chains[fresh, pitch // 2:] = rng.integers(1, 2**63, size=(int(fresh.sum()), pitch - pitch // 2), dtype=np.uint64)
    nb = rng.integers(0, pitch + 1, size=(batches, R)).astype(np.uint32)
    subs = C.c_uint32(0)
    rc = hc.fihc_lru_plan_check(E, cap, eps.ctypes.data, np.ascontiguousarray(chains).ctypes.data, pitch, nb.ctypes.data, R,
                                batches, plan_cap, cap_touches, cap_requests, C.byref(subs))
    assert rc == 0
    assert subs.value >= min_subs
