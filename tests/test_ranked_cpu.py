"""CPU: the ranked pick's configuration entry point and its oracle (docs/SPEC.md S.6a).

fi_epp_config_picker_endpoints reads each profile's max-score-picker maxNumOfEndpoints through the same loader as
fi_epp_config_from_yaml.  The ranked oracle (tests/ranked_oracle.cpp) is checked against a ranking built here with
numpy from tests/restate.py's independent match, eligibility and score pieces.
"""
import ctypes as C

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi
from fusioninfer_b200 import config_from_yaml, make_config, synth
from fusioninfer_b200.picker import FiEppError, config_picker_endpoints
from tests import helpers as H
from tests import restate
from tests.ranked_oracle import RankedOracle
from tests.test_host_logic import PD_YAML, PREFIX_YAML, _single

P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA


def _with_k(doc, k):
    """the document with `maxNumOfEndpoints: k` on its (single) max-score-picker plugin"""
    return doc.replace("- type: max-score-picker\n", f"- type: max-score-picker\n  parameters:\n    maxNumOfEndpoints: {k}\n")


# ---- fi_epp_config_picker_endpoints -------------------------------------------------------------------------------
@pytest.mark.parametrize("doc,n", [(PREFIX_YAML, 1), (PD_YAML, 2), (_single("queue-scorer"), 1),
                                   (_single("lora-affinity-scorer"), 1)])
def test_picker_endpoints_default_to_one(doc, n):
    assert config_picker_endpoints(doc) == [1] * n


@pytest.mark.parametrize("k", [1, 3, 16])
def test_picker_endpoints_read_the_parameter(k):
    assert config_picker_endpoints(_with_k(PREFIX_YAML, k)) == [k]
    assert config_picker_endpoints(_with_k(PD_YAML, k)) == [k, k]


def test_picker_endpoints_per_profile_with_pd():
    """two pickers: prefill asks for 4 fallbacks, decode keeps the default"""
    doc = PD_YAML.replace("- type: max-score-picker\n",
                          "- type: max-score-picker\n  parameters:\n    maxNumOfEndpoints: 4\n"
                          "- type: max-score-picker\n  name: single\n")
    doc = doc.replace("""  - pluginRef: decode-pods
  - pluginRef: max-score-picker""", """  - pluginRef: decode-pods
  - pluginRef: single""")
    cfg = config_from_yaml(doc)
    ks = config_picker_endpoints(doc)
    assert ks[cfg.pd_prefill_profile] == 4 and ks[cfg.pd_decode_profile] == 1 and len(ks) == 2


@pytest.mark.parametrize("bad", ["0", "17", '"three"', "three", "-1", "2.5", "[2]"])
def test_picker_endpoints_reject_values_out_of_range(bad):
    doc = _with_k(PREFIX_YAML, bad)
    with pytest.raises(FiEppError) as ei:
        config_picker_endpoints(doc)
    assert ei.value.status == abi.FI_ERR_CONFIG and "maxNumOfEndpoints" in str(ei.value)
    config_from_yaml(doc)  # the loader itself does not look at the parameter


def test_config_from_yaml_still_accepts_any_picker_width():
    for v in ("100", "0", "three"):
        cfg = config_from_yaml(_with_k(PREFIX_YAML, v))
        assert (cfg.n_profiles, cfg.max_blocks) == (1, 256)


@pytest.mark.parametrize("bad", [
    "kind: Foo\napiVersion: inference.networking.x-k8s.io/v1alpha1\n",
    PREFIX_YAML.replace("max-score-picker\nschedulingProfiles", "random-picker\nschedulingProfiles"),
    PREFIX_YAML.replace("  - pluginRef: max-score-picker\n", ""),
    PREFIX_YAML.replace("pluginRef: prefix-cache-scorer", "pluginRef: nope"),
    PREFIX_YAML.replace("256", "100000"),
    PD_YAML.replace("- name: decode", "- name: dec"),
    "",
])
def test_picker_endpoints_reject_what_the_loader_rejects(bad):
    with pytest.raises(FiEppError) as want:
        config_from_yaml(bad)
    with pytest.raises(FiEppError) as got:
        config_picker_endpoints(bad)
    assert got.value.status == want.value.status == abi.FI_ERR_CONFIG
    assert str(got.value).split(": ", 2)[-1] == str(want.value).split(": ", 2)[-1]  # the same message


def test_picker_endpoints_null_arguments():
    lib = abi.load()
    out = (C.c_uint32 * abi.FI_EPP_MAX_PROFILES)()
    assert lib.fi_epp_config_picker_endpoints(None, 0, out, None, 0) == abi.FI_ERR_INVALID
    raw = PREFIX_YAML.encode()
    assert lib.fi_epp_config_picker_endpoints(raw, len(raw), None, None, 0) == abi.FI_ERR_INVALID


# ---- the ranked oracle against a numpy ranking from tests/restate.py -----------------------------------------------
def _numpy_ranking(rs, prompts, offsets, h0, k, adapters=None):
    """[R, P, k] (endpoint, match, n, total) rows: every eligible endpoint's total from restate's pieces, ordered by
    np.lexsort on (rotation distance, -total)"""
    R = len(offsets) - 1
    raw = bytes(np.ascontiguousarray(prompts).view(np.uint8))
    h0 = np.broadcast_to(np.asarray(h0, dtype=np.uint64), (R,))
    out = np.zeros((R, len(rs.profiles), k), dtype=H.PICK_DTYPE)
    for r in range(R):
        p = raw[int(offsets[r]):int(offsets[r + 1])]
        ch = restate.chain(p, rs.B, rs.M, int(h0[r]))
        n = len(ch)
        counts = rs.match(ch)
        start = restate.tie_start(n, ch[0] if n else 0, int(h0[r]), r, rs.E)
        ad = int(adapters[r]) if adapters is not None else 0
        for pi, prof in enumerate(rs.profiles):
            el = np.array([e for e in range(rs.E) if rs._eligible(e, prof)], dtype=np.int64)
            row = np.zeros(k, dtype=H.PICK_DTYPE)
            row["endpoint"] = restate.NO_ENDPOINT
            row["n_blocks"] = n
            if len(el):
                m = np.array([counts.get(int(e), 0) for e in el], dtype=np.float64)
                q = np.array([rs.state[int(e)]["queue"] for e in el], dtype=np.float64)
                mn, mx = q.min(), q.max()
                total = np.zeros(len(el))
                for kind, w in prof["scorers"]:
                    if kind == restate.KIND_PREFIX:
                        s = m / n if n else np.zeros(len(el))
                    elif kind == restate.KIND_KV:
                        s = 1.0 - np.array([rs.state[int(e)]["kv_util"] for e in el])
                    elif kind == restate.KIND_QUEUE:
                        s = np.ones(len(el)) if mx == mn else (mx - q) / (mx - mn)
                    else:
                        s = np.array([rs._lora_score(int(e), ad) for e in el])
                    total = total + np.clip(s, 0.0, 1.0) * float(w)
                order = np.lexsort(((el - start) % rs.E, -total))[:k]
                j = len(order)
                row["endpoint"][:j] = el[order]
                row["match_blocks"][:j] = m[order]
                row["score"][:j] = total[order]
            out[r, pi] = row
        if rs.pd:
            d = out[r, rs.pd["decode"], 0]
            hit = (int(d["match_blocks"]) / n) if (d["endpoint"] != restate.NO_ENDPOINT and n) else 0.0
            if not ((1.0 - hit) * float(len(p)) >= float(rs.pd.get("threshold", 0.0))):
                out[r, rs.pd["prefill"]] = (restate.NO_ENDPOINT, 0, n, 0.0)
    return out


def _random_states(E, rng, dead_frac=0.2):
    st = H.states_array(E, kv=rng.integers(0, 8, E) / 8.0, queue=rng.integers(0, 4, E),
                        roles=rng.integers(1, 32, E).astype(np.uint32))
    st["flags"] = np.where(rng.random(E) < dead_frac, 0, abi.FI_ENDPOINT_ALIVE)
    return st


def _random_lora(E, rng):
    from fusioninfer_b200 import LORA_DTYPE

    st = np.zeros(E, dtype=LORA_DTYPE)
    st["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 4)), int(rng.integers(0, 3))
        ids = rng.permutation(8)[: na + nw] + 100
        st[e]["n_active"], st[e]["n_waiting"] = na, nw
        st[e]["active"][:na] = ids[:na]
        st[e]["waiting"][:nw] = ids[na:]
        st[e]["max_active"] = int(rng.integers(0, 6))
    return st


CASES = {
    "prefix": dict(profiles=[{"name": "default", "scorers": [(P, 100)]}]),
    "weighted": dict(profiles=[{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]),
    "filters": dict(profiles=[{"name": "a", "role_mask": 3, "more_filters": [12], "scorers": [(P, 10), (Q, 3)]},
                              {"name": "b", "role_mask": 16, "scorers": [(K, 1)]}]),
    "lora": dict(profiles=[{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5)]}]),
    "pd": dict(profiles=[{"name": "prefill", "role_mask": 1, "scorers": [(P, 50), (K, 5)]},
                         {"name": "decode", "role_mask": 2, "scorers": [(P, 50), (Q, 5)]}],
               pd={"prefill": 0, "decode": 1, "threshold": 320.0}),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("E", [1, 5, 40])
def test_ranked_oracle_matches_numpy_ranking(case, mode, E):
    rng = np.random.default_rng(E * 7 + mode)
    wl = synth.Workload(R=24, E=E, T=160, seed=synth.SEEDS[1], max_blocks=8, lru_capacity=64, holes=True)
    cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=wl.R,
                      match_mode=mode, **CASES[case])
    orc, rs = RankedOracle(cfg), restate.from_config(cfg)
    st = _random_states(E, rng)
    orc.update_endpoints(st)
    rs.update_endpoints(st)
    if case == "lora":
        lo = _random_lora(E, rng)
        orc.update_endpoints_lora(lo)
        rs.update_lora(lo)
    for ops in wl.index_ops():
        orc.index_apply(ops)
        rs.apply(ops)
    tok, offs = wl.prompts()
    # the first quarter of the requests are prompts shorter than a block (n = 0: every total ties)
    offs = offs.copy()
    offs[1:7] = offs[0] + np.arange(1, 7, dtype=np.uint64) * 5
    adapters = (rng.integers(0, 10, wl.R) + 100).astype(np.uint64) if case == "lora" else None
    for k in (1, 3, E + 2):
        got = orc.pick_batch_ranked(tok, offs, wl.h0, k, adapters=adapters)
        want = _numpy_ranking(rs, tok, offs, wl.h0, k, adapters=adapters)
        assert H.picks_equal(got, want), f"k={k}\n" + H.describe_diff(got, want)
        # entry 0 is the oracle's single pick
        single = orc.pick_batch(tok, offs, wl.h0, adapters=adapters)
        assert H.picks_equal(np.ascontiguousarray(got[:, :, 0]), single)
    orc.close()
