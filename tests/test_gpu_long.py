"""GPU (-m gpu): prompts of up to FI_EPP_MAX_BLOCKS = 1023 blocks, and every tile shape of the fused block-hash +
chain-walk kernel, bit-exact against the CPU oracle.

Several paths only start above 256 blocks:
- match_pick's dynamic shared memory is 160 bytes per block of the chain pitch MP = roundup8(max_blocks); from
  max_blocks = 305 on it is above 48 KiB and needs the per-kernel opt-in (160 KiB at 1023);
- resolve_request_nodes verifies 256 blocks per speculation round; a cached chain of more than 257 blocks takes a
  second round, and a scattered one runs out of speculation tries and probes the table 64 blocks at a time;
- the bit-plane match counters use plane 9 only from a count of 512 on; 1023 sets all ten planes;
- chains_out has a pitch of max_blocks, the device buffers one of MP.
hash_chain runs tiles of 32 * WALK requests, WALK = 1, 2 or 4 by batch size and SM count, and its ring of
pre-states wraps ceil(n / 8) / ring-slots times per tile.
"""
import dataclasses

import numpy as np
import pytest

from fusioninfer_b200 import LORA_DTYPE, EndpointPicker, make_config, synth
from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import helpers as H

pytestmark = pytest.mark.gpu
P, K, Q, L = H.P, H.K, H.Q, abi.FI_SCORER_LORA
WEIGHTED = [{"name": "default", "scorers": [(P, 100), (K, 13), (Q, 7)]}]
WITH_LORA = [{"name": "default", "scorers": [(P, 60), (L, 30), (K, 5), (Q, 5)]}]


def _match_smem(max_blocks):
    """match_pick's dynamic shared memory: 8 warps x MP x (two chain words + one node word)"""
    return 8 * ((max_blocks + 7) // 8 * 8) * 20


def _long_workload(E, M, R=128, pd=False):
    """Prompts of M + 2 whole 64-byte blocks and a partial one: n is capped at M and the tail is ignored.  Shared
    prefixes are T/4 .. 3T/4 long (about 256 .. 768 blocks at M = 1023).  Few groups per endpoint and no filler
    keep the index (and the oracle) small."""
    gpe = 4 if E <= 8 else (2 if E <= 128 else 1)
    return synth.Workload(R=R, E=E, T=16 * (M + 2) + 5, seed=synth.SEEDS[2], max_blocks=M, lru_capacity=gpe * M,
                          groups_per_endpoint=gpe, pd=pd)


def _index_ops(wl, holes):
    """{holes: SET ops of wl's initial index}; the group chains are hashed once for all variants"""
    chains = wl.group_chains(wl.endpoint_groups())
    out = {}
    for h in holes:
        w = dataclasses.replace(wl, holes=h)
        w.group_chains = lambda groups: chains
        out[h] = np.concatenate(list(w.index_ops(chunk_endpoints=256)))
    return out


def _direct_chain(wl, tok, r, endpoint):
    """SET ops of request r's whole chain for one endpoint, in chain order"""
    chain = synth.chain_py(tok[r].tobytes(), wl.block_bytes, wl.max_blocks, wl.h0)
    assert len(chain) == wl.max_blocks
    ops = np.zeros(len(chain), dtype=H.OP_DTYPE)
    ops["hash"] = chain
    ops["endpoint"] = endpoint
    ops["op"] = abi.FI_OP_SET
    return ops


def _slots(*ops):
    keys = len(np.unique(np.concatenate([o["hash"] for o in ops])))
    slots = 4096
    while slots < 2 * keys:
        slots *= 2
    return slots


def _handles(wl, ops_list, states, **cfg_kw):
    """a GPU handle and the oracle, each with the endpoint states and every op list applied (one call per list on
    the oracle, slices of 64 Ki ops on the GPU)"""
    cfg = H.config_for(wl, index_slots=_slots(*ops_list), max_prompt_bytes=wl.R * wl.T * 4, **cfg_kw)
    gpu, cpu = EndpointPicker(cfg), eo.Oracle(cfg)
    gpu.update_endpoints(states)
    cpu.update_endpoints(states)
    for ops in ops_list:
        for lo in range(0, len(ops), 1 << 16):
            gpu.index_apply(ops[lo:lo + (1 << 16)])
        cpu.index_apply(ops)
    return gpu, cpu


def _unique_request(wl):
    _, shared = wl.request_params()
    return int(np.flatnonzero(shared == 0)[0])  # no group prefix: only the direct chain matches it


# ---------------------------------------------------------------------------------------
# match + pick over long prompts
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [305, 517, 1023])
@pytest.mark.parametrize("E", [8, 100, 1024])
def test_long_prompt_pick_parity(E, M):
    """Both match modes, with and without holes, over pools of one, four and 32 row words.  One unique prompt's
    whole chain is SET for one endpoint in chain order: that request matches all M blocks (1023 sets every bit
    plane), through every 256-block speculation round."""
    wl = _long_workload(E, M)
    tok, offs = wl.prompts()
    states = wl.endpoint_states()
    r_direct, e_direct = _unique_request(wl), E // 2
    direct = _direct_chain(wl, tok, r_direct, e_direct)
    ops = _index_ops(wl, (False, True))
    for holes in (False, True):
        for mode in (abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM):
            tag = f"holes={holes} mode={mode}"
            gpu, cpu = _handles(wl, [ops[holes], direct], states, profiles=WEIGHTED, match_mode=mode)
            got, gch = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
            want, wch = cpu.pick_batch(tok, offs, wl.h0, want_chains=True)
            gpu.close()
            cpu.close()
            assert np.array_equal(gch, wch), tag
            assert H.picks_equal(got, want), tag + "\n" + H.describe_diff(got, want)
            mb = want[:, 0]["match_blocks"]
            assert (want[:, 0]["n_blocks"] == M).all(), tag  # every prompt reaches the cap
            assert want[r_direct, 0]["endpoint"] == e_direct and mb[r_direct] == M, tag
            if holes:  # 5 % of the pairs missing cut most long prefixes short
                assert (mb > 0).sum() >= 3, tag
            else:
                assert (mb > 0).mean() > 0.2, tag
                if 3 * M // 4 > 512:  # shared group prefixes (up to 3/4 of the prompt) above 512 blocks
                    assert (mb > 512).sum() > 10, tag


@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
def test_long_prompt_pick_parity_shuffled_index(mode):
    """The same kind of index inserted in shuffled order: no cached chain has consecutive nodes, so each request
    runs out of speculation tries and its remaining blocks probe the table 64 at a time, up to 16 rounds."""
    M = 1023
    wl = _long_workload(100, M)
    tok, offs = wl.prompts()
    r_direct = _unique_request(wl)
    ops = np.concatenate([_index_ops(wl, (False,))[False], _direct_chain(wl, tok, r_direct, 7)])
    ops = ops[np.random.default_rng(5).permutation(len(ops))]
    gpu, cpu = _handles(wl, [ops], wl.endpoint_states(), profiles=WEIGHTED, match_mode=mode)
    got = gpu.pick_batch(tok, offs, wl.h0)
    want = cpu.pick_batch(tok, offs, wl.h0)
    gpu.close()
    assert H.picks_equal(got, want), H.describe_diff(got, want)
    mb = want[:, 0]["match_blocks"]
    assert mb[r_direct] == M and want[r_direct, 0]["endpoint"] == 7
    assert (mb > 512).sum() > 10


def test_long_prompt_pd_threshold_splits():
    """PD profiles over 1023-block prompts: the prefill profile runs iff (1 - hit) * len(prompt) >= threshold, with
    thresholds that send some long prompts to prefill and skip it for others."""
    wl = _long_workload(128, 1023, pd=True)
    profiles, _ = synth.baseline_profiles(5)
    tok, offs = wl.prompts()
    ops = _index_ops(wl, (False,))[False]
    split = 0
    for thr in (0.0, 20000.0, 40000.0, 1e9):
        gpu, cpu = _handles(wl, [ops], wl.endpoint_states(), profiles=profiles,
                            pd={"decode": 1, "prefill": 0, "threshold": thr})
        got = gpu.pick_batch(tok, offs, wl.h0)
        want = cpu.pick_batch(tok, offs, wl.h0)
        gpu.close()
        assert H.picks_equal(got, want), f"threshold {thr}\n" + H.describe_diff(got, want)
        skipped = (want[:, 0]["endpoint"] == abi.FI_NO_ENDPOINT).mean()
        if thr == 0.0:
            assert skipped == 0.0
        elif thr == 1e9:
            assert skipped == 1.0
        else:
            split += 0.0 < skipped < 1.0
    assert split == 2


def _lora_states(E, rng, n_adapters=12):
    st = np.zeros(E, dtype=LORA_DTYPE)
    st["endpoint"] = np.arange(E)
    for e in range(E):
        na, nw = int(rng.integers(0, 5)), int(rng.integers(0, 3))
        ids = rng.permutation(n_adapters)[: na + nw] + 1000
        st[e]["n_active"], st[e]["n_waiting"] = na, nw
        st[e]["active"][:na] = ids[:na]
        st[e]["waiting"][:nw] = ids[na:]
        st[e]["max_active"] = int(rng.integers(0, 7))
    return st


def test_every_match_variant_opts_into_its_shared_memory():
    """The four match kernels of one row shape (upstream / LPM, with / without a LoRA scorer) each need their own
    shared-memory opt-in above 48 KiB.  Four handles of the same pool size, one per variant, are created one after
    the other and each must pick exactly like the oracle: at 1023 blocks (160 KiB), at 305 (just above 48 KiB) and
    at 304 (just below)."""
    assert _match_smem(304) <= 48 * 1024 < _match_smem(305)
    E = 100
    rng = np.random.default_rng(17)
    lora = _lora_states(E, rng)
    for M in (1023, 305, 304):
        wl = _long_workload(E, M, R=64)
        tok, offs = wl.prompts()
        ops = _index_ops(wl, (False,))[False]
        adapters = (rng.integers(0, 14, size=wl.R) + 1000).astype(np.uint64)
        for mode in (abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM):
            for profiles in (WEIGHTED, WITH_LORA):
                tag = f"max_blocks={M} mode={mode} lora={profiles is WITH_LORA}"
                gpu, cpu = _handles(wl, [ops], wl.endpoint_states(), profiles=profiles, match_mode=mode)
                if profiles is WITH_LORA:
                    gpu.update_endpoints_lora(lora)
                    cpu.update_endpoints_lora(lora)
                    got = gpu.pick_batch(tok, offs, wl.h0, adapters=adapters)
                    want = cpu.pick_batch(tok, offs, wl.h0, adapters=adapters)
                else:
                    got = gpu.pick_batch(tok, offs, wl.h0)
                    want = cpu.pick_batch(tok, offs, wl.h0)
                gpu.close()
                assert H.picks_equal(got, want), tag + "\n" + H.describe_diff(got, want)
                assert (want[:, 0]["match_blocks"] > 0).any(), tag


# ---------------------------------------------------------------------------------------
# block hashing: every hash_chain tile shape
# ---------------------------------------------------------------------------------------
def _hash_walk(R, sms):
    """requests per hash_chain tile / 32, chosen like launch_hash_chain: the smallest tile whose grid fits one CTA
    per SM, 128 requests beyond that"""
    walk = 1
    while walk < 4 and -(-R // (32 * walk)) > sms:
        walk *= 2
    return walk


@pytest.mark.parametrize("M", [5, 24, 1023])
@pytest.mark.parametrize("B", [32, 64, 128, 96, 160, 256])
def test_hash_parity_every_tile_shape(B, M):
    """Batches of 1 .. 128 * SMs + 45 requests: the smallest batch of each tile shape (WALK = 1, 2, 4), partial last
    tiles, and a grid larger than the SM count.  Ragged lengths and unaligned starts; about one request in 32 is
    longer than the cap (it sets its tile's group count and wraps the ring), the rest are short.  B = 96, 160 and
    256 take hash_chain<0, WALK>, which reads the stripe count at run time.  Chains, block counts and the zero tail
    beyond n are compared with the oracle."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [1, 33, 32 * sms - 7, 32 * sms + 1, 64 * sms - 3, 64 * sms + 1, 128 * sms + 45]
    walks = [_hash_walk(R, sms) for R in sizes]
    assert walks == [1, 1, 1, 2, 2, 4, 4] and -(-sizes[-1] // 128) > sms
    R = sizes[-1]
    rng = np.random.default_rng(1000 * B + M)
    lens = rng.integers(0, min(M, 6) * B + B, size=R)
    full = np.arange(0, R, 32) + rng.integers(0, 32, size=-(-R // 32))
    full = np.append(full[full < R], 0)
    lens[full] = M * B + rng.integers(0, 2 * B, size=len(full))  # at or past the cap, with a ragged tail
    offs = np.zeros(R + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    data = np.frombuffer(rng.bytes(int(offs[-1]) + 16), dtype=np.uint8)
    h0 = rng.integers(0, 2**63, size=R, dtype=np.uint64)
    cfg = make_config(num_endpoints=1, block_bytes=B, max_blocks=M, max_batch=R, max_prompt_bytes=int(offs[-1]))
    gpu, cpu = EndpointPicker(cfg), eo.Oracle(cfg)
    wc, wn = cpu.hash_batch(data, offs, h0)
    assert (wn[full] == M).all() and (wn < M).any()
    for n, walk in zip(sizes, walks):
        gc, gn = gpu.hash_batch(data, offs[: n + 1], h0[:n])
        tag = f"R={n} WALK={walk}"
        assert np.array_equal(gn, wn[:n]), tag
        assert np.array_equal(gc, wc[:n]), tag
        assert not gc[np.arange(M)[None, :] >= gn[:, None]].any(), tag
    gpu.close()
