#!/usr/bin/env python
"""Per-endpoint LRU capacities (fi_epp_set_lru_capacities, docs/SPEC.md S.2b) at the headline pool (cfg 3).

1. Churn, as tools/bench_churn.py runs it (pick + indexer.Add of every decision through the device LRU, the LRUs
   filled to capacity first), in three variants:
     never     capacities never set;
     uniform   every capacity set to lru_capacity;
     hetero    a third of the pods at 31 250, a third at 15 625, a third at 7 813.
   Reported: decisions/s over the timed steps.  Exactness: `never` is checked bit for bit against the oracle on the
   first --oracle-steps steps; `uniform` must give byte-identical picks to `never` at every step; `hetero` is checked
   bit for bit against the capacity oracle (the CPU oracle with per-endpoint capacities, tests/ext_oracle.cpp,
   built by `make`) fed the same calls, on the first --oracle-steps steps.
2. Resize: the time of fi_epp_set_lru_capacities(want_evicted) halving the capacity of 1, 64 and 1 024 pods of a
   full index (a fresh handle each), and the entries evicted.

    python tools/bench_lru_capacity.py [--cfg 3] [--steps 8] [--oracle-steps 2]

Prints one JSON line, with the card's name, power limit and SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def fill(wl, adders):
    """the initial state through the LRUs, as tools/bench_churn.py builds it (filler first: it is the oldest)"""
    nb = wl.n_blocks
    for ops in wl.index_ops(chunk_endpoints=64):
        e, h = ops["endpoint"], ops["hash"]
        rows, eps = [], []
        for ep in np.unique(e):
            he = h[e == ep]
            seq = np.concatenate([he[wl.groups_per_endpoint * nb:], he[: wl.groups_per_endpoint * nb]])
            seq = np.concatenate([seq, np.zeros((-len(seq)) % nb, dtype=np.uint64)])
            rows.append(seq.reshape(-1, nb))
            eps.append(np.full(rows[-1].shape[0], ep, dtype=np.uint32))
        ch, ee = np.concatenate(rows), np.concatenate(eps)
        valid = (ch != 0).sum(axis=1).astype(np.uint32)
        for add in adders:
            add(ee, ch, valid)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--oracle-steps", type=int, default=2)
    args = ap.parse_args()

    from fusioninfer_b200 import EndpointPicker, PinnedBuffer, make_config, synth
    from oracle import epp_oracle as eo
    from tests.ext_oracle import ExtOracle

    wl = synth.baseline_workload(args.cfg)
    profiles, pd = synth.baseline_profiles(args.cfg)
    C, E, R = wl.lru_capacity, wl.E, wl.R
    slots = 4096
    while slots < 2 * E * C:
        slots *= 2
    cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=C,
                      max_batch=max(R, 8192), max_prompt_bytes=max(R, 8192) * wl.T * 4, index_slots=slots,
                      profiles=profiles, pd=pd)
    main_p = cfg.pd_decode_profile if cfg.pd_enabled else 0
    third = E // 3
    hetero = np.array([C] * third + [C // 2] * third + [(C + 3) // 4] * (E - 2 * third), dtype=np.uint32)
    all_eps = np.arange(E, dtype=np.uint32)
    card_before = card()

    def handle(device_lru):
        g = EndpointPicker(cfg)
        g.set_option("device_lru", device_lru)
        g.update_endpoints(wl.endpoint_states())
        return g

    # ---- 1. churn
    P = cfg.n_profiles
    pin_tok, pin_off, pin_h0 = PinnedBuffer(R * wl.T * 4), PinnedBuffer(8 * (R + 1)), PinnedBuffer(8 * R)
    pin_out, pin_ch = PinnedBuffer(16 * R * P), PinnedBuffer(8 * R * wl.max_blocks)
    pin_h0.array(np.uint64)[:] = np.uint64(wl.h0)
    picks_v = pin_out.array(np.uint8).view(np.dtype([("endpoint", "<u4"), ("match_blocks", "<u2"), ("n_blocks", "<u2"),
                                                      ("score", "<f8")])).reshape(R, P)
    chains_v = pin_ch.array(np.uint64).reshape(R, wl.max_blocks)
    churn, never_picks = {}, []
    for variant in ("never", "uniform", "hetero"):
        gpu = handle(1)
        if variant == "uniform":
            gpu.set_lru_capacities(all_eps, np.full(E, C, dtype=np.uint32))
        elif variant == "hetero":
            gpu.set_lru_capacities(all_eps, hetero)
        fill(wl, [gpu.index_add_chains])  # (allocates the device LRU before the mirror takes any HBM)
        gpu.index_sync()
        mirror = None
        if variant == "never":
            mirror = eo.Oracle(cfg)
            mirror.update_endpoints(wl.endpoint_states())
            mirror.index_reserve(2 * E * C)
        elif variant == "hetero":
            mirror = ExtOracle(cfg)
            mirror.update_endpoints(wl.endpoint_states())
            mirror.index_reserve(2 * E * C)
            mirror.set_lru_capacities(all_eps, hetero)
        if mirror is not None:
            fill(wl, [mirror.index_add_chains])
        rebuilds0 = None
        times, exact, identical = [], True, True
        first_timed = max(1, args.oracle_steps)  # step 0 warms up; mirrored steps also copy the chains back
        for step in range(args.steps):
            tok, offs = wl.prompts(batch=step)
            pin_tok.array(np.uint32)[:] = tok.reshape(-1)
            pin_off.array(np.uint64)[:] = offs
            mirrored = step < args.oracle_steps
            if step == first_timed:
                rebuilds0 = int(gpu.index_stats().rebuilds)
            t0 = time.perf_counter()
            # pinned host buffers, as tools/bench_churn.py times it
            gpu.pick_batch_raw(pin_tok.ptr, pin_off.ptr, pin_h0.ptr, R, pin_out.ptr, pin_ch.ptr if mirrored else 0)
            got, ch = picks_v, chains_v
            ends = np.ascontiguousarray(got[:, main_p]["endpoint"])
            nbl = np.ascontiguousarray(got[:, main_p]["n_blocks"]).astype(np.uint32)
            gpu.index_add_chains_device(ends, 0, 0, nbl)  # the chains of the pick just made, from the handle's buffer
            if step == args.steps - 1:
                gpu.index_sync()
            if step >= first_timed:
                times.append(time.perf_counter() - t0)
            if variant == "never":
                never_picks.append(got.tobytes())
            elif variant == "uniform":
                identical = identical and got.tobytes() == never_picks[step]
            if mirror is not None and mirrored:
                want = mirror.pick_batch(tok, offs, wl.h0, nthreads=os.cpu_count() or 1)
                exact = exact and got.tobytes() == want.tobytes()
                mirror.index_add_chains(ends, ch, nbl)
        t = np.array(times)
        st = gpu.index_stats()
        # an index rebuild (every ~16 M new keys) makes one step far slower: the median step is the steady rate
        churn[variant] = {"decisions_per_s": R * len(t) / float(t.sum()), "decisions_per_s_median_step": R / float(np.median(t)),
                          "step_ms": {"p50": 1e3 * float(np.median(t)), "min": 1e3 * float(t.min()), "max": 1e3 * float(t.max())},
                          "index_rebuilds_in_timed_steps": int(st.rebuilds) - rebuilds0, "lru_entries": int(st.lru_entries)}
        if variant == "never":
            churn[variant]["oracle_bit_exact_steps"] = {"steps": min(args.oracle_steps, args.steps), "exact": bool(exact)}
        elif variant == "uniform":
            churn[variant]["picks_identical_to_never"] = bool(identical)
        else:
            churn[variant]["capacity_oracle_bit_exact_steps"] = {"steps": min(args.oracle_steps, args.steps), "exact": bool(exact)}
        gpu.close()
        if mirror is not None:
            mirror.close()

    # ---- 2. resize: halve 1, 64 and 1 024 pods of a full index
    resize = []
    for n in (1, 64, E):
        gpu = handle(1)
        fill(wl, [gpu.index_add_chains])
        gpu.index_sync()
        eps = all_eps[:n]
        t0 = time.perf_counter()
        evicted = gpu.set_lru_capacities(eps, np.full(n, C // 2, dtype=np.uint32), want_evicted=True)
        dt = time.perf_counter() - t0
        tok, offs = wl.prompts(batch=0)  # the handle still serves picks after the resize
        gpu.pick_batch(tok, offs, wl.h0)
        resize.append({"pods": n, "new_capacity": C // 2, "entries_evicted": int(evicted), "ms": 1e3 * dt,
                       "lru_entries_after": int(gpu.index_stats().lru_entries)})
        gpu.close()

    out = {
        "mode": "per-endpoint LRU capacities: churn (pick + indexer.Add per decision, LRUs filled first) and resize time",
        "workload": f"cfg{args.cfg}: {R} req/step x {E} endpoints x {wl.T}-token prompts, lruCapacityPerServer {C}",
        "card (name, power limit, SM clock, max SM clock)": {"before": card_before, "after": card()},
        "steps_timed": args.steps - max(1, args.oracle_steps), "churn": churn,
        "hetero_capacities": {str(C): third, str(C // 2): third, str((C + 3) // 4): E - 2 * third},
        "resize": resize,
        "lib": os.environ.get("FI_EPP_LIB", "default"),
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
