#!/usr/bin/env python
"""Cost of the subset pick (fi_epp_pick_batch_device_subset, docs/SPEC.md S.5a) against the single and ranked picks.

The stream-ordered device call is timed with CUDA events on the bench.py workload for: the single pick, the ranked
pick at k = 1, the subset call with NULL subsets (k = 1), random per-request subsets of 8, 64 and all endpoints at
k = 1, and 64-endpoint subsets at k = 4.  The variants are alternated round by round, so clock or thermal drift hits
them all alike; the median, min and max per variant are reported.  The card's name, power limit and SM clock are read
in the same run.  After timing, each variant's picks of the first --check requests are compared bit for bit with the
CPU oracle's subset pick (tests/ext_oracle.cpp, built by `make`).

    python tools/bench_subset.py [--cfg 3] [--rounds 30] [--check 512]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--check", type=int, default=512, help="requests per variant checked against the oracle (0: none)")
    args = ap.parse_args()
    card_before = card()

    import torch

    from fusioninfer_b200 import EndpointPicker, make_config, subset_bitsets, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_subset needs a CUDA device")
    wl = synth.baseline_workload(args.cfg)
    profiles, pd = synth.baseline_profiles(args.cfg)
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    R, P, E = wl.R, len(profiles), wl.E
    cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=R,
                      max_prompt_bytes=R * wl.T * 4, index_slots=slots, profiles=profiles, pd=pd)
    g = EndpointPicker(cfg)
    states = wl.endpoint_states()
    g.update_endpoints(states)
    for ops in wl.index_ops():
        g.index_apply(ops)
    g.index_sync()

    rng = np.random.default_rng(7)
    subsets = {}
    for size in (8, 64):
        pick = np.argsort(rng.random((R, E)), axis=1)[:, :size]
        subsets[size] = subset_bitsets(list(pick), E)
    subsets[E] = subset_bitsets([None] * R, E)
    d_sub = {n: torch.from_numpy(s.view(np.int32)).cuda() for n, s in subsets.items()}

    s = torch.cuda.current_stream()
    tok, offs = wl.prompts(batch=0)
    d_tok = torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs.view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")

    # (name, kind, subset size or None, k)
    variants = [("single pick", "single", None, 1), ("ranked k=1", "ranked", None, 1), ("subset NULL k=1", "subset", None, 1),
                ("subset 8 k=1", "subset", 8, 1), ("subset 64 k=1", "subset", 64, 1), (f"subset {E} k=1", "subset", E, 1),
                ("subset 64 k=4", "subset", 64, 4)]
    d_out = {v[0]: torch.zeros(R * P * v[3] * 16, dtype=torch.uint8, device="cuda") for v in variants}

    def run(v):
        name, kind, size, k = v
        out = d_out[name].data_ptr()
        if kind == "single":
            g.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, out, 0, s.cuda_stream)
        elif kind == "ranked":
            g.pick_batch_device_ranked(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, k, out, 0,
                                       s.cuda_stream)
        else:
            g.pick_batch_device_subset(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, k, out,
                                       d_sub[size].data_ptr() if size else 0, 0, s.cuda_stream)

    for v in variants:  # warm-up: first launches, the result buffers, the variants' shared-memory opt-in
        for _ in range(3):
            run(v)
    torch.cuda.synchronize()
    times = {v[0]: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            run(v)
            b.record(s)
            b.synchronize()
            times[v[0]].append(a.elapsed_time(b) * 1e3)
    clock_after = card()
    res = {name: {"median_us": float(np.median(t)), "min_us": float(min(t)), "max_us": float(max(t))}
           for name, t in times.items()}

    checked = {}
    if args.check:
        from tests.ext_oracle import ExtOracle

        n = min(args.check, R)
        cpu = ExtOracle(cfg)
        cpu.update_endpoints(states)
        for ops in wl.index_ops():
            cpu.index_apply(ops)
        t, o = tok, offs[: n + 1]
        from fusioninfer_b200 import PICK_DTYPE

        for name, kind, size, k in variants:
            got = d_out[name].cpu().numpy().view(PICK_DTYPE)
            if kind == "single":
                got = got.reshape(R, P)[:n]
                want = cpu.pick_batch(t, o, wl.h0)
            else:
                got = got.reshape(R, P, k)[:n]
                want = cpu.pick_batch_subset(t, o, wl.h0, subsets[size][:n] if size else None, k)
            checked[name] = "bit-exact" if got.tobytes() == want.tobytes() else "MISMATCH"
        cpu.close()

    out = {
        "mode": "stream-ordered device call (hash + match), CUDA events, variants alternated",
        "workload": f"cfg{args.cfg}: {R} requests x {E} endpoints, {P} profile(s)",
        "card (name, power limit, SM clock, max SM clock)": {"before": card_before, "after": clock_after},
        "rounds": args.rounds, "results": res, "oracle_check": {"requests": min(args.check, R), "variants": checked},
        "lib": os.environ.get("FI_EPP_LIB", "default"),
    }
    print(json.dumps(out), flush=True)
    g.close()
    if any(v != "bit-exact" for v in checked.values()):
        raise SystemExit("picks differ from the oracle")


if __name__ == "__main__":
    main()
