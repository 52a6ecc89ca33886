#!/usr/bin/env python
"""Cost of the ranked pick (fi_epp_pick_batch_device_ranked, docs/SPEC.md S.6a) against the single pick.

The stream-ordered device call is timed with CUDA events on the bench.py workload, for the single pick and the ranked
pick at k = 1, 4 and 16, and on a second handle whose profiles also carry a lora-affinity-scorer (the single LoRA pick
and the ranked pick at k = 4).  The variants are alternated round by round, so clock or thermal drift hits them all
alike; the median, min and max per variant are reported.  The card's name and power limit are read in the same run.

    python tools/bench_ranked.py [--cfg 3] [--rounds 30]
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=30)
    args = ap.parse_args()

    import torch

    from fusioninfer_b200 import EndpointPicker, _abi, make_config, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_ranked needs a CUDA device")
    wl = synth.baseline_workload(args.cfg)
    profiles, pd = synth.baseline_profiles(args.cfg)
    lora_profiles = [dict(p, scorers=list(p["scorers"]) + [(_abi.FI_SCORER_LORA, 10)]) for p in profiles]
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    R, P = wl.R, len(profiles)
    handles = {}
    for name, profs in (("plain", profiles), ("lora", lora_profiles)):
        cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=R,
                          max_prompt_bytes=R * wl.T * 4, index_slots=slots, profiles=profs, pd=pd)
        g = EndpointPicker(cfg)
        g.update_endpoints(wl.endpoint_states())
        for ops in wl.index_ops():
            g.index_apply(ops)
        g.index_sync()
        handles[name] = g
    lora = np.zeros(wl.E, dtype=_abi.lora_dtype())
    lora["endpoint"] = np.arange(wl.E)
    lora["max_active"] = 4
    lora["n_active"] = 2
    lora["active"][:, 0] = 1000 + np.arange(wl.E) % 7
    lora["active"][:, 1] = 1000 + np.arange(wl.E) % 11
    handles["lora"].update_endpoints_lora(lora)

    s = torch.cuda.current_stream()
    tok, offs = wl.prompts(batch=0)
    d_tok = torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs.view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_ad = torch.from_numpy((1000 + np.arange(R) % 13).astype(np.int64)).cuda()
    d_out = torch.zeros(R * P * 16 * 16, dtype=torch.uint8, device="cuda")

    def run(variant):
        h, k = variant
        g = handles[h]
        if k == 0 and h == "plain":
            g.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_out.data_ptr(), 0,
                                s.cuda_stream)
        elif k == 0:
            rc = g._lib.fi_epp_pick_batch_device_lora(g._h, d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(),
                                                      d_ad.data_ptr(), R, tok.nbytes, d_out.data_ptr(), None, s.cuda_stream)
            assert rc == 0, rc
        else:
            g.pick_batch_device_ranked(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, k, d_out.data_ptr(),
                                       0, s.cuda_stream, d_ad.data_ptr() if h == "lora" else 0)

    variants = [("plain", 0), ("plain", 1), ("plain", 4), ("plain", 16), ("lora", 0), ("lora", 4)]
    for v in variants:  # warm-up: first launches, the ranked buffers, the variants' shared-memory opt-in
        for _ in range(3):
            run(v)
    torch.cuda.synchronize()
    times = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            run(v)
            b.record(s)
            b.synchronize()
            times[v].append(a.elapsed_time(b) * 1e3)
    res = {}
    for (h, k), t in times.items():
        name = ("lora " if h == "lora" else "") + ("single pick" if k == 0 else f"ranked k={k}")
        res[name] = {"median_us": float(np.median(t)), "min_us": float(min(t)), "max_us": float(max(t))}
    out = {
        "mode": "stream-ordered device call (hash + match), CUDA events, variants alternated",
        "workload": f"cfg{args.cfg}: {R} requests x {wl.E} endpoints, {P} profile(s)",
        "card": card(), "rounds": args.rounds, "results": res,
        "lib": os.environ.get("FI_EPP_LIB", "default"),
    }
    print(json.dumps(out), flush=True)
    for g in handles.values():
        g.close()


if __name__ == "__main__":
    main()
