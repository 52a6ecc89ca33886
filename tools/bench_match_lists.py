#!/usr/bin/env python
"""Cost of fi_epp_match_lists (docs/SPEC.md S.3b) against the dense fi_epp_match_counts and the single pick, on
bench.py's warmed synthetic index.

For each config, fi_epp_match_lists_device, fi_epp_match_counts_device and fi_epp_pick_batch_device run on the same
device inputs, alternated call by call and timed with CUDA events, for at least --seconds of timed work per variant.
The host calls fi_epp_match_lists, fi_epp_match_counts and fi_epp_pick_batch (pinned prompt and result buffers) are
timed, alternated, with a host clock around the blocking call.  A profiled pass reads each device variant's match-kernel
time (ms_match_pick per call) and, for the lists, the pack step's (ms_other per call) from fi_epp_stats.  Printed per
variant: µs per batch (median, min, max), requests/s, result bytes per batch; for the lists, entries per request (mean,
p99, max).  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_match_lists.py [--cfgs 2 3] [--seconds 2]
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def bench_cfg(cfg_id: int, seconds: float):
    import torch

    from fusioninfer_b200 import EndpointPicker, PinnedBuffer, make_config, synth

    wl = synth.baseline_workload(cfg_id)
    profiles, pd = synth.baseline_profiles(cfg_id)
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    R, P, E = wl.R, len(profiles), wl.E
    cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=R,
                      max_prompt_bytes=R * wl.T * 4, index_slots=slots, profiles=profiles, pd=pd)
    g = EndpointPicker(cfg)
    g.update_endpoints(wl.endpoint_states())
    for ops in wl.index_ops():
        g.index_apply(ops)
    g.index_sync()

    s = torch.cuda.current_stream()
    tok, offs = wl.prompts(batch=0)
    d_tok = torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda()
    d_off = torch.from_numpy(offs.view(np.int64)).cuda()
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    d_counts = torch.zeros(R * E, dtype=torch.int16, device="cuda")
    d_nb = torch.zeros(R, dtype=torch.int32, device="cuda")

    cap = R * E
    d_loff = torch.zeros(R + 1, dtype=torch.int64, device="cuda")
    d_ent = torch.zeros(cap * 8, dtype=torch.uint8, device="cuda")

    def pick():
        g.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_out.data_ptr(), 0,
                            s.cuda_stream)

    def counts():
        g.match_counts_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_counts.data_ptr(),
                              d_nb.data_ptr(), 0, s.cuda_stream)

    def lists():
        g.match_lists_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, tok.nbytes, d_loff.data_ptr(),
                             d_ent.data_ptr(), cap, d_nb.data_ptr(), 0, s.cuda_stream)

    variants = {"match_lists_device": lists, "match_counts_device": counts, "pick_batch_device": pick}
    for f in variants.values():  # warm-up: first launches, the variants' shared-memory opt-in, the lists' scratch
        for _ in range(5):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    spent = 0.0
    while spent < len(variants) * seconds:  # alternate, call by call, until each has `seconds` of timed work
        for k, f in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            f()
            b.record(s)
            b.synchronize()
            t = a.elapsed_time(b) * 1e-3
            times[k].append(t)
            spent += t
    loff = d_loff.cpu().numpy().view(np.uint64)
    lens = np.diff(loff).astype(np.float64)
    total = int(loff[-1])

    # the host calls: pinned prompts in, pinned results out
    pin_tok = PinnedBuffer(tok.nbytes)
    pin_tok.array(np.uint8)[:] = tok.reshape(-1).view(np.uint8)
    pin_cnt = PinnedBuffer(R * E * 2)
    pin_ent = PinnedBuffer(cap * 8)
    pin_loff = PinnedBuffer((R + 1) * 8)
    pin_pick = PinnedBuffer(R * P * 16)
    h0 = np.full(R, wl.h0, dtype=np.uint64)
    nb = np.zeros(R, dtype=np.uint32)

    def host_lists():
        rc = g._lib.fi_epp_match_lists(g._h, pin_tok.ptr, offs.ctypes.data, h0.ctypes.data, R, pin_loff.ptr,
                                       pin_ent.ptr, cap, nb.ctypes.data, None)
        assert rc == 0, rc

    def host_counts():
        rc = g._lib.fi_epp_match_counts(g._h, pin_tok.ptr, offs.ctypes.data, h0.ctypes.data, R, pin_cnt.ptr,
                                        nb.ctypes.data, None)
        assert rc == 0, rc

    def host_pick():
        rc = g._lib.fi_epp_pick_batch(g._h, pin_tok.ptr, offs.ctypes.data, h0.ctypes.data, R, pin_pick.ptr, None)
        assert rc == 0, rc

    hosts = {"match_lists (host, pinned)": host_lists, "match_counts (host, pinned)": host_counts,
             "pick_batch (host, pinned)": host_pick}
    for f in hosts.values():
        for _ in range(3):
            f()
    for k in hosts:
        times[k] = []
    t_end = time.perf_counter() + len(hosts) * seconds
    while time.perf_counter() < t_end:
        for k, f in hosts.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)

    # profiled pass: the match kernel's and the pack step's device time per call
    kernel_us = {}
    for k, f in variants.items():
        g.reset_stats()
        g.set_profiling(True)
        for _ in range(20):
            f()
        torch.cuda.synchronize()
        st = g.stats()
        g.set_profiling(False)
        kernel_us[k] = {"match_kernel_us": st.ms_match_pick * 1e3 / max(st.n_match_pick, 1)}
        if k == "match_lists_device":
            kernel_us[k]["pack_us"] = st.ms_other * 1e3 / 20

    result_bytes = {"lists": (R + 1) * 8 + total * 8, "counts": R * E * 2, "pick": R * P * 16}
    res = {}
    for k, t in times.items():
        med = float(np.median(t))
        res[k] = {"median_us": med * 1e6, "min_us": float(min(t)) * 1e6, "max_us": float(max(t)) * 1e6,
                  "calls": len(t), "requests_per_s": R / med,
                  "result_bytes": result_bytes[next(n for n in result_bytes if n in k)]}
        res[k].update(kernel_us.get(k, {}))
    for b in (pin_tok, pin_cnt, pin_ent, pin_loff, pin_pick):
        b.free()
    g.close()
    return {"workload": f"cfg{cfg_id}: {R} requests x {E} endpoints, {P} profile(s)", "results": res,
            "entries_per_request": {"mean": float(lens.mean()), "p99": float(np.percentile(lens, 99)),
                                    "max": int(lens.max()), "empty_share": float((lens == 0).mean())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfgs", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--seconds", type=float, default=2.0)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_match_lists needs a CUDA device")
    out = {"mode": "stream-ordered device calls alternated (CUDA events); host call timed around the blocking call",
           "card": card(), "seconds_per_variant": args.seconds,
           "configs": [bench_cfg(c, args.seconds) for c in args.cfgs]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
