#!/usr/bin/env python
"""Snapshot captures (fi_epp_snapshot_capture / _read / _free) against the blocking save, at the cfg 3 scale: 1 024
endpoints, lruCapacityPerServer 31 250, device LRU, aged by pick + Add steps as in tools/bench_snapshot.py.

Reported, with the card's name, power limit and SM clock read in the same run:
- call times: capture, read and free on a host clock, median and range of --runs runs with nothing else running, and
  the device time of one capture's kernels and copies (torch.profiler, in a pass of its own);
- the stall: one thread issues stream-ordered device picks back to back (each call timed on the host until its stream
  is synchronised) while the main thread does a blocking save, then a capture + read + free, alternated --runs times.
  For each window: the picks completed, their longest and p99 latency; also a quiet window with no snapshot.  Every
  pick is compared with the picks of a run without snapshots;
- the update cost: an Add (fi_epp_index_add_chains) issued right after a capture, against the same Add without one.

    python tools/bench_snapshot_capture.py [--runs 3] [--age-steps 6]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from tools.bench_snapshot import card  # noqa: E402


def spread(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} if v else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--age-steps", type=int, default=6)
    ap.add_argument("--quiet-ms", type=float, default=150.0, help="pause between the windows of the stall test")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from fusioninfer_b200 import EndpointPicker, make_config, synth
    from fusioninfer_b200 import _abi as abi

    if not torch.cuda.is_available():
        raise SystemExit("bench_snapshot_capture needs a CUDA device")
    PICK = abi.np_dtypes()[0]
    wl = synth.baseline_workload(3)
    profiles, pd = synth.baseline_profiles(3)
    R, P = wl.R, len(profiles)
    main_p = pd["decode"] if pd else 0
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    batches = []
    for b in range(2):
        tok, offs = wl.prompts(batch=200 + b)
        batches.append((torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda(), torch.from_numpy(offs.view(np.int64)).cuda(),
                        tok.nbytes))
    cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=wl.lru_capacity,
                      max_batch=R, max_prompt_bytes=R * wl.T * 4, profiles=profiles, pd=pd)
    gpu = EndpointPicker(cfg)
    gpu.set_option("device_lru", 1)
    gpu.update_endpoints(wl.endpoint_states())
    s = torch.cuda.current_stream()
    d_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    d_ch = torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda")
    last_add = None
    for k in range(args.age_steps):
        d_tok, d_off, nbytes = batches[k % 2]
        gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, d_out.data_ptr(), d_ch.data_ptr(),
                              s.cuda_stream)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy().view(PICK).reshape(R, P)
        eps = np.ascontiguousarray(got[:, main_p]["endpoint"])
        nb = np.ascontiguousarray(got[:, main_p]["n_blocks"]).astype(np.uint32)
        ch = d_ch.cpu().numpy().view(np.uint64).reshape(R, wl.max_blocks).copy()
        gpu.index_add_chains(eps, ch, nb)
        last_add = (eps, ch, nb)
    gpu.index_sync()
    st = gpu.index_stats()

    # ---- call times, nothing else running
    cap_ms, read_ms, free_ms, save_ms = [], [], [], []
    nbytes_blob = 0
    for run in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c = gpu.capture_snapshot()
        t1 = time.perf_counter()
        blob = c.read()
        t2 = time.perf_counter()
        c.close()
        t3 = time.perf_counter()
        cap_ms.append(1e3 * (t1 - t0))
        read_ms.append(1e3 * (t2 - t1))
        free_ms.append(1e3 * (t3 - t2))
        nbytes_blob = len(blob)
        t0 = time.perf_counter()
        saved = gpu.save_snapshot()
        save_ms.append(1e3 * (time.perf_counter() - t0))
        same = saved.tobytes() == blob.tobytes()
        del blob, saved
        print(f"[capture] run {run}: capture {cap_ms[-1]:.2f} ms, read {read_ms[-1]:.1f} ms, free {free_ms[-1]:.2f} ms, "
              f"save {save_ms[-1]:.1f} ms, same bytes {same}", file=sys.stderr, flush=True)
        assert same, "a capture's read differs from the save"

    # device time of one capture + read, in a pass of its own
    kern = {}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        c = gpu.capture_snapshot()
        c.read()
        c.close()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if re.search(r"snap|lru_dump|Memcpy|Memset", ev.key) and ev.device_time_total > 0:
            kern[ev.key[:60]] = {"count": ev.count, "ms_total": round(ev.device_time_total / 1e3, 3)}

    # ---- the stall: picks back to back on a thread of their own
    def pick_once(stream, out):
        d_tok, d_off, nbytes = batches[0]
        gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, out.data_ptr(), 0, stream.cuda_stream)
        stream.synchronize()

    ps = torch.cuda.Stream()
    p_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    for _ in range(20):
        pick_once(ps, p_out)
    ref = p_out.cpu().numpy().copy()  # the picks of a run without snapshots
    log, stop, mismatches = [], threading.Event(), [0]

    def picker():
        with torch.cuda.stream(ps):
            while not stop.is_set():
                t0 = time.perf_counter()
                pick_once(ps, p_out)
                t1 = time.perf_counter()
                if not np.array_equal(p_out.cpu().numpy(), ref):
                    mismatches[0] += 1
                log.append((t0, t1))

    windows = []
    th = threading.Thread(target=picker)
    th.start()
    time.sleep(args.quiet_ms / 1e3)
    for run in range(args.runs):
        t0 = time.perf_counter()
        time.sleep(args.quiet_ms / 1e3)
        windows.append(("quiet", t0, time.perf_counter()))
        t0 = time.perf_counter()
        gpu.save_snapshot()
        windows.append(("save", t0, time.perf_counter()))
        time.sleep(args.quiet_ms / 1e3)
        t0 = time.perf_counter()
        c = gpu.capture_snapshot()
        t1 = time.perf_counter()
        c.read()
        c.close()
        windows.append(("capture_call", t0, t1))
        windows.append(("capture_read_free", t0, time.perf_counter()))
        time.sleep(args.quiet_ms / 1e3)
    stop.set()
    th.join()

    def window_stats(t0, t1):
        # picks that overlap the window (a pick stalled by the window ends after it starts)
        lat = [1e3 * (b - a) for a, b in log if b >= t0 and a <= t1]
        done = sum(1 for a, b in log if t0 <= b <= t1)
        return {"window_ms": 1e3 * (t1 - t0), "picks_completed": done, "picks_overlapping": len(lat),
                "max_ms": max(lat) if lat else None, "p99_ms": float(np.percentile(lat, 99)) if lat else None}

    stall = {}
    for what, t0, t1 in windows:
        stall.setdefault(what, []).append(window_stats(t0, t1))

    # ---- the update cost: an Add right after a capture, and the same Add alone
    eps, ch, nb = last_add
    add_ms = {"after_capture": [], "alone": []}
    for run in range(args.runs):
        for what in ("alone", "after_capture"):
            gpu.index_sync()
            torch.cuda.synchronize()
            c = gpu.capture_snapshot() if what == "after_capture" else None
            t0 = time.perf_counter()
            gpu.index_add_chains(eps, ch, nb)
            gpu.index_sync()
            add_ms[what].append(1e3 * (time.perf_counter() - t0))
            if c is not None:
                c.close()

    out = {
        "mode": "fi_epp_snapshot_capture / _read / _free against fi_epp_snapshot_save, cfg-3-scale handle (device LRU) aged by pick + Add steps",
        "workload": f"cfg3: lruCapacityPerServer {wl.lru_capacity}, {R}-request batches, {args.age_steps} aging steps",
        "card": card(),
        "source": {"index_keys": int(st.used - st.tombstones), "lru_entries": int(st.lru_entries), "slots": int(st.slots)},
        "blob_bytes": nbytes_blob,
        "call_ms": {"capture": spread(cap_ms), "read": spread(read_ms), "free": spread(free_ms), "save": spread(save_ms)},
        "capture_device_time": kern,
        "stall": stall,
        "picks_total": len(log),
        "picks_differing_from_the_run_without_snapshots": mismatches[0],
        "add_ms": {k: spread(v) for k, v in add_ms.items()},
    }
    print(json.dumps(out), flush=True)
    gpu.close()


if __name__ == "__main__":
    main()
