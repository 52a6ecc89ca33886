#!/usr/bin/env python
"""Index snapshots (fi_epp_snapshot_save / fi_epp_snapshot_load) at the cfg 3 scale: 1 024 endpoints,
lruCapacityPerServer 31 250, device LRU.

A source handle is aged with pick + indexer.Add steps (stream-ordered device picks, fi_epp_index_add_chains of the picked
endpoints' chains).  Then, --runs times each: its snapshot is saved into a pageable numpy buffer, and loaded into a
second handle (created with a smaller LRU table, fed the same endpoint states), each call on a host clock (both block).
Reported: the blob's size and counts, the save and load call times (median and range), the device-side kernels and
copies of one save and one load (torch.profiler, in a pass of its own), and the pipelined pick step
(fi_epp_pick_submit_ex, CUDA events over --steps steps) on the source and the loaded handle, alternated in one run, whose
picks must be bit-equal.  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_snapshot.py [--runs 3] [--age-steps 6] [--steps 200]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

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
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--age-steps", type=int, default=6)
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from fusioninfer_b200 import EndpointPicker, make_config, snapshot_info, synth
    from fusioninfer_b200 import _abi as abi

    if not torch.cuda.is_available():
        raise SystemExit("bench_snapshot needs a CUDA device")
    PICK = abi.np_dtypes()[0]
    wl = synth.baseline_workload(3)
    profiles, pd = synth.baseline_profiles(3)
    R = wl.R
    s = torch.cuda.current_stream()
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    batches = []
    for b in range(2):
        tok, offs = wl.prompts(batch=200 + b)
        batches.append((torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda(), torch.from_numpy(offs.view(np.int64)).cuda(),
                        tok.nbytes))
    states = wl.endpoint_states()

    def new_handle(table_slots=0):
        cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=wl.lru_capacity,
                          max_batch=R, max_prompt_bytes=R * wl.T * 4, profiles=profiles, pd=pd)
        gpu = EndpointPicker(cfg)
        gpu.set_option("device_lru", 1)
        if table_slots:
            gpu.set_option("lru_table_slots", table_slots)
        gpu.update_endpoints(states)
        return gpu

    main_p = pd["decode"] if pd else 0
    P = len(profiles)

    def age(gpu):
        d_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
        d_ch = torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda")
        for k in range(args.age_steps):
            d_tok, d_off, nbytes = batches[k % 2]
            gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, d_out.data_ptr(),
                                  d_ch.data_ptr(), s.cuda_stream)
            torch.cuda.synchronize()
            got = d_out.cpu().numpy().view(PICK).reshape(R, P)
            eps = np.ascontiguousarray(got[:, main_p]["endpoint"])
            nb = np.ascontiguousarray(got[:, main_p]["n_blocks"]).astype(np.uint32)
            ch = d_ch.cpu().numpy().view(np.uint64).reshape(R, wl.max_blocks).copy()
            gpu.index_add_chains(eps, ch, nb)
        gpu.index_sync()

    def step_ms(handles, steps):
        """pipelined submit_ex steps, the handles alternated per block of 20 steps; -> ms per step each, last picks"""
        outs = [torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda") for _ in handles]
        tot = [0.0] * len(handles)
        n = [0] * len(handles)
        for blk in range(2 + steps // 20):
            for i, g in enumerate(handles):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                for k in range(20):
                    d_tok, d_off, nbytes = batches[k % 2]
                    t = g.pick_submit_ex(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, outs[i].data_ptr(),
                                         stream=s.cuda_stream)
                g.pick_wait_batch(t, s.cuda_stream)
                b.record(s)
                b.synchronize()
                if blk >= 2:  # two warm-up blocks
                    tot[i] += a.elapsed_time(b)
                    n[i] += 20
        return [tot[i] / n[i] for i in range(len(handles))], [o.cpu().numpy().view(PICK).reshape(R, P) for o in outs]

    src = new_handle()
    age(src)
    st = src.index_stats()
    dst = new_handle(table_slots=1 << 18)
    save_ms, load_ms = [], []
    blob = None
    for run in range(args.runs):
        del blob
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        blob = src.save_snapshot()
        save_ms.append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        dst.load_snapshot(blob)
        torch.cuda.synchronize()
        load_ms.append(1e3 * (time.perf_counter() - t0))
        print(f"[snapshot] run {run}: save {save_ms[-1]:.1f} ms, load {load_ms[-1]:.1f} ms", file=sys.stderr, flush=True)
    info = snapshot_info(blob)
    same_bytes = bool(dst.save_snapshot().tobytes() == blob.tobytes())

    # device time of one save and one load, in a pass of its own
    kern = {}
    for what, fn in (("save", lambda: src.save_snapshot()), ("load", lambda: dst.load_snapshot(blob))):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern[what] = {}
        for ev in prof.key_averages():
            if re.search(r"snap|lru_dump|lru_load|Memcpy|Memset", ev.key) and ev.device_time_total > 0:
                kern[what][ev.key[:60]] = {"count": ev.count, "ms_total": round(ev.device_time_total / 1e3, 3)}

    (step_src, step_dst), (pa, pb) = step_ms([src, dst], args.steps)

    def spread(v):
        return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}

    out = {
        "mode": "fi_epp_snapshot_save / _load of a cfg-3-scale handle (device LRU) aged by pick + Add steps",
        "workload": f"cfg3: lruCapacityPerServer {wl.lru_capacity}, {R}-request batches, {args.age_steps} aging steps",
        "card": card(),
        "source": {"index_keys": int(st.used - st.tombstones), "tombstones": int(st.tombstones), "lru_entries": int(st.lru_entries),
                   "slots": int(st.slots)},
        "blob": {"bytes": int(info.bytes), "n_nodes": int(info.n_nodes), "n_lru": int(info.n_lru), "pairs": int(info.pairs)},
        "save_ms": spread(save_ms),
        "load_ms": spread(load_ms),
        "save_of_load_same_bytes": same_bytes,
        "device_time": kern,
        "pipelined_step_ms": {"source": step_src, "loaded": step_dst, "picks_bit_equal": bool(pa.tobytes() == pb.tobytes())},
    }
    print(json.dumps(out), flush=True)
    src.close()
    dst.close()


if __name__ == "__main__":
    main()
