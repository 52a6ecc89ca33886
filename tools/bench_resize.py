#!/usr/bin/env python
"""fi_epp_resize_pool at the cfg 3 scale: 1 024 endpoints, lruCapacityPerServer 31 250, device LRU.

Each run creates a handle at 1 024 endpoints and ages it with pick + indexer.Add steps (stream-ordered device picks,
fi_epp_index_add_chains of the picked endpoints' chains), then times three resizes, each one call on a host clock (the
call blocks until the new pool is in place):
  - 1 024 -> 1 000: the same row width and slots, so only the removal of 24 endpoints (then back to 1 024, untimed);
  - 1 024 -> 512: rows of 32 -> 16 words, half the slots: removal, index rebuild, device-LRU copy;
  - 512 -> 1 024: the way back.
--runs such runs.  A separate run traces one 1 024 -> 512 resize with torch.profiler for the kernel and copy times.  The
step times are of the pipelined pick (fi_epp_pick_submit_ex, CUDA events over --steps steps): the resized handle at 512
against a handle created at 512 and fed the same Adds with those to the dropped endpoints left out (alternated; their
picks must be bit-equal), and the 1 024-endpoint handle before the shrink.  The card's name, power limit and SM clock are
read in the same run.

    python tools/bench_resize.py [--runs 3] [--age-steps 6] [--steps 200]
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

    from fusioninfer_b200 import EndpointPicker, make_config, synth
    from fusioninfer_b200 import _abi as abi

    if not torch.cuda.is_available():
        raise SystemExit("bench_resize needs a CUDA device")
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

    def new_handle(E):
        cfg = make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=wl.lru_capacity,
                          max_batch=R, max_prompt_bytes=R * wl.T * 4, profiles=profiles, pd=pd)
        gpu = EndpointPicker(cfg)
        gpu.set_option("device_lru", 1)
        st = wl.endpoint_states()
        gpu.update_endpoints(st[st["endpoint"] < E])
        return gpu

    main_p = pd["decode"] if pd else 0
    P = len(profiles)

    def age(gpu, history=None, replay=None):
        """pick + Add steps; `history` records (endpoints, chains, nblocks); `replay` feeds recorded ones instead"""
        d_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
        d_ch = torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda")
        if replay is not None:
            for eps, ch, nb in replay:
                gpu.index_add_chains(eps, ch, nb)
            return
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
            if history is not None:
                history.append((eps, ch, nb))
        gpu.index_sync()

    def timed_resize(gpu, E):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        removed = gpu.resize_pool(E, count=True)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), int(removed)

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

    runs = []
    step = {}
    for run in range(args.runs):
        gpu = new_handle(1024)
        hist = []
        age(gpu, history=hist)
        st = gpu.index_stats()
        r = {"index_keys": int(st.used - st.tombstones), "lru_entries": int(st.lru_entries), "slots_1024": int(st.slots)}
        r["1024->1000_ms"], r["1024->1000_pairs"] = timed_resize(gpu, 1000)
        timed_resize(gpu, 1024)
        if run == 0:
            (step["1024"],), _ = step_ms([gpu], args.steps)
        r["1024->512_ms"], r["1024->512_pairs"] = timed_resize(gpu, 512)
        r["slots_512"] = int(gpu.index_stats().slots)
        if run == 0:
            fresh = new_handle(512)
            filt = []
            for eps, ch, nb in hist:
                e2 = eps.copy()
                e2[(e2 != abi.FI_NO_ENDPOINT) & (e2 >= 512)] = abi.FI_NO_ENDPOINT
                filt.append((e2, ch, nb))
            age(fresh, replay=filt)
            (step["512_resized"], step["512_fresh"]), (pa, pb) = step_ms([gpu, fresh], args.steps)
            step["512_picks_bit_equal"] = bool(pa.tobytes() == pb.tobytes())
            fresh.close()
        r["512->1024_ms"], _ = timed_resize(gpu, 1024)
        runs.append(r)
        gpu.close()
        print(f"[resize] run {run}: {r}", file=sys.stderr, flush=True)

    # kernel times of one 1 024 -> 512 resize, in a run of their own
    gpu = new_handle(1024)
    age(gpu)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gpu.resize_pool(512, count=True)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if re.search(r"index_rebuild|index_remove|lru_reset|Memcpy DtoD|Memset", ev.key):
            kern[ev.key[:60]] = {"count": ev.count, "ms_total": ev.device_time_total / 1e3}
    gpu.close()

    def spread(key):
        v = [r[key] for r in runs]
        return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}

    out = {
        "mode": "fi_epp_resize_pool on a cfg-3-scale handle (device LRU) aged by pick + Add steps",
        "workload": f"cfg3: lruCapacityPerServer {wl.lru_capacity}, {R}-request batches, {args.age_steps} aging steps",
        "card": card(),
        "resize_ms": {k: spread(k) for k in ("1024->1000_ms", "1024->512_ms", "512->1024_ms")},
        "runs": runs,
        "kernels_1024_to_512": kern,
        "pipelined_step_ms": step,
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
