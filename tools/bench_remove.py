#!/usr/bin/env python
"""fi_epp_index_remove_endpoints (upstream indexer.RemovePod) on a full index.

The index is built at capacity through the device LRU (every endpoint's LRU full, as in tools/bench_churn.py), aged
by a few pick + indexer.Add steps, and then endpoints are removed: 1 (one 32-byte sector of every row), 32 (one
whole row word) and all of them.  Each removal is timed once — it changes the index — after a warm-up removal of
each sweep shape.  Per removal it reports:
  - the call (host clock; pairs_removed makes it block until applied),
  - the kernels (torch.profiler: index_remove_words_kernel / index_remove_rows_kernel, lru_reset_kernel),
  - the sweep's sector bytes (live nodes x 32-byte sectors holding a listed word) over its kernel time,
  - the stream-ordered pick right after the removal, against the median pick that follows none.
The card's name and power limit are read in the same run.

    python tools/bench_remove.py [--cfg 3] [--age-steps 4]
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def sectors(eps, ep_begin=0):
    """32-byte row sectors (8 words) holding a listed endpoint"""
    return len({((e - ep_begin) >> 5) >> 3 for e in eps})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--age-steps", type=int, default=4)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from fusioninfer_b200 import EndpointPicker, make_config, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_remove needs a CUDA device")
    wl = synth.baseline_workload(args.cfg)
    profiles, pd = synth.baseline_profiles(args.cfg)
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    cfg = make_config(num_endpoints=wl.E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, lru_capacity=wl.lru_capacity,
                      max_batch=wl.R, max_prompt_bytes=wl.R * wl.T * 4, index_slots=slots, profiles=profiles, pd=pd)
    gpu = EndpointPicker(cfg)
    gpu.set_option("device_lru", 1)
    gpu.update_endpoints(wl.endpoint_states())

    # ---- the index at capacity through the LRUs (filler first, then the shared group chains), then aged
    t0 = time.time()
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
        gpu.index_add_chains(ee, ch, (ch != 0).sum(axis=1).astype(np.uint32))
    R, P = wl.R, gpu.n_profiles
    main_p = cfg.pd_decode_profile if cfg.pd_enabled else 0
    s = torch.cuda.current_stream()
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda")
    batches = []
    for b in range(2):
        tok, offs = wl.prompts(batch=100 + b)
        batches.append((torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda(), torch.from_numpy(offs.view(np.int64)).cuda(),
                        tok.nbytes))

    def pick(k):
        d_tok, d_off, nbytes = batches[k % 2]
        gpu.pick_batch_device(d_tok.data_ptr(), d_off.data_ptr(), d_h0.data_ptr(), R, nbytes, d_out.data_ptr(), 0, s.cuda_stream)

    def timed_pick(k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        pick(k)
        b.record(s)
        b.synchronize()
        return a.elapsed_time(b)

    for step in range(args.age_steps):
        pick(step)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy().view(np.dtype([("endpoint", "<u4"), ("match_blocks", "<u2"), ("n_blocks", "<u2"),
                                                 ("score", "<f8")])).reshape(R, P)
        gpu.index_add_chains_device(np.ascontiguousarray(got[:, main_p]["endpoint"]), 0, 0,
                                    np.ascontiguousarray(got[:, main_p]["n_blocks"]).astype(np.uint32), s.cuda_stream)
    gpu.index_sync()
    st0 = gpu.index_stats()
    print(f"[remove] index: {st0.used} keys, {st0.lru_entries} LRU entries, built in {time.time() - t0:.1f}s", file=sys.stderr)
    for k in range(3):
        timed_pick(k)
    base_picks = [timed_pick(k) for k in range(6)]

    # ---- warm-up: one removal of each sweep shape (first launches load the kernels)
    W = 1
    while W * 32 < wl.E:
        W *= 2
    warm = [[wl.E - 1], [e for e in (1, 257, 513, 769) if e < wl.E]]
    for eps in warm:
        gpu.remove_endpoints(eps, count=True)
    cases = [("1 endpoint", [2]), ("32 endpoints (one row word)", list(range(32, 64))), (f"all {wl.E} endpoints", list(range(wl.E)))]
    results = []
    for name, eps in cases:
        used = int(gpu.index_stats().used)
        nodes = min(used, int(st0.slots)) + 2
        nsec = sectors(eps)
        whole_rows = W >= 4 and nsec == (W + 7) // 8
        lru_before = int(gpu.index_stats().lru_entries)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            c0 = time.perf_counter()
            removed = gpu.remove_endpoints(eps, count=True)
            call_ms = 1e3 * (time.perf_counter() - c0)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "remove" in ev.key or "lru_reset" in ev.key:
                short = "sweep" if "remove" in ev.key else "lru_reset"
                kname = re.search(r"index_remove_\w+|lru_reset_kernel", ev.key)
                kern[short] = {"kernel": kname.group(0) if kname else ev.key, "ms": ev.device_time_total / 1e3 / max(ev.count, 1)}
        pick_after = timed_pick(0)
        sweep_ms = kern.get("sweep", {}).get("ms")
        # per-word shape: one sector per listed sector and node; whole rows: the row (W/8 sectors, or 16 B when W = 4)
        nbytes = nodes * (nsec * 32 if not whole_rows else max(W * 4, 16))
        results.append({
            "removal": name, "shape": "whole_rows" if whole_rows else "words", "pairs_removed": int(removed),
            "lru_entries_dropped": lru_before - int(gpu.index_stats().lru_entries),
            "call_ms": call_ms, "kernels": kern, "nodes_swept": nodes, "sector_bytes": nbytes,
            "sweep_GBps": None if not sweep_ms else nbytes / (sweep_ms * 1e-3) / 1e9,
            "pick_ms_after": pick_after,
        })
    out = {
        "mode": "fi_epp_index_remove_endpoints on an index at capacity (device LRU), aged by pick + Add steps",
        "workload": f"cfg{args.cfg}: {wl.E} endpoints x lruCapacityPerServer {wl.lru_capacity}, {R}-request picks",
        "card": card(), "index_keys": int(st0.used), "index_slots": int(st0.slots), "row_words": W,
        "pick_ms_after_no_removal": {"median": float(np.median(base_picks)), "min": float(min(base_picks)), "max": float(max(base_picks))},
        "removals": results,
        "lib": os.environ.get("FI_EPP_LIB", "default"),
    }
    print(json.dumps(out), flush=True)
    gpu.close()


if __name__ == "__main__":
    main()
