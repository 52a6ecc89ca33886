#!/usr/bin/env python
"""Early-exit hashing (hash_kernels.cu "early exit") at cfg 3 and cfg 2, on bench.py's KV-event-fed index
(lru_capacity == 0, chain order).  Per configuration, from profiled stream-ordered device picks:
  - hashed_blocks per request (fi_epp_stats, blocks whose prompt bytes hash_chain read) against N_probe per request
    (probed_blocks: matched rows + the miss, the blocks a pick needs) and the prompt's n_blocks;
  - hash_chain time (CUDA events around the kernel, profiling on) with early exit and with whole chains (the same
    call with chains_out);
  - prompt bytes read (block_bytes * hashed_blocks) over that time, against the HBM peak bench.py uses.
Without early exit the prompt bytes are block_bytes * n_blocks per request, bench.py's 4 * T.  The card's name,
power limit and SM clock are read in the same run.

    python tools/bench_early_exit.py [--cfgs 3,2] [--steps 8]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def profiled(sc, steps, with_chains):
    """-> (hash_chain ms per call, hashed blocks per call, probed blocks per call) over `steps` stream-ordered picks"""
    import torch

    wl, pk = sc.wl, sc.picker
    d_chain = torch.zeros(wl.R * wl.max_blocks, dtype=torch.int64, device="cuda") if with_chains else None
    for warm in (True, False):
        pk.reset_stats()
        pk.set_profiling(not warm)
        for i in range(2 if warm else steps):
            b = i % sc.nb
            pk.pick_batch_device(sc.d_tok[b].data_ptr(), sc.d_off[b].data_ptr(), sc.d_h0.data_ptr(), wl.R, wl.R * wl.T * 4,
                                 sc.d_out.data_ptr(), d_chain.data_ptr() if with_chains else 0, sc.stream)
        torch.cuda.synchronize()
    st = pk.stats()
    pk.set_profiling(False)
    return st.ms_hash_blocks / max(st.n_hash_blocks, 1), st.hashed_blocks / steps, st.probed_blocks / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfgs", default="3,2")
    ap.add_argument("--steps", type=int, default=8)
    args = ap.parse_args()

    import torch

    import bench

    if not torch.cuda.is_available():
        raise SystemExit("bench_early_exit needs a CUDA device")
    peak, peak_src = bench.measured_peak_gbs()
    out = {"card": card(), "hbm_peak_gbs": peak, "hbm_peak_source": peak_src, "configs": {}}
    for cfg in (int(c) for c in args.cfgs.split(",")):
        sargs = types.SimpleNamespace(batches=2, churn_rounds=0)
        sc = bench.Scenario(sargs, cfg, "replicas", 0, 1, 0).build()
        wl = sc.wl
        ms_early, hashed, probed = profiled(sc, args.steps, with_chains=False)
        ms_full, hashed_full, _ = profiled(sc, args.steps, with_chains=True)
        nbytes = hashed * wl.block_bytes
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        rec = {
            "R": wl.R, "block_bytes": wl.block_bytes, "n_blocks": wl.n_blocks,
            # early exit runs in half-SM tiles only: smaller batches hash whole chains in both passes
            "early_exit_tiles": wl.R > 64 * sms,
            "n_probe_per_request": probed / wl.R,
            "hashed_blocks_per_request": hashed / wl.R,
            "hash_chain_ms_early": ms_early,
            "hash_chain_ms_whole_chains": ms_full,
            "prompt_mb_read_early": nbytes / 1e6,
            "prompt_mb_read_whole_chains": hashed_full * wl.block_bytes / 1e6,
            "early_gbs": nbytes / (ms_early * 1e-3) / 1e9,
            "early_frac_of_peak": nbytes / (ms_early * 1e-3) / 1e9 / peak,
            "whole_chains_gbs": hashed_full * wl.block_bytes / (ms_full * 1e-3) / 1e9,
        }
        out["configs"][f"cfg{cfg}"] = rec
        print(f"cfg{cfg}: hashed {rec['hashed_blocks_per_request']:.1f} blocks/request (N_probe "
              f"{rec['n_probe_per_request']:.1f}, n {wl.n_blocks}); hash_chain {ms_early * 1e3:.1f} us early, "
              f"{ms_full * 1e3:.1f} us whole chains; {rec['early_gbs']:.0f} GB/s of prompt = "
              f"{rec['early_frac_of_peak']:.2f} of {peak:.0f} GB/s", file=sys.stderr)
        sc.close()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
