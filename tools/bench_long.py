#!/usr/bin/env python
"""Picks over long prompts: max_blocks = M in {1023, 2047, 4095} at 1 024 endpoints (DESIGN.md §4.9).

Each M gets its own handle and index: 256 group prompts of M 64-byte blocks, endpoint e caching the whole chain of
group e % 256, inserted in chain order.  Request r copies a prefix of M/4 .. M blocks of group r % 256 and continues
with bytes of its own; every prompt is M blocks and a partial one.  M = 1023 runs match_pick_kernel, 2047 and 4095
match_window_kernel, which counts 1 024 blocks (one window) at a time.

Per M: µs per batch of the stream-ordered device pick (CUDA events) and of the pipelined submit (fi_epp_pick_submit_ex,
--inflight batches per wait), the match kernel's time per call and the rows it read (fi_epp_stats, a separate profiled
pass), rows read per µs.  Then the cost of the windowed kernel itself: the M = 1023 prompts through a handle with
max_blocks = 4095 (no boundary crossed) against the same prompts through max_blocks = 1023.  Last, the cost of one
window boundary on its own (`boundary` below): one handle, one index, cached runs just below and just above block
1 024.  The card's name, power limit and SM clock are
read in the same run.

    python tools/bench_long.py [--R 1024] [--seconds 2]
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

E, GROUPS, B = 1024, 256, 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def workload(M, R, seed=1):
    rng = np.random.default_rng(seed + M)
    T = M * B + B // 2
    groups = rng.integers(0, 256, size=(GROUPS, M * B), dtype=np.uint8)
    tok = rng.integers(0, 256, size=(R, T), dtype=np.uint8)
    keep = rng.integers(M // 4, M + 1, size=R)
    for r in range(R):
        tok[r, : keep[r] * B] = groups[r % GROUPS, : keep[r] * B]
    offs = np.arange(R + 1, dtype=np.uint64) * T
    return groups, tok.reshape(-1), offs


class Handle:
    def __init__(self, max_blocks, M, R, groups, tok, offs):
        import torch

        from fusioninfer_b200 import EndpointPicker, make_config, synth

        profiles, _ = synth.baseline_profiles(3)
        slots = 1 << 16
        while slots < 4 * GROUPS * M:
            slots *= 2
        cfg = make_config(num_endpoints=E, block_bytes=B, max_blocks=max_blocks, max_batch=max(R, GROUPS),
                          max_prompt_bytes=max(int(offs[-1]), groups.nbytes), index_slots=slots, profiles=profiles)
        self.g = g = EndpointPicker(cfg)
        from fusioninfer_b200 import _abi as abi

        _, op_dtype, ep_dtype = abi.np_dtypes()
        rng = np.random.default_rng(7)
        st = np.zeros(E, dtype=ep_dtype)
        st["endpoint"] = np.arange(E)
        st["kv_util"] = rng.random(E)
        st["queue_depth"] = rng.integers(0, 16, size=E)
        st["role_mask"] = abi.FI_ROLE_WORKER
        st["flags"] = abi.FI_ENDPOINT_ALIVE
        g.update_endpoints(st)
        goffs = np.arange(GROUPS + 1, dtype=np.uint64) * (M * B)
        chains, nb = g.hash_batch(groups.reshape(-1), goffs, np.zeros(GROUPS, dtype=np.uint64))
        assert (nb == min(M, max_blocks)).all()
        n = int(nb[0])
        for e0 in range(0, E, 16):  # endpoint e caches group e % GROUPS in chain order
            eps = np.arange(e0, e0 + 16)
            ops = np.zeros(16 * n, dtype=op_dtype)
            ops["hash"] = chains[eps % GROUPS, :n].reshape(-1)
            ops["endpoint"] = np.repeat(eps, n)
            ops["op"] = abi.FI_OP_SET
            g.index_apply(ops)
        g.index_sync()
        self.R, self.P = R, len(profiles)
        self.nbytes = int(offs[-1])
        self.d_tok = torch.from_numpy(tok.view(np.uint8)).cuda()
        self.d_off = torch.from_numpy(offs.view(np.int64)).cuda()
        self.d_h0 = torch.zeros(R, dtype=torch.int64, device="cuda")
        self.d_out = torch.zeros(R * self.P * 16, dtype=torch.uint8, device="cuda")

    def pick(self, s):
        self.g.pick_batch_device(self.d_tok.data_ptr(), self.d_off.data_ptr(), self.d_h0.data_ptr(), self.R, self.nbytes,
                                 self.d_out.data_ptr(), 0, s)

    def submit(self, s):
        return self.g.pick_submit_ex(self.d_tok.data_ptr(), self.d_off.data_ptr(), self.d_h0.data_ptr(), self.R,
                                     self.nbytes, self.d_out.data_ptr(), stream=s)

    def picks(self):
        return self.d_out.cpu().numpy().view([("endpoint", "<u4"), ("match_blocks", "<u2"), ("n_blocks", "<u2"),
                                              ("score", "<f8")]).reshape(self.R, self.P)


def timed(h, seconds, inflight):
    import torch

    s = torch.cuda.current_stream()
    for _ in range(5):
        h.pick(s.cuda_stream)
    torch.cuda.synchronize()
    ordered, spent = [], 0.0
    while spent < seconds:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        h.pick(s.cuda_stream)
        b.record(s)
        b.synchronize()
        ordered.append(a.elapsed_time(b) * 1e-3)
        spent += ordered[-1]
    piped, spent = [], 0.0
    while spent < seconds:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(inflight):
            t = h.submit(s.cuda_stream)
        h.g.pick_wait_batch(t, s.cuda_stream)
        b.record(s)
        b.synchronize()
        piped.append(a.elapsed_time(b) * 1e-3 / inflight)
        spent += piped[-1] * inflight
    # profiled pass: match-kernel time and rows read per call
    h.g.reset_stats()
    h.g.set_profiling(True)
    for _ in range(20):
        h.pick(s.cuda_stream)
    torch.cuda.synchronize()
    st = h.g.stats()
    h.g.set_profiling(False)
    calls = max(st.n_match_pick, 1)
    match_us = st.ms_match_pick * 1e3 / calls
    rows = st.probed_blocks / calls
    return {"stream_ordered_us": {"median": float(np.median(ordered)) * 1e6, "min": float(min(ordered)) * 1e6,
                                  "max": float(max(ordered)) * 1e6, "calls": len(ordered)},
            "pipelined_us": {"median": float(np.median(piped)) * 1e6, "min": float(min(piped)) * 1e6,
                             "max": float(max(piped)) * 1e6, "inflight": inflight},
            "match_kernel_us": match_us, "rows_per_call": rows, "rows_per_us": rows / match_us,
            "ns_per_row": 1e3 * match_us / max(rows, 1)}


# The cost of one window boundary, isolated: one max_blocks = 4095 handle and one index, every prompt 1 100 blocks long,
# request r holding the first K blocks of group r % 256 and bytes of its own after them, so the walk reads K rows and
# ends at block K.  K < 1024 stays in window 0; K >= 1024 also stages window 1 and resolves it.  The match kernel's time
# per call against K, the cached lengths alternated round by round: the line through the K < 1024 points is the cost
# of the rows, and a point past the boundary minus that line is what crossing it costs.
BOUNDARY_K = (992, 1000, 1008, 1016, 1023, 1024, 1025, 1032, 1040, 1048, 1056)


def boundary(R, rounds):
    import torch

    M = 1100
    rng = np.random.default_rng(11)
    groups = rng.integers(0, 256, size=(GROUPS, M * B), dtype=np.uint8)
    own = rng.integers(0, 256, size=(R, M * B + B // 2), dtype=np.uint8)
    offs = np.arange(R + 1, dtype=np.uint64) * own.shape[1]
    feeds = {}
    for k in BOUNDARY_K:
        tok = own.copy()
        tok[:, : k * B] = groups[np.arange(R) % GROUPS, : k * B]
        feeds[k] = torch.from_numpy(tok.reshape(-1)).cuda()
    h = Handle(4095, M, R, groups, own.reshape(-1), offs)
    s = torch.cuda.current_stream().cuda_stream
    us = {k: [] for k in BOUNDARY_K}
    rows = {}
    for k in BOUNDARY_K:  # warm-up
        h.d_tok = feeds[k]
        h.pick(s)
    for _ in range(rounds):
        for k in BOUNDARY_K:
            h.d_tok = feeds[k]
            h.g.reset_stats()
            h.g.set_profiling(True)
            for _ in range(20):
                h.pick(s)
            torch.cuda.synchronize()
            st = h.g.stats()
            h.g.set_profiling(False)
            us[k].append(st.ms_match_pick * 1e3 / max(st.n_match_pick, 1))
            rows[k] = st.probed_blocks / max(st.n_match_pick, 1)
    h.g.close()
    med = {k: float(np.median(v)) for k, v in us.items()}
    below = [k for k in BOUNDARY_K if k < 1024]
    slope, icpt = np.polyfit(below, [med[k] for k in below], 1)
    excess = {k: med[k] - (slope * k + icpt) for k in BOUNDARY_K}
    above = [k for k in BOUNDARY_K if k >= 1024]
    return {"requests": R, "prompt_blocks": M,
            "match_kernel_us": {str(k): {"median": med[k], "min": min(us[k]), "max": max(us[k]), "rows_per_call": rows[k]}
                                for k in BOUNDARY_K},
            "row_cost_ns_per_request_block": slope * 1e3 / R,
            "excess_over_row_line_us": {str(k): excess[k] for k in BOUNDARY_K},
            "boundary_cost_ns_per_request": float(np.median([excess[k] for k in above])) * 1e3 / R,
            "boundary_cost_in_blocks": float(np.median([excess[k] for k in above])) / slope}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--R", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--inflight", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3, help="boundary sweep: rounds over every cached length")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_long needs a CUDA device")
    out = {"card": card(), "endpoints": E, "requests": args.R, "block_bytes": B, "results": {}}
    for M in (1023, 2047, 4095):
        groups, tok, offs = workload(M, args.R)
        h = Handle(M, M, args.R, groups, tok, offs)
        out["results"][f"M={M}"] = timed(h, args.seconds, args.inflight)
        if M == 1023:  # the same prompts and index through the windowed kernel: no boundary is crossed
            base = h.picks()
            h.g.close()
            hw = Handle(4095, M, args.R, groups, tok, offs)
            out["results"]["M=1023 windowed"] = timed(hw, args.seconds, args.inflight)
            assert np.array_equal(hw.picks(), base), "windowed picks differ on 1023-block prompts"
            hw.g.close()
        else:
            h.g.close()
        print(json.dumps({f"M={M}": out["results"][f"M={M}"]}), file=sys.stderr, flush=True)
    r = out["results"]
    out["window_variant_cost_ns_per_row"] = r["M=1023 windowed"]["ns_per_row"] - r["M=1023"]["ns_per_row"]
    out["boundary"] = boundary(args.R, args.rounds)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
