#!/usr/bin/env python
"""The pipelined calls of a serving loop (fi_epp_pick_submit_ex / _wait_batch / fi_epp_index_add_submitted,
docs/SPEC.md S.9) against the stream-ordered calls, on the bench.py workload.

1. Picks: microseconds per step of each variant (single, single with chains_out, LoRA, ranked k = 1 / 4 / 16,
   64-endpoint subsets at k = 4), pipelined (--steps submits back to back, one wait) against the stream-ordered
   counterpart (--steps calls), timed with CUDA events; variants alternated round by round, median / min / max
   reported.  Also the device-to-device copy fi_epp_index_add_submitted makes of a batch's chains, timed alone.
2. Serving loop with PreRequest: submit_ex(k+1) -> wait_batch(k) -> read the picks on the host -> add_submitted(k),
   against two stream-ordered loops: pick_batch_device(k) -> read -> fi_epp_index_add_chains_device(.., NULL, ..), and
   the same calls in the pipelined loop's logical order (pick k+1 before Add k, with pick k's chains_out), each on a
   fresh handle in the same initial state.  Reported: wall time per step (host clock, every step ends in a host read
   of its picks), host time spent inside each call, and whether the pipelined loop's picks agree bit for bit with the
   stream-ordered loop of the same logical order (the NULL-chains loop adds batch k before batch k+1 is picked).
3. --trace N: only the pipelined loop, with FI_EPP_TRACE=N (kernel timelines on stderr; run apart from the timing).

The card's name, power limit and SM clock are read in the same run.

    python tools/bench_pipeline.py [--cfg 3] [--steps 20] [--rounds 5] [--loop-steps 30] [--trace N]
"""
from __future__ import annotations

import argparse
import hashlib
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # pragma: no cover
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20, help="batches per timed window of a pick variant")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=30)
    ap.add_argument("--trace", type=int, default=-1, help="FI_EPP_TRACE call index: trace the pipelined loop only")
    args = ap.parse_args()
    card_before = card()

    import torch

    from fusioninfer_b200 import PICK_DTYPE, EndpointPicker, make_config, subset_bitsets, synth
    from fusioninfer_b200 import _abi as abi

    if not torch.cuda.is_available():
        raise SystemExit("bench_pipeline needs a CUDA device")
    wl = synth.baseline_workload(args.cfg)
    profiles, pd = synth.baseline_profiles(args.cfg)
    slots = 4096
    while slots < 2 * wl.E * wl.lru_capacity:
        slots *= 2
    R, E = wl.R, wl.E
    L = abi.FI_SCORER_LORA
    lora_profiles = [{"name": "default", "scorers": [(abi.FI_SCORER_PREFIX, 60), (L, 30), (abi.FI_SCORER_KV_UTIL, 5),
                                                     (abi.FI_SCORER_QUEUE, 5)]}]

    def config(prof, pd_):
        return make_config(num_endpoints=E, block_bytes=wl.block_bytes, max_blocks=wl.max_blocks, max_batch=R,
                           lru_capacity=wl.lru_capacity, max_prompt_bytes=R * wl.T * 4, index_slots=slots,
                           profiles=prof, pd=pd_)

    states = wl.endpoint_states()
    ops = list(wl.index_ops())

    def handle(prof, pd_):
        g = EndpointPicker(config(prof, pd_))
        g.update_endpoints(states)
        for o in ops:
            g.index_apply(o)
        g.index_sync()
        return g

    s = torch.cuda.current_stream()
    NB = 3
    batches = []
    for i in range(NB):
        tok, offs = wl.prompts(batch=i)
        batches.append((torch.from_numpy(tok.reshape(-1).view(np.int32)).cuda(), torch.from_numpy(offs.view(np.int64)).cuda(),
                        tok.nbytes))
    d_h0 = torch.full((R,), np.uint64(wl.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(7)
    d_ad = torch.from_numpy((rng.integers(0, 14, R) + 1000).astype(np.int64)).cuda()
    d_sub = torch.from_numpy(subset_bitsets(list(np.argsort(rng.random((R, E)), axis=1)[:, :64]), E).view(np.int32)).cuda()
    out = {"card (name, power limit, SM clock, max SM clock)": {"before": card_before},
           "workload": f"cfg{args.cfg}: {R} requests x {E} endpoints, {wl.n_blocks} blocks per prompt",
           "lib": os.environ.get("FI_EPP_LIB", "default")}

    def loop(g, kind, steps, stats):
        """kind: "pipelined", "same_order" (stream-ordered calls in the pipelined loop's logical order: pick k+1 is made
        before Add k, whose chains come from pick k's chains_out) or "null_chains" (pick k, then Add k with the chains
        of the handle's buffer).  -> digests of every step's picks"""
        P = g.n_profiles
        d_out = [torch.zeros(R * P * 16, dtype=torch.uint8, device="cuda") for _ in range(NB)]
        d_ch = [torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda") for _ in range(2)]
        host = np.zeros((R, P), dtype=PICK_DTYPE)
        digests = []

        def timed(name, fn):
            t0 = time.perf_counter()
            r = fn()
            stats[name] = stats.get(name, 0.0) + (time.perf_counter() - t0)
            return r

        def args_of(k):
            b = batches[k % NB]
            return b[0].data_ptr(), b[1].data_ptr(), d_h0.data_ptr(), R, b[2], d_out[k % NB].data_ptr()

        def read(k):
            host.view(np.uint8).reshape(-1)[:] = d_out[k % NB].cpu().numpy()  # (waits for the stream)
            digests.append(hashlib.sha256(host.tobytes()).hexdigest()[:16])
            return host[:, 0]["endpoint"].copy(), host[:, 0]["n_blocks"].astype(np.uint32)

        if kind == "pipelined":
            tk = {0: timed("submit_ex", lambda: g.pick_submit_ex(*args_of(0), stream=s.cuda_stream))}
            for k in range(steps):
                tk[k + 1] = timed("submit_ex", lambda: g.pick_submit_ex(*args_of(k + 1), stream=s.cuda_stream))
                timed("wait_batch", lambda: g.pick_wait_batch(tk[k], s.cuda_stream))
                eps, nb = timed("read picks", lambda: read(k))
                timed("add_submitted", lambda: g.index_add_submitted(tk[k], eps, nb))
            g.pick_wait(s.cuda_stream)
        elif kind == "same_order":
            g.pick_batch_device(*args_of(0), d_ch[0].data_ptr(), s.cuda_stream)
            for k in range(steps):
                timed("pick_batch_device", lambda: g.pick_batch_device(*args_of(k + 1), d_ch[(k + 1) % 2].data_ptr(),
                                                                       s.cuda_stream))
                eps, nb = timed("read picks", lambda: read(k))
                timed("add_chains_device", lambda: g.index_add_chains_device(eps, d_ch[k % 2].data_ptr(), wl.max_blocks, nb,
                                                                             s.cuda_stream))
        else:
            for k in range(steps):
                timed("pick_batch_device", lambda: g.pick_batch_device(*args_of(k), 0, s.cuda_stream))
                eps, nb = timed("read picks", lambda: read(k))
                timed("add_chains_device(NULL)", lambda: g.index_add_chains_device(eps, 0, 0, nb, s.cuda_stream))
        g.index_sync()
        torch.cuda.synchronize()
        return digests

    if args.trace >= 0:
        os.environ["FI_EPP_TRACE"] = str(args.trace)
        g = handle(profiles, pd)
        loop(g, "pipelined", args.trace + 6, {})
        g.close()
        print(json.dumps({"trace": f"FI_EPP_TRACE={args.trace}: pipelined loop, timelines on stderr", **out}), flush=True)
        return

    # ---- 1. pick variants
    def variants(g, lora):
        # (name, k, adapters, subsets, chains_out): "single k=0 + chains_out" against "single k=0" is the cost of the
        # chains_out copy
        v = [("LoRA k=0", 0, True, False, False)] if lora else [
            ("single k=0", 0, False, False, False), ("single k=0 + chains_out", 0, False, False, True),
            ("ranked k=1", 1, False, False, False), ("ranked k=4", 4, False, False, False),
            ("ranked k=16", 16, False, False, False), ("subset 64 k=4", 4, False, True, False)]
        P = g.n_profiles
        res = {}
        bufs = {name: [torch.zeros(R * P * max(k, 1) * 16, dtype=torch.uint8, device="cuda") for _ in range(2)]
                for name, k, *_ in v}
        d_chains = torch.zeros(R * wl.max_blocks, dtype=torch.int64, device="cuda")

        def run(name, k, ad, sub, ch, pipelined):
            dc = d_chains.data_ptr() if ch else 0
            o = bufs[name][0 if pipelined else 1]
            for i in range(args.steps):
                b = batches[i % NB]
                a = (b[0].data_ptr(), b[1].data_ptr(), d_h0.data_ptr(), R, b[2])
                if pipelined:
                    g.pick_submit_ex(*a, o.data_ptr(), k=k, d_adapters=d_ad.data_ptr() if ad else 0,
                                     d_subsets=d_sub.data_ptr() if sub else 0, d_chains=dc, stream=s.cuda_stream)
                elif k == 0:
                    rc = abi.load().fi_epp_pick_batch_device_lora(g._h, a[0], a[1], a[2], d_ad.data_ptr() if ad else None, R,
                                                                  a[4], o.data_ptr(), dc or None, s.cuda_stream)
                    g._check(rc, "fi_epp_pick_batch_device_lora")
                else:
                    g.pick_batch_device_subset(*a, k, o.data_ptr(), d_sub.data_ptr() if sub else 0, dc, s.cuda_stream,
                                               d_ad.data_ptr() if ad else 0)
            if pipelined:
                g.pick_wait(s.cuda_stream)

        for item in v:  # warm-up
            for p in (True, False):
                run(*item, p)
        torch.cuda.synchronize()
        times = {(item[0], p): [] for item in v for p in (True, False)}
        for _ in range(args.rounds):
            for item in v:
                for p in (True, False):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(s)
                    run(*item, p)
                    b.record(s)
                    b.synchronize()
                    times[(item[0], p)].append(a.elapsed_time(b) * 1e3 / args.steps)
        for name, *_ in v:
            same = bufs[name][0].cpu().numpy().tobytes() == bufs[name][1].cpu().numpy().tobytes()
            res[name] = {kind: {"median_us": round(float(np.median(times[(name, p)])), 1),
                                "min_us": round(float(min(times[(name, p)])), 1),
                                "max_us": round(float(max(times[(name, p)])), 1)}
                         for kind, p in (("pipelined", True), ("stream_ordered", False))}
            res[name]["last batch bit-exact"] = same
        return res

    g = handle(profiles, pd)
    res = variants(g, False)
    g.close()
    g = handle(lora_profiles, None)
    lo = np.zeros(E, dtype=__import__("fusioninfer_b200").LORA_DTYPE)
    lo["endpoint"] = np.arange(E)
    lo["n_active"] = rng.integers(0, 5, E)
    for e in range(E):
        lo[e]["active"][: lo[e]["n_active"]] = rng.permutation(12)[: lo[e]["n_active"]] + 1000
    lo["max_active"] = 4
    g.update_endpoints_lora(lo)
    res.update(variants(g, True))
    g.close()
    out["picks (us per step)"] = res
    # fi_epp_index_add_submitted's chain copy (R x MP u64, device to device) alone: it overlaps the match in the loop
    src = torch.zeros(R * ((wl.max_blocks + 7) // 8 * 8), dtype=torch.int64, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    ts = []
    for _ in range(20):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        dst.copy_(src)
        b.record(s)
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    out["add_submitted chain copy alone (us)"] = {"bytes": src.numel() * 8, "median_us": round(float(np.median(ts)), 1)}

    # ---- 2. serving loop with PreRequest
    loops = {}
    digests = {}
    kinds = ("pipelined", "same_order", "null_chains")
    g = handle(profiles, pd)
    for kind in kinds:  # warm-up: first launches of every kernel the loops use
        loop(g, kind, 3, {})
    g.close()
    for name in kinds:
        g = handle(profiles, pd)
        st = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        digests[name] = loop(g, name, args.loop_steps, st)
        wall = time.perf_counter() - t0
        loops[name] = {"us_per_step": round(wall * 1e6 / args.loop_steps, 1),
                       "host_us_per_step_inside": {k: round(v * 1e6 / args.loop_steps, 1) for k, v in st.items()},
                       "lru_counters": g.lru_counters(), "index_rebuilds": int(g.index_stats().rebuilds)}
        g.close()
    # (null_chains adds batch k before batch k+1 is picked: a different logical order, so its picks may differ)
    loops["picks agree bit for bit"] = digests["pipelined"] == digests["same_order"]
    out["serving loop with PreRequest"] = loops
    out["card (name, power limit, SM clock, max SM clock)"]["after"] = card()
    print(json.dumps(out), flush=True)
    if not loops["picks agree bit for bit"] or not all(v["last batch bit-exact"] for v in res.values()):
        raise SystemExit("pipelined and stream-ordered picks differ")


if __name__ == "__main__":
    main()
