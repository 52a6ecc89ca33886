#!/usr/bin/env python
"""Decode per-instruction stall counts (control bits 105..108 of the 128-bit instruction word: the layout of Volta
through Hopper SASS, Jia et al., "Dissecting the NVIDIA Volta GPU Architecture via Microbenchmarking", 2018; on
sm_90a builds the fields decode to stall counts of 0-15, barrier indices 0-5 and write barriers on the loads) from
`cuobjdump -sass` output and sum them over an address range: a single-warp, in-order issue-time
estimate for fixed-latency regions (e.g. the serial link of the chain walker).
usage: sass_stalls.py <obj> <function-substring> [start_hex end_hex]"""
import re, subprocess, sys

obj, fn = sys.argv[1], sys.argv[2]
out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
blocks = out.split("Function : ")
body = next(b for b in blocks if fn in b.split("\n")[0])
lines = body.split("\n")
ins = []
i = 0
pat = re.compile(r"^\s+/\*([0-9a-f]{4})\*/\s+(.*?);\s+/\* (0x[0-9a-f]{16}) \*/")
pat2 = re.compile(r"^\s+/\* (0x[0-9a-f]{16}) \*/")
while i < len(lines):
    m = pat.match(lines[i])
    if m and i + 1 < len(lines):
        m2 = pat2.match(lines[i + 1])
        if m2:
            hi = int(m2.group(1), 16)
            stall = (hi >> 41) & 0xF
            yield_ = (hi >> 45) & 1
            wait = (hi >> 52) & 0x3F
            wbar = (hi >> 46) & 7
            rbar = (hi >> 49) & 7
            ins.append((int(m.group(1), 16), m.group(2).strip() + (f"   [wbar {wbar}]" if wbar != 7 else "") + (f" [rbar {rbar}]" if rbar != 7 else ""), stall, wait))
            i += 2
            continue
    i += 1
lo = int(sys.argv[3], 16) if len(sys.argv) > 3 else 0
hi_ = int(sys.argv[4], 16) if len(sys.argv) > 4 else 1 << 30
sel = [x for x in ins if lo <= x[0] <= hi_]
print(f"{len(sel)} instructions, sum of stall counts = {sum(x[2] for x in sel)} cycles, with wait-masks: {sum(1 for x in sel if x[3])}")
if "-v" in sys.argv:
    for a, t, s, w in sel:
        print(f"{a:04x} stall={s:2d} wait={w:02x}  {t[:90]}")
