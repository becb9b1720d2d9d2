#!/usr/bin/env python3
"""Shared-memory wavefronts, instructions and sample share per barrier-separated phase of one kernel of an ncu report:
  python tools/ncu_phase_lsu.py report.ncu-rep NTH_LAUNCH [SMS=132]
(wavefronts / SMS vs share-of-lifetime x cycles tells which phases are bound by the LSU, which by issue slots)."""
import csv, io, subprocess, sys
rep, kid = sys.argv[1], sys.argv[2]
sms = int(sys.argv[3]) if len(sys.argv) > 3 else 132   # H100 SXM
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-id", ":::" + kid], capture_output=True, text=True).stdout
lines = out.splitlines()
print(lines[0][:120])
rows = list(csv.reader(io.StringIO("\n".join(lines[1:]))))
h = rows[0]; body = []
for r in rows[1:]:
    if r == h: break
    if len(r) == len(h): body.append(r)
S = h.index("# Samples"); EX = h.index("Instructions Executed")
W = h.index("L1 Wavefronts Shared"); WI = h.index("L1 Wavefronts Shared Ideal")
tot = sum(int(r[S]) for r in body)
start = 0
print("  phase [first,last) instr | share of samples | smem wavefronts per SM (ideal) | warp-instr per SM per scheduler")
for i, r in enumerate(body + [None]):
    if r is None or "BAR.SYNC" in r[1]:
        end = i + 1 if r is not None else i
        seg = body[start:end]
        if seg:
            w = sum(int(x[W]) for x in seg); wi = sum(int(x[WI]) for x in seg); sm = sum(int(x[S]) for x in seg); ex = sum(int(x[EX]) for x in seg)
            print(f"  [{start:5d},{end:5d}) {100 * sm / tot:5.1f}%  wavefronts/SM {w / sms:9.0f} ({wi / sms:9.0f})  instr/SM/sched {ex / sms / 4:9.0f}")
        start = end
