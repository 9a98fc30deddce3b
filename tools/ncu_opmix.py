"""Dynamic opcode mix of a kernel from an .ncu-rep captured with --import-source on:
    python tools/ncu_opmix.py prof.ncu-rep [pixels_per_launch]
"""
import collections
import csv
import io
import re
import subprocess
import sys

raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
h = rows[hdr]
si, ei = h.index("Source"), h.index("Instructions Executed")
ops = collections.Counter()
total = 0
for r in rows[hdr + 1:]:
    if len(r) <= ei or not r[ei].isdigit():
        continue
    m = re.match(r"\s*(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", r[si])
    if not m:
        continue
    n = int(r[ei])
    ops[m.group(1)] += n
    total += n
px = float(sys.argv[2]) if len(sys.argv) > 2 else None
print(f"total warp instructions {total}" + (f" = {total * 32 / px:.1f} thread-instr per pixel" if px else ""))
for k, v in ops.most_common(28):
    print(f"  {k:10s} {v:12d} {100.0 * v / total:5.1f}%" + (f"  {v * 32 / px:6.1f}/px" if px else ""))
