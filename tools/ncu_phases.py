#!/usr/bin/env python
"""Attribute a kernel's executed instructions to barrier-delimited segments (phases) from an .ncu-rep source page.
    python tools/ncu_phases.py k1_v2.ncu-rep <units_in_launch>"""
import collections, csv, subprocess, sys
rep, units = sys.argv[1], float(sys.argv[2])
raw = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr = rows[1]
ia, ie, iss = hdr.index("Source"), hdr.index("Instructions Executed"), hdr.index("# Samples")
ins = [(r[ia].strip(), int(r[ie]), int(r[iss])) for r in rows[2:] if len(r) > ie]
tot, tots = sum(e for _, e, _ in ins), sum(s for _, _, s in ins)
print("total thread-instr/unit %.0f  static SASS %d" % (tot * 32 / units, len(ins)))
seg, segs = 0, collections.defaultdict(lambda: [0, 0, collections.Counter()])
for src, e, s in ins:
    parts = src.split()
    op = (parts[1] if parts[0].startswith("@") else parts[0]).split(".")[0]
    segs[seg][0] += e; segs[seg][1] += s; segs[seg][2][op] += e
    if op == "BAR":
        seg += 1
for k, (e, s, c) in segs.items():
    print("seg %d: instr/unit %7.0f share %.3f stall-samples %.3f | %s" % (k, e * 32 / units, e / tot, s / max(tots, 1),
          ", ".join("%s:%.0f" % (o, v * 32 / units) for o, v in c.most_common(10))))
