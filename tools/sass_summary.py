#!/usr/bin/env python
"""Per-kernel SASS census of libmww_b200.so (cuobjdump -sass): registers are in the ptxas log, this lists which
instruction families each kernel actually contains -- tensor-core (HMMA / IMMA / HGMMA), asynchronous copies (LDGSTS,
UBLKCP / UBLKPF, UTMALDG), barriers, 64/128-bit shared and global accesses -- so the claims in DESIGN.md can be checked
against the binary.    python tools/sass_summary.py"""
import collections
import os
import re
import subprocess
import sys

so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "microwakeword_b200", "libmww_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
FAMILIES = ["HMMA", "IMMA", "HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "UBLKPF", "LDGSTS", "LDG", "STG", "LDS", "STS",
            "BAR", "SYNCS", "FFMA", "IMAD", "DFMA", "MUFU", "SHFL", "REDUX", "ATOM"]
kern, counts, total = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        counts[kern] = collections.Counter()
        total[kern] = 0
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and kern:
        op = m.group(1)
        total[kern] += 1
        base = op.split(".")[0]
        for f in FAMILIES:
            if base == f:
                counts[kern][f] += 1
        for wide in ("LDS", "STS", "LDG", "STG"):
            if base == wide and (".64" in op or ".128" in op):
                counts[kern][wide + (".128" if ".128" in op else ".64")] += 1
        if base == "HMMA" or base == "IMMA":
            counts[kern][op] += 1
print("SASS census of %s (sm_90a)\n" % os.path.basename(so))
for k, c in counts.items():
    if total[k] < 50:
        continue
    print("%-60s %6d instructions" % (k[:60], total[k]))
    print("    " + "  ".join("%s:%d" % (f, n) for f, n in sorted(c.items(), key=lambda kv: -kv[1])))
