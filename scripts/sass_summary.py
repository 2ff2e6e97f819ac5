"""Per-kernel SASS counts of the built library (cuobjdump -sass): 256-bit / 128-bit global accesses, IMAD.WIDE, IMAD, IADD3,
barriers, TMA and tensor-core instructions (none, by design).  No GPU needed.
usage: python scripts/sass_summary.py [out.txt]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "circom_b200", "libcircom_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
cur, counts = None, collections.OrderedDict()
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        counts[cur][m.group(1)] += 1
lines = ["SASS summary of circom_b200/libcircom_b200.so (cuobjdump -sass, sm_90a), scripts/sass_summary.py",
         "kernel | instructions | LDG/STG.E.ENL2.256 (one 32-byte element per access) | LDG.128 / STG.128 | LDG.64 | IMAD.WIDE | IMAD | IADD3 | "
         "BAR | UTMALDG/UBLKCP (TMA) | HMMA/UTC*MMA (tensor)"]
for k, c in counts.items():
    def n(pred):
        return sum(v for op, v in c.items() if pred(op))
    name = re.sub(r"^_ZN2cw", "", k)[:86]
    lines.append("%s | %d | %d / %d | %d / %d | %d | %d | %d | %d | %d | %d | %d" % (
        name, sum(c.values()),
        n(lambda o: o.startswith("LDG") and "256" in o), n(lambda o: o.startswith("STG") and "256" in o),
        n(lambda o: o.startswith("LDG") and ".128" in o), n(lambda o: o.startswith("STG") and ".128" in o),
        n(lambda o: o.startswith("LDG") and ".64" in o),
        n(lambda o: o.startswith("IMAD.WIDE")), n(lambda o: o.startswith("IMAD") and not o.startswith("IMAD.WIDE")),
        n(lambda o: o.startswith("IADD3")), n(lambda o: o.startswith("BAR")),
        n(lambda o: o.startswith("UTMA") or o.startswith("UBLKCP")), n(lambda o: "MMA" in o)))
out = "\n".join(lines) + "\n"
if len(sys.argv) > 1:
    open(sys.argv[1], "w").write(out)
else:
    sys.stdout.write(out)
