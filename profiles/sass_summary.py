"""Per-kernel SASS instruction summary of libinterdiff_b200.so (cuobjdump -sass): the mnemonics that prove which hardware
path a kernel uses - HGMMA (wgmma), UTMALDG (TMA tensor loads), UBLKCP (bulk copies),
SYNCS (mbarrier), HMMA (legacy mma.sync), FFMA, LDS/STS, LDG/STG, red/atom.   python profiles/sass_summary.py"""
import collections
import os
import re
import subprocess
import sys

so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "interdiff_b200", "libinterdiff_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
KEYS = ["HGMMA", "UTMALDG", "UBLKCP", "SYNCS", "HMMA", "FFMA", "MUFU", "LDS", "STS", "LDG", "STG", "RED", "ATOM", "SHFL", "BAR", "UCGABAR", "ACQBULK"]
cur, counts, total = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        total[cur] = 0
        continue
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1).split(".")[0]
        total[cur] += 1
        for k in KEYS:
            if op == k or (k in ("HGMMA", "UTMALDG", "UBLKCP", "SYNCS", "HMMA", "UCGABAR") and op.startswith(k)):
                counts[cur][k] += 1
def demangle(n):
    try:
        d = subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
        d = d.replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
        m = re.search(r"([A-Za-z_][\w:]*(?:<[^()]*>)?)\(", d)
        return (m.group(1) if m else d)[-70:]
    except Exception:
        return n[-70:]
print("%-70s %7s  %s" % ("kernel", "instrs", "  ".join("%s" % k for k in KEYS)))
for fn, c in counts.items():
    print("%-70s %7d  %s" % (demangle(fn), total[fn], "  ".join("%*d" % (len(k), c[k]) for k in KEYS)))
