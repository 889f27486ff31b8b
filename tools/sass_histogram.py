"""Developer tool: per-kernel SASS opcode histogram of libsmot.so (cuobjdump -sass), the mnemonics that prove which hardware paths
a kernel uses (wgmma: HGMMA, TMA: UTMALDG / UBLKCP, mbarrier: SYNCS, legacy tensor
cores: HMMA, ldmatrix: LDSM, cp.async: LDGSTS, PDL: ACQBULK / PREEXIT ...).  Usage: python tools/sass_histogram.py [lib] > <file>"""
import collections
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(REPO, "siammot_b200", "libsmot.so")
KEY = ["UTCHMMA", "UTCQMMA", "UTCBAR", "UTCATOMSWS", "LDTM", "STTM", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "HMMA", "LDSM", "LDGSTS",
       "ACQBULK", "PREEXIT", "BAR", "LDG", "STG", "LDS", "STS", "FFMA", "HFMA2", "MUFU", "SHFL", "ATOM", "RED"]
out = subprocess.run(["cuobjdump", "-sass", lib], stdout=subprocess.PIPE, text=True, check=True).stdout
demangle = {}
kernels = collections.OrderedDict()
cur = None
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1)
        kernels[cur] = collections.Counter()
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)(\.[A-Z0-9_.]+)?", line)
    if m and cur:
        kernels[cur][m.group(1)] += 1
        kernels[cur]["__total__"] += 1
names = list(kernels)
dem = subprocess.run(["c++filt"] + names, stdout=subprocess.PIPE, text=True).stdout.splitlines()
print("# SASS opcode histogram of %s (cuobjdump -sass; static instruction counts per kernel)" % os.path.relpath(lib, REPO))
print("# columns: total instructions, then the counts of the path-proving mnemonics that occur")
for n, d in zip(names, dem):
    c = kernels[n]
    short = re.sub(r"\(.*", "", d).replace("void ", "").replace("smot::", "")
    keys = " ".join("%s=%d" % (k, c[k]) for k in KEY if c[k])
    print("%-58s %6d  %s" % (short[:58], c["__total__"], keys))
