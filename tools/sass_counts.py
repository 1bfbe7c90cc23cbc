#!/usr/bin/env python3
"""SASS of libmgb200.so by kernel: size, instruction mix, and the bulk-copy / barrier sequence of the chaining kernels.

    python tools/sass_counts.py [minigraph_b200/libmgb200.so] > sass_counts.txt

(cuobjdump -sass; no GPU needed.)  UBLKCP = cp.async.bulk, SYNCS = mbarrier, VIMNMX/REDUX = the integer paths of the WFA cell and of the
warp reductions.  Device functions kept out of line (MG_NOINLINE) are counted with the kernel they belong to."""
import collections
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(REPO, "minigraph_b200", "libmgb200.so")
txt = subprocess.run(["cuobjdump", "-sass", so], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
kern, cur = collections.OrderedDict(), None
for line in txt.split("\n"):
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = m.group(1)
        mm = re.match(r"_Z\d+(k_[a-z_0-9]*[a-z])\d", name) or re.match(r"_ZN3mgb\d+(k_[a-z_]+)E", name)
        cur = mm.group(1) if mm else None
        if cur:
            kern.setdefault(cur, [])
        continue
    if cur:
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(.*?);", line)
        if m:
            kern[cur].append((m.group(1), re.sub(r"\s+", " ", m.group(2))))
COLS = ("LDG", "LDS", "STG", "STS", "LDL", "STL", "SHFL", "VOTE", "REDUX", "VIMNMX", "UBLKCP", "SYNCS")
print("# SASS of minigraph_b200/libmgb200.so (cuobjdump -sass, sm_90a): size and instruction mix of every kernel of the path (tools/sass_counts.py),")
print("# then the bulk-copy / barrier sequence of the chaining kernels (UBLKCP = cp.async.bulk, SYNCS = mbarrier).\n")
print("%-18s %7s " % ("kernel", "instr") + " ".join("%6s" % c for c in COLS))
for k, ins in kern.items():
    cnt = collections.Counter()
    for _, t in ins:
        op = t.split()[1] if t.startswith("@") else t.split()[0]
        cnt[op.split(".")[0]] += 1
    print("%-18s %7d " % (k, len(ins)) + " ".join("%6d" % cnt[c] for c in COLS))
for k in ("k_chain", "k_chain_rescue"):
    print("\n# %s: every UBLKCP / SYNCS instruction" % k)
    for a, t in kern.get(k, []):
        if "UBLKCP" in t or "SYNCS" in t:
            print("        /*%s*/  %s ;" % (a, t))
