"""SASS evidence: per-kernel instruction-mnemonic histogram of libccsim.so (cuobjdump -sass) and the lines that prove the bulk-async
(TMA) / mbarrier / warp-reduction instructions. No GPU needed:  python scripts/sass_summary.py > sass_summary.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "cluster-capacity_b200", "libccsim.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
kern, hist, proof = None, {}, {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        hist[kern] = collections.Counter()
        proof[kern] = []
        continue
    m = re.match(r"\s+/\*([0-9a-f]+)\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and kern:
        op = m.group(3)
        hist[kern][op.split(".")[0]] += 1
        if re.match(r"(UBLKCP|UTMALDG|SYNCS|CREDUX|REDUX|VOTE|BAR|MEMBAR|FENCE|ST\.E\.64\.STRONG\.SYS|LD\.E\.64\.STRONG\.SYS)", op):
            if len(proof[kern]) < 400:
                proof[kern].append(line.strip()[:120])
print("SASS summary of", os.path.relpath(so, ROOT), "(sm_90a, nvcc %s)" % subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout.split("release ")[-1].split(",")[0])
for k in sorted(hist):
    tot = sum(hist[k].values())
    print("\n== %s: %d instructions" % (k, tot))
    print("   " + "  ".join("%s:%d" % kv for kv in hist[k].most_common(18)))
    keys = collections.Counter(re.match(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", p).group(1) for p in proof[k])
    if keys:
        print("   evidence: " + "  ".join("%s x%d" % kv for kv in sorted(keys.items())))
    for p in proof[k]:
        if re.search(r"UBLKCP|SYNCS|UTMALDG", p):
            print("     " + p)
