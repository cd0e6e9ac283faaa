"""SASS census of libptranking_b200.so: per kernel, the counts of the Hopper-specific instructions that prove which
hardware paths the binary uses (wgmma.mma_async = HGMMA, wgmma.fence = WARPGROUP, TMA bulk copy = UBLKCP, mbarrier = SYNCS,
SFU = MUFU) -> profiles/<tag>_sass_census.md.  Runs without a GPU:  python tools/sass_census.py [tag]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ptranking_b200", "lib", "libptranking_b200.so")
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
WANT = ["HGMMA", "WARPGROUP", "UBLKCP", "SYNCS", "MUFU", "SHFL", "STS", "LDG", "STG"]
kern, counts, size = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        kern = m.group(1)
        counts[kern] = collections.Counter()
        size[kern] = 0
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and kern:
        size[kern] += 1
        op = m.group(1)
        for w in WANT:
            if op.startswith(w):
                counts[kern][w] += 1
dem = subprocess.run(["c++filt"], input="\n".join(counts), capture_output=True, text=True).stdout.splitlines()
rows = []
for k, d in zip(counts, dem):
    short = re.sub(r"\(.*", "", d.replace("ptrb200::", "").replace("void ", ""))[:64]
    rows.append((short, size[k], counts[k]))
rows.sort(key=lambda r: (-r[2]["HGMMA"], -r[1]))
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
path = os.path.join(ROOT, "profiles", f"{tag}_sass_census.md")
with open(path, "w") as f:
    f.write(f"# {tag}: SASS census of libptranking_b200.so (`cuobjdump -sass`, sm_90a; `python tools/sass_census.py`)\n\n")
    f.write("HGMMA = wgmma.mma_async, WARPGROUP = wgmma fences / waits, UBLKCP = cp.async.bulk (TMA engine),\n"
            "SYNCS = mbarrier ops, MUFU = special-function unit.  Static instruction counts per kernel (not executed counts).\n\n")
    f.write("| kernel | SASS instr | " + " | ".join(WANT) + " |\n|---|---|" + "---|" * len(WANT) + "\n")
    tot = collections.Counter()
    for short, n, c in rows:
        f.write(f"| `{short}` | {n} | " + " | ".join(str(c[w]) for w in WANT) + " |\n")
        tot.update(c)
    f.write(f"| **total ({len(rows)} kernels)** | {sum(r[1] for r in rows)} | " + " | ".join(str(tot[w]) for w in WANT) + " |\n")
print(open(path).read()[:3000])
