"""Per-launch table (kernel, grid, block, microseconds) of the LAST step in an ncu launch-list CSV.
    python tools/launch_table.py ncu_out/launches_c.csv <launches per step>"""
import csv
import re
import sys

rows = []
with open(sys.argv[1]) as f:
    lines = [l for l in f if l.startswith('"')]
for r in csv.DictReader(lines):
    if r["Metric Name"] == "gpu__time_duration.sum":
        rows.append((r["Kernel Name"], r["Grid Size"], r["Block Size"], float(r["Metric Value"]) / 1e3))
per = int(sys.argv[2]) if len(sys.argv) > 2 else len(rows)
last = rows[-per:]
print(f"{len(rows)} launches captured; last {len(last)}: {sum(t for *_, t in last) / 1e3:.3f} ms")
for name, grid, block, us in last:
    short = re.sub(r"^void ", "", name)
    short = re.sub(r"\(.*", "", short).replace("ptrb200::", "")
    print(f"{short[:58]:58s} {grid:>16s} {block:>14s} {us:9.1f}")
