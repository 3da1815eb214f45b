"""Markdown table of saved bench lines (one bench.py JSON line per file) for README.md:  python scripts/results_table.py DIR/*.json"""
import glob
import json
import os
import sys

rows = []
for f in sorted(sum((glob.glob(a) for a in sys.argv[1:]), [])):
    try:
        d = json.loads(open(f).read().strip().splitlines()[-1])
    except Exception:
        continue
    if d.get("impl") == "reference":
        rows.append((os.path.basename(f), d["config"]["workload"].split(":")[0], "CPU oracle port, %s threads" % d["cpu_baseline"]["cores"], d["config"]["nodes"],
                     d["ms_per_step"], d.get("placements_per_sec"), d["value"], None, None, None, d["cpu_baseline"]["sample"].split(" (")[0]))
        continue
    lat = d["roofline"].get("latency", {})
    rows.append((os.path.basename(f), d["config"]["workload"].split(":")[0], "%d x H100, %s" % (d["n_gpus"], lat.get("engine", "?")), d["config"]["nodes"], d["ms_per_step"],
                 d["placements_per_sec"], d["value"], d["e2e"]["value"], lat.get("placements_per_wave"), lat.get("us_per_wave"),
                 "parity ok, %d placements%s" % (d["parity"]["checked_placements"], "" if d["parity"]["full_run"] else " (prefix)") if d.get("parity") else ""))
print("| file | workload | arm | nodes | ms / analysis | placements/s | evals/s | e2e evals/s (flat C-ABI) | placements / wave | us / wave | check |")
print("|---|---|---|---|---|---|---|---|---|---|---|")
for r in rows:
    f = lambda x, fmt: "" if x is None else fmt % x
    print("| %s | %s | %s | %d | %s | %s | %s | %s | %s | %s | %s |" % (r[0], r[1], r[2], r[3], f(r[4], "%.2f"), f(r[5], "%.3g"), f(r[6], "%.3g"), f(r[7], "%.3g"), f(r[8], "%.2f"), f(r[9], "%.2f"), r[10]))
