"""ncu report -> small text summaries (no GPU needed):
   python scripts/summarize_ncu.py wave_c4.ncu-rep out/wave_c4"""
import csv, io, json, subprocess, sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "lts__t_bytes.sum", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "launch__grid_size", "launch__block_size",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__cycles_active.avg"]

def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    lines, traffic = [], {}
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        lines.append("kernel: %s  grid %s block %s" % (d.get("Kernel Name"), d.get("Grid Size"), d.get("Block Size")))
        for k in KEYS:
            if k in d:
                lines.append("  %-70s %s %s" % (k, d[k], units[hdr.index(k)]))
        def b(k):
            v, u = float(d[k]), units[hdr.index(k)]
            return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
        traffic = {"kernel": d.get("Kernel Name"), "dram_bytes_read": b("dram__bytes_read.sum"), "dram_bytes_write": b("dram__bytes_write.sum"),
                   "traffic_bytes_per_launch": b("dram__bytes_read.sum") + b("dram__bytes_write.sum"), "source": rep}
    open(out + "_raw_summary.txt", "w").write("\n".join(lines) + "\n")
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(src)))
    if len(rows) > 2:
        h = rows[1]; iS = h.index("# Samples"); data = [r for r in rows[2:] if len(r) > iS and r[iS].isdigit()]
        tot = sum(int(r[iS]) for r in data)
        st = [i for i, x in enumerate(h) if x.startswith("stall_") and "Not Issued" not in x]
        agg = {h[i]: sum(int(r[i]) for r in data if r[i].isdigit()) for i in st}
        top = sorted(data, key=lambda r: -int(r[iS]))[:25]
        with open(out + "_stalls.txt", "w") as f:
            f.write("warp-state samples: %d\n" % tot)
            for k, v in sorted(agg.items(), key=lambda x: -x[1]):
                if v: f.write("  %-28s %9d  %5.1f%%\n" % (k, v, 100.0 * v / max(1, tot)))
            f.write("\ntop instructions by samples:\n")
            for r in top:
                f.write("  %s  %-70s %8s\n" % (r[0][-6:], r[1].strip()[:70], r[iS]))
    json.dump(traffic, open(out + "_traffic.json", "w"), indent=1)
    print("\n".join(lines))

if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
