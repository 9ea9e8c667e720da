"""Turn an .ncu-rep (ncu --set full) into a compact per-launch table (profiles/ is git-ignored)."""
import csv, io, subprocess, sys
rep, out = sys.argv[1], sys.argv[2]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
cols = [("Kernel Name", "kernel"), ("launch__grid_size", "grid"), ("launch__block_size", "block"), ("launch__registers_per_thread", "regs"),
        ("gpu__time_duration.sum", "time_us"), ("dram__bytes_read.sum", "dram_rd_MB"), ("dram__bytes_write.sum", "dram_wr_MB"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"), ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_pct"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue_pct"), ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_pct"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pct"), ("smsp__inst_executed.sum", "warp_instr")]
idx = [(hdr.index(c), n) for c, n in cols if c in hdr]
with open(out, "w") as f:
    f.write("# %s (ncu --set full --clock-control none; cold caches, serialised launches: compare SHARES, not absolutes)\n\n" % rep.split("/")[-1])
    f.write("| " + " | ".join(n for _, n in idx) + " | GB/s |\n|" + "---|" * (len(idx) + 1) + "\n")
    for r in data:
        vals = []
        d = {}
        for i, n in idx:
            v = r[i]
            d[n] = v
            if n == "kernel":
                v = v.replace("b200::", "")[:58]
            else:
                try: v = "%.3g" % float(v) if n not in ("grid", "block", "regs", "warp_instr") else str(int(float(v)))
                except ValueError: pass
            vals.append(v)
        try: gbs = "%.0f" % ((float(d["dram_rd_MB"]) + float(d["dram_wr_MB"])) / float(d["time_us"]) * 1e3)
        except Exception: gbs = ""
        f.write("| " + " | ".join(vals) + " | " + gbs + " |\n")
    f.write("\nunits: time %s, dram %s\n" % (units[hdr.index("gpu__time_duration.sum")], units[hdr.index("dram__bytes_read.sum")]))
print("wrote", out)
