#!/usr/bin/env python3
"""Summarise an .ncu-rep (here, no GPU needed): headline metrics, stall reasons, hottest source lines.
usage: python profiles/ncu_summarize.py prof.ncu-rep [top_n] [kernel-name substring]"""
import csv, io, subprocess, sys

rep = sys.argv[1]
top = int(sys.argv[2]) if len(sys.argv) > 2 else 30
want = sys.argv[3] if len(sys.argv) > 3 else None
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
sel = 2
if want:
    ki = rows[0].index("Kernel Name")
    sel = [i for i in range(2, len(rows)) if want in rows[i][ki]][0]
d = {h: (u, v) for h, u, v in zip(rows[0], rows[1], rows[sel])}
print("kernel:", d["Kernel Name"][1][:80])
for k in ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
          "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
          "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
          "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
          "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "smsp__thread_inst_executed_per_inst_executed.ratio",
          "lts__t_bytes.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]:
    if k in d:
        print(f"{k:70s} {d[k][1]} {d[k][0]}")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--print-source", "cuda,sass", "--csv"],
                     capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
hdr = None
cur = None
agg = []
stall_tot = {}
active = want is None
for r in rows:
    if len(r) >= 2 and r[0] in ("Kernel Name", "Function Name"):
        active = want is None or want in r[1]
        continue
    if not active:
        continue
    if len(r) >= 2 and r[0] == "File Path":
        cur = r[1].split("/")[-1]
        continue
    if len(r) > 8 and r[0] == "Line No":
        hdr = r
        continue
    if hdr and len(r) > 8 and r[2] == "-" and r[0].isdigit():
        try:
            agg.append((cur, int(r[0]), r[1].strip()[:100], int(r[7] or 0), int(r[6] or 0)))
        except ValueError:
            pass
    if hdr and len(r) > 8 and r[2] != "-" and r[2].startswith("0x"):
        for i, h in enumerate(hdr):
            if h.startswith("stall_") and "Not Issued" not in h and i < len(r):
                try:
                    stall_tot[h] = stall_tot.get(h, 0) + int(r[i])
                except ValueError:
                    pass
ti, ts = sum(a[3] for a in agg) or 1, sum(a[4] for a in agg) or 1
print("\nstall reasons (sampled):")
T = sum(stall_tot.values()) or 1
for s, v in sorted(stall_tot.items(), key=lambda x: -x[1])[:8]:
    print(f"  {s:26s} {100 * v / T:5.1f}%")
print(f"\nhottest source lines (of {ti} warp-instructions, {ts} samples):")
for a in sorted(agg, key=lambda a: -a[3])[:top]:
    print(f"  {a[0]}:{a[1]:4d} inst {100 * a[3] / ti:5.1f}%  samp {100 * a[4] / ts:5.1f}%  {a[2]}")
