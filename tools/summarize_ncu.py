"""Text summary of an .ncu-rep (duration, DRAM bytes, pipes, stall reasons, hottest source lines).
usage: python tools/summarize_ncu.py prof.ncu-rep > prof.txt"""
import csv, io, subprocess, sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
for vals in rows[2:]:
    d = dict(zip(hdr, vals)); u = dict(zip(hdr, units))
    print("kernel:", d.get("Kernel Name"), "grid", d.get("Grid Size"), "block", d.get("Block Size"))
    keys = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
            "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active",
            "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
            "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
            "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__inst_executed.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
            "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum"]
    for k in keys:
        if k in d: print(f"  {k:75s} {d[k]:>18s} {u.get(k, '')}")
    st = [(float(d[h]), h.replace("smsp__pcsamp_warps_issue_stalled_", "")) for h in hdr
          if "pcsamp_warps_issue_stalled" in h and not h.endswith("not_issued") and d[h] not in ("", "n/a")]
    tot = sum(x for x, _ in st) or 1
    print("  stall reasons (pc sampling): " + ", ".join(f"{h} {100 * x / tot:.1f}%" for x, h in sorted(st, reverse=True)[:8]))
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
cur, data = None, []
for r in csv.reader(io.StringIO(src)):
    if not r: continue
    if r[0] == "File Path": cur = r[1].split("/")[-1]; continue
    if r[0].isdigit():
        try: data.append((float(r[4]), float(r[7]), cur, int(r[0]), r[1].strip()))
        except ValueError: pass
tot = sum(x[0] for x in data) or 1
print("  hottest source lines (share of stall samples, warp instructions executed):")
for s, n, f, ln, text in sorted(data, reverse=True)[:14]:
    print(f"    {100 * s / tot:5.2f}% {int(n):>12d}  {f}:{ln}  {text[:100]}")
