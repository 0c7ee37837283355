#!/usr/bin/env python
"""Selected figures of one `ncu --set full` report: selected raw metrics,
the warp-state sample breakdown, executed warp instructions by opcode.   tools/ncu_raw_summary.py <report> <samples>"""
import collections, csv, re, subprocess, sys
rep, samples = sys.argv[1], int(sys.argv[2])
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rr = list(csv.reader(raw.split("\n"))); h, u, r = rr[0], rr[1], rr[2]
keep = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
        "sm__inst_executed_pipe_alu.sum.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.sum.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.sum.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.sum.pct_of_peak_sustained_active",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed"]
print(f"# {rep}: first captured launch")
for i, n in enumerate(h):
    if n in keep:
        print(f"{n} [{u[i]}] = {r[i]}")
st = [(float(r[i]), n) for i, n in enumerate(h) if "pcsamp_warps_issue_stalled" in n and not n.endswith("not_issued") and r[i] not in ("", "n/a")]
tot = sum(v for v, _ in st)
print("# warp-state samples (smsp__pcsamp_warps_issue_stalled_*), share of all samples")
for v, n in sorted(st, reverse=True)[:12]:
    print(f"{n.replace('smsp__pcsamp_warps_issue_stalled_', ''):32s} {100 * v / tot:6.2f} %")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(src.split("\n"))); hdr = rows[1]; data = [x for x in rows[2:] if len(x) == len(hdr)]
si, ie = hdr.index("Source"), hdr.index("Instructions Executed")
agg = collections.Counter()
for x in data:
    m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_]+)", x[si].strip())
    if m:
        agg[m.group(2)] += int(x[ie])
t = sum(agg.values())
print(f"# executed warp instructions by opcode (SASS page): total {t} = {t * 32 / samples:.1f} issue slots per sample")
for k, v in agg.most_common(26):
    print(f"{k:10s} {v:12d} {100 * v / t:5.1f} %  {v * 32 / samples:6.2f} slots/sample")
