#!/usr/bin/env python
"""Aggregate an ncu report's per-SASS-instruction counters by CUDA source line.

    tools/ncu_by_line.py gpurun_out/prof.ncu-rep [kernel-substring] [top-n]

Needs the product built with -lineinfo (it is) and nvdisasm/cuobjdump from the toolkit.
Correlates `ncu --page source --csv` rows (in SASS order) with `nvdisasm -g` line markers
of the sm_90a cubin embedded in hacktv_b200/libhacktv_b200.so."""
import collections, csv, os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rep = sys.argv[1]
kern = sys.argv[2] if len(sys.argv) > 2 else "k_lines"
topn = int(sys.argv[3]) if len(sys.argv) > 3 else 45

with tempfile.TemporaryDirectory() as td:
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(ROOT, "hacktv_b200", "libhacktv_b200.so")], cwd=td, capture_output=True)
    cubin = [f for f in os.listdir(td) if "sm_90a" in f][0]
    dis = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(td, cubin)], capture_output=True, text=True).stdout.split("\n")
    # a report with several kernels: NCU_KERNEL=<base name> selects one (ncu --kernel-name)
    sel = ["--kernel-name", os.environ["NCU_KERNEL"]] if os.environ.get("NCU_KERNEL") else []
    src_csv = subprocess.run(["ncu", "-i", rep] + sel + ["--page", "source", "--csv"], capture_output=True, text=True).stdout
    raw_csv = subprocess.run(["ncu", "-i", rep] + sel + ["--page", "raw", "--csv"], capture_output=True, text=True).stdout

# several sections can match (k_raster / k_raster_secam, template instantiations): take the shortest
# name, and pass a longer substring (e.g. k_mod_mmaILi256) to pick an instantiation
starts = sorted((i for i, l in enumerate(dis) if l.startswith(".text.") and kern in l), key=lambda i: len(dis[i]))
start = starts[0]
ends = [i for i, l in enumerate(dis) if l.startswith(".text.") and i > start]
end = ends[0] if ends else len(dis)
seq, cur = [], None
for l in dis[start:end]:
    m = re.search(r'//## File "(.*?)", line (\d+)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2))); continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l):
        seq.append((cur, l.strip()))

rows = list(csv.reader(src_csv.split("\n")))
hdr = rows[1]; data = [r for r in rows[2:] if len(r) == len(hdr)]
ie, ss = hdr.index("Instructions Executed"), hdr.index("# Samples")
n = len(seq)
data = data[:n]
agg, samp = collections.Counter(), collections.Counter()
for (ln, _), r in zip(seq, data):
    agg[ln] += int(r[ie]); samp[ln] += int(r[ss])
tot, ts = sum(agg.values()), sum(samp.values())
srcs = {}
def text_of(ln):
    if not ln:
        return ""
    f, n = ln
    if f not in srcs:
        try:
            srcs[f] = open(os.path.join(ROOT, "hacktv_b200", "csrc", f)).read().split("\n")
        except OSError:
            srcs[f] = []
    pre = "" if f == "htv_kernels.cu" else "[" + f + "] "
    return pre + (srcs[f][n - 1].strip()[:100] if 0 < n <= len(srcs[f]) else "")
print(f"# {kern}: {n} SASS instructions, {tot} warp-instructions executed, {ts} stall samples")
for ln, c in agg.most_common(topn):
    text = text_of(ln)
    print(f"{(ln[1] if ln else 0):5d} {100 * c / tot:5.1f}% inst {100 * samp[ln] / max(ts, 1):5.1f}% stall | {text}")

rr = list(csv.reader(raw_csv.split("\n")))
h, u, r0 = rr[0], rr[1], rr[2]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.sum.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.sum.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.sum.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.sum.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.sum.pct_of_peak_sustained_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__shared_mem_per_block_dynamic", "lts__t_bytes.sum", "launch__grid_size", "launch__block_size"]
print("# raw metrics (first captured launch)")
for i, name in enumerate(h):
    if name in want:
        print(f"{name} [{u[i]}] = {r0[i]}")
stall = [(float(r0[i]), name) for i, name in enumerate(h) if "smsp__average_warp" in name and "issue_stalled" in name and name.endswith("_per_warp_active.pct") ] 
for v, name in sorted(stall, reverse=True)[:8]:
    print(f"{name} = {v:.1f}")
