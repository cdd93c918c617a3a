"""Summarise an .ncu-rep (ncu --set full) into a small markdown table.
usage: ncu_summary.py report.ncu-rep out.md [title]"""
import csv, io, subprocess, sys
rep, out = sys.argv[1], sys.argv[2]
title = sys.argv[3] if len(sys.argv) > 3 else rep
txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(txt)))
hdr, units, data = rows[0], rows[1], rows[2:]
want = [
    ("Kernel Name", "kernel"), ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"), ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active", "tensor pipe (hmma subpipe) % active"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe cycles active %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
]
lines = [f"# {title}", "", f"source: `{rep}` (`ncu --set full --clock-control none --import-source on`), read with "
         "`ncu -i ... --page raw --csv`", ""]
seen = set()
ik = hdr.index("Kernel Name"); ig = hdr.index("launch__grid_size"); ism = hdr.index("launch__shared_mem_per_block_dynamic")
for r in data:
    sig = (r[ik], r[ig], r[ism])
    if sig in seen:
        continue                      # repeated launches of the same configuration: keep the first
    seen.add(sig)
    lines.append("| metric | value |"); lines.append("|---|---|")
    for key, label in want:
        for i, h in enumerate(hdr):
            if h == key:
                lines.append(f"| {label} (`{key}`) | {r[i]} {units[i]} |")
    lines.append("")
open(out, "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
