"""Summarise an .ncu-rep (read with `ncu -i`, no GPU needed) into a small CSV of the metrics below."""
import csv, subprocess, sys
KEEP = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sector_hit_rate.pct",
        "l1tex__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "smsp__inst_executed.sum",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "lts__t_bytes.sum"]
rep, out = sys.argv[1], sys.argv[2]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
tensor_cols = [h for h in hdr if "tensor" in h and h not in KEEP][:12]
cols = [k for k in KEEP if k in idx] + tensor_cols
with open(out, "w", newline="") as f:
    w = csv.writer(f)
    w.writerow(["kernel"] + cols)
    w.writerow(["unit"] + [units[idx[c]] for c in cols])
    for r in rows[2:]:
        w.writerow([r[idx["Kernel Name"]][:70]] + [r[idx[c]] for c in cols])
print("wrote", out, len(rows) - 2, "kernels")
