"""Summarise an .ncu-rep (raw page) into a handful of numbers (time, DRAM bytes, pipe use)."""
import csv
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed.sum", "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__warps_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "launch__grid_size", "launch__block_size",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "sm__cycles_elapsed.max",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
    "sm__pipe_tensor_op_hmma_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
]


def main(path, out=None):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    lines = []
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        lines.append(f"== {name}")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                lines.append(f"{k:75s} {r[i]:>18s} {units[i]}")
        for i, h in enumerate(hdr):
            if "issue_stalled" in h and h.endswith("per_warp_active.pct"):
                try:
                    if float(r[i]) >= 2.0:
                        lines.append(f"{h:75s} {r[i]:>18s} {units[i]}")
                except ValueError:
                    pass
    text = "\n".join(lines) + "\n"
    if out:
        open(out, "w").write(text)
    print(text)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else None)
