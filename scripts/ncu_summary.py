"""Summarises .ncu-rep captures into markdown tables (runs without a GPU)."""
import csv
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("sm__cycles_elapsed.max", "SM cycles"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "XU (MUFU) pipe %"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput %"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "smem wavefronts %"),
    ("launch__registers_per_thread", "registers/thread"),
    ("launch__occupancy_limit_shared_mem", "CTAs/SM (smem limit)"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("smsp__inst_executed.sum", "warp instructions"),
]


def summarise(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, vals = rows[0], rows[1], rows[-1]
    name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
    d = {}
    for h, u, v in zip(hdr, units, vals):
        d[h] = (v, u)
    lines = [f"kernel: `{name}`", "", "| metric | value |", "|---|---|"]
    for k, label in KEYS:
        if k in d:
            lines.append(f"| {label} (`{k}`) | {d[k][0]} {d[k][1]} |")
    return "\n".join(lines)


if __name__ == "__main__":
    for pth in sys.argv[1:]:
        print(f"### {pth}\n")
        print(summarise(pth))
        print()
