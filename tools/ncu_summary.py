"""Summarise an .ncu-rep (captured with `ncu --set full --clock-control none --import-source on`) as a markdown
table: one row per captured kernel with the metrics the H100 profiling recipe asks for.

    python tools/ncu_summary.py bench_out/prof_step.ncu-rep > profiles/r1_ncu_step.md
"""
import csv
import subprocess
import sys

COLS = [
    ("Kernel Name", "kernel"),
    ("gpu__time_duration.sum", "time"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM %"),
    ("sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "tensor pipe %"),
    ("gpu__compute_memory_throughput.avg.pct_of_peak_sustained_elapsed", "mem %"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM %"),
    ("dram__bytes_read.sum", "DRAM rd"),
    ("dram__bytes_write.sum", "DRAM wr"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1 %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "occupancy %"),
    ("smsp__cycles_active.avg", "SMSP active cyc"),
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units, body = rows[0], rows[1], rows[2:]
    idx = {}
    for i, h in enumerate(hdr):
        idx.setdefault(h, i)
        idx.setdefault(h.split(".TriageCompute.")[-1], i)
    cols = [(k, lbl) for k, lbl in COLS if k in idx]
    print(f"# ncu summary of `{path}`\n")
    print("| # | " + " | ".join(f"{lbl}{' [' + units[idx[k]] + ']' if units[idx[k]] else ''}" for k, lbl in cols) + " |")
    print("|" + "---|" * (len(cols) + 1))
    for n, r in enumerate(body):
        cells = []
        for k, _ in cols:
            v = r[idx[k]]
            if k == "Kernel Name":
                v = v.replace("|", "/")[:70]
            else:
                try:
                    v = f"{float(v):.4g}"
                except ValueError:
                    pass
            cells.append(v)
        print(f"| {n} | " + " | ".join(cells) + " |")


if __name__ == "__main__":
    main(sys.argv[1])
