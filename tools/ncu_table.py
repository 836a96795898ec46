"""Compact per-launch table from an `ncu --set full` report (run where ncu is installed; no GPU needed):

    python tools/ncu_table.py report.ncu-rep > kernels_ncu.txt

One row per profiled launch: duration, DRAM bytes read + written (the `traffic` of the roofline object), DRAM / tensor /
MUFU (XU) pipe utilisation, issue-slot utilisation, achieved occupancy, registers, dynamic shared memory, grid / block.
"""
import csv
import io
import re
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "dur_us", 1e-3),                                   # ns -> us
    ("dram__bytes_read.sum", "dram_rd_MB", 1e-6),
    ("dram__bytes_write.sum", "dram_wr_MB", 1e-6),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_%", 1),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_%", 1),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "xu_%", 1),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu_%", 1),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma_%", 1),
    ("sm__issue_active.avg.pct_of_peak_sustained_active", "issue_%", 1),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "occ_%", 1),
    ("lts__t_sector_hit_rate.pct", "l2_hit_%", 1),
    ("launch__registers_per_thread", "regs", 1),
    ("launch__shared_mem_per_block_dynamic", "smem_dyn", 1),
    ("launch__grid_size", "grid", 1),
    ("launch__block_size", "block", 1),
]
UNIT_SCALE = {"ns": 1.0, "us": 1e3, "ms": 1e6, "s": 1e9, "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def short(name):
    name = re.sub(r"\(.*", "", name)
    name = name.replace("fresco::", "").replace("void ", "")
    return name[:58]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    hdr, units = rows[hi], rows[hi + 1]
    col = {h: i for i, h in enumerate(hdr)}
    have = [(m, lab, sc) for m, lab, sc in WANT if m in col]
    missing = [m for m, _, _ in WANT if m not in col]
    print("# %s" % path)
    print("%-58s " % "kernel" + " ".join("%10s" % lab for _, lab, _ in have))
    for r in rows[hi + 2:]:
        if len(r) < len(hdr):
            continue
        out = []
        for m, lab, sc in have:
            v = r[col[m]].replace(",", "")
            try:
                f = float(v) * UNIT_SCALE.get(units[col[m]], 1.0) * sc
                out.append("%10.2f" % f if abs(f) < 1e6 else "%10.3g" % f)
            except ValueError:
                out.append("%10s" % v[:10])
        print("%-58s " % short(r[col["Kernel Name"]]) + " ".join(out))
    if missing:
        print("# metrics not in this report: " + ", ".join(missing))


if __name__ == "__main__":
    main(sys.argv[1])
