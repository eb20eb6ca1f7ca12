"""Per-kernel summary (one CSV row per kernel launch) of an `ncu --set full` report: duration, DRAM bytes, registers, issue / tensor-pipe
utilisation. usage (CPU container, on a .ncu-rep brought back from the GPU box):
  python tools/ncu_summary.py prof.ncu-rep > ncu_kernels.csv"""
import csv
import re
import subprocess
import sys

COLS = [("gpu__time_duration.sum", "gpu__time_duration.sum [us]", 1.0),
        ("dram__bytes_read.sum", "dram__bytes_read.sum [Mbyte]", 1.0),
        ("dram__bytes_write.sum", "dram__bytes_write.sum [Mbyte]", 1.0),
        ("launch__registers_per_thread", "launch__registers_per_thread [register/thread]", 1.0),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed [%]", 1.0),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active [%]", 1.0),
        ("smsp__inst_executed.sum", "smsp__inst_executed.sum [inst]", 1.0),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active [%]", 1.0),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active [%]", 1.0),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed [%]", 1.0),
        ("lts__t_bytes.sum", "lts__t_bytes.sum [Mbyte]", 1.0),
        ("launch__grid_size", "launch__grid_size []", 1.0), ("launch__block_size", "launch__block_size []", 1.0)]
UNIT = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}


def main():
    out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units = rows[0], rows[1]
    ki = h.index("Kernel Name")
    w = csv.writer(sys.stdout)
    w.writerow(["kernel"] + [c[1] for c in COLS])
    for r in rows[2:]:
        name = re.sub(r"\(.*", "", r[ki]).replace("void ", "").replace("<unnamed>::", "").strip()
        vals = []
        for key, _, _ in COLS:
            if key not in h:
                vals.append("")
                continue
            i = h.index(key)
            try:
                v = float(r[i].replace(",", ""))
            except ValueError:
                vals.append(r[i])
                continue
            v *= UNIT.get(units[i], 1.0)
            vals.append("%.6f" % v)
        w.writerow([name] + vals)


if __name__ == "__main__":
    main()
