"""Summarise an .ncu-rep (captured with --set full) into a small markdown table.
    python scripts/ncu_summary.py prof.ncu-rep summary.md "title"
"""
import csv
import io
import subprocess
import sys

METRICS = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram rd"),
    ("dram__bytes_write.sum", "dram wr"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %"),
    ("lts__t_sectors_srcunit_tex_op_read.sum", "L2 rd sectors"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps %"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
]


def main():
    rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else ""
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(out, "w") as f:
        f.write(f"# {title}\n\nSource: `{rep}` (ncu --set full --clock-control none; cold-cache, serialised launches)\n\n")
        f.write("| # | kernel | " + " | ".join(n for _, n in METRICS) + " |\n")
        f.write("|---|---|" + "---|" * len(METRICS) + "\n")
        for k, r in enumerate(rows[2:]):
            name = r[idx["Kernel Name"]].split("(")[0].replace("void ", "")
            cells = []
            for m, _ in METRICS:
                if m in idx:
                    v, u = r[idx[m]], units[idx[m]]
                    try:
                        v = f"{float(v):.4g}"
                    except ValueError:
                        pass
                    cells.append(f"{v} {u}".strip())
                else:
                    cells.append("n/a")
            f.write(f"| {k} | `{name}` | " + " | ".join(cells) + " |\n")


if __name__ == "__main__":
    main()
