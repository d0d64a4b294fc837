"""Summarise an `ncu --set full` report into a markdown table incl. the top warp-stall reasons.

    python tools/ncu_summary.py x.ncu-rep "title" out.md
"""
import csv
import io
import subprocess
import sys

COLS = [
    ("us", "gpu__time_duration.sum"), ("grid", "launch__grid_size"), ("block", "launch__block_size"),
    ("regs", "launch__registers_per_thread"), ("smem KB", "launch__shared_mem_per_block_dynamic"),
    ("warps act %", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("issue %", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("tensor %", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
    ("L1 %", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed"), ("L2 %", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("DRAM %", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    ("DRAM rd MB", "dram__bytes_read.sum"), ("DRAM wr MB", "dram__bytes_write.sum"), ("inst M", "smsp__inst_executed.sum"),
]
UNIT = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}


def main():
    rep, title, out_md = sys.argv[1:4]
    if rep.endswith(".csv"):  # `ncu -i x.ncu-rep --page raw --csv` already run on the GPU box (the report itself is too big to ship)
        raw = open(rep).read()
    else:
        raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    stalls = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
    lines = [f"# {title}", "", "`ncu --set full --clock-control none` (kernels serialised, caches cold-ish: durations are NOT bench values).", "",
             "| kernel | " + " | ".join(c[0] for c in COLS) + " | top stalls (warps per issue slot) |", "|---|" + "---:|" * len(COLS) + "---|"]
    for r in rows[2:]:
        name = r[idx["Kernel Name"]].replace("void ", "").replace("<unnamed>::", "").split("(<")[0].replace("(int)", "").replace("(bool)", "")
        vals = []
        for label, key in COLS:
            if key not in idx:
                vals.append("n/a")
                continue
            v = float(r[idx[key]].replace(",", "") or 0)
            u = units[idx[key]]
            if "MB" in label:
                v *= UNIT.get(u, 1.0)
            elif "KB" in label:
                v *= {"byte": 1e-3, "Kbyte": 1.0, "Mbyte": 1e3}.get(u, 1.0)
            elif label == "inst M":
                v *= 1e-6
            vals.append(f"{v:.3g}")
        top = sorted(((float(r[idx[h]] or 0), h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]) for h in stalls), reverse=True)[:4]
        lines.append(f"| `{name}` | " + " | ".join(vals) + " | " + ", ".join(f"{n} {v:.2f}" for v, n in top) + " |")
    open(out_md, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
