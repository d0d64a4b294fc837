"""Summarise an `ncu --set full` report (.ncu-rep) into a markdown table + a traffic JSON for bench.py.

    python tools/summarize_ncu.py native_full.ncu-rep "title" ncu.md [warp_corr_traffic.json]

The traffic JSON carries `mean_dram_bytes_per_launch` over the K-A (warp_corr*) launches of the capture: bench.py's `roofline.traffic`.
"""
import csv
import io
import json
import subprocess
import sys

COLS = [
    ("us", "gpu__time_duration.sum", 1.0),
    ("grid", "launch__grid_size", 1.0),
    ("regs", "launch__registers_per_thread", 1.0),
    ("warps act %", "sm__warps_active.avg.pct_of_peak_sustained_active", 1.0),
    ("SM %", "sm__throughput.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("L1 %", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("L2 %", "lts__throughput.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("DRAM %", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", 1.0),
    ("DRAM rd MB", "dram__bytes_read.sum", None),
    ("DRAM wr MB", "dram__bytes_write.sum", None),
    ("inst M", "smsp__inst_executed.sum", 1e-6),
    ("issue %", "smsp__issue_active.avg.pct_of_peak_sustained_active", 1.0),
    ("stall long-sb", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", 1.0),
    ("stall short-sb", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", 1.0),
    ("stall not-sel", "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", 1.0),
]


def to_mb(value, unit):
    v = float(value.replace(",", ""))
    return v * {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(unit, 1.0)


def main():
    rep, title, out_md = sys.argv[1:4]
    traffic_json = sys.argv[4] if len(sys.argv) > 4 else None
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    lines = [f"# {title}", "",
             "`ncu --set full --clock-control none --import-source on` on ONE eager forward (cold-ish caches, kernels serialised;",
             "durations here are NOT bench values).  Units: us, MB, percent of peak sustained.", "",
             "| kernel | " + " | ".join(c[0] for c in COLS) + " |", "|---|" + "---:|" * len(COLS)]
    traffic = {}
    for r in rows[2:]:
        name = r[idx["Kernel Name"]].replace("void ", "").replace("<unnamed>::", "")
        name = name.split("(")[0]
        vals = []
        rd = wr = 0.0
        for label, key, scale in COLS:
            if key not in idx:
                vals.append("n/a")
                continue
            v = r[idx[key]]
            if scale is None:
                mb = to_mb(v, units[idx[key]])
                vals.append(f"{mb:.2f}")
                if "read" in key:
                    rd = mb
                else:
                    wr = mb
            else:
                try:
                    vals.append(f"{float(v.replace(',', '')) * scale:.3g}")
                except ValueError:
                    vals.append(v)
        lines.append(f"| `{name}` | " + " | ".join(vals) + " |")
        traffic.setdefault(name, []).append(round((rd + wr) * 1e6))
    open(out_md, "w").write("\n".join(lines) + "\n")
    if traffic_json:
        ka = [b for name, launches in traffic.items() if "warp_corr" in name for b in launches]
        out = {"capture": title, "mean_dram_bytes_per_launch": (sum(ka) / len(ka)) if ka else None, "warp_corr_launches": len(ka),
               "dram_bytes_per_launch_by_kernel": traffic}
        json.dump(out, open(traffic_json, "w"), indent=1)
    print("\n".join(lines[:12]))


if __name__ == "__main__":
    main()
