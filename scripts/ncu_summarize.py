"""Reduce .ncu-rep files to the metrics the profiling recipe asks for (CSV per report, one row per kernel launch).

    python scripts/ncu_summarize.py gpurun_out/ncu/*.ncu-rep --out profiles/
"""
import csv
import io
import os
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "lts__t_bytes.sum", "l1tex__t_bytes.sum", "smsp__cycles_active.avg", "launch__occupancy_limit_registers",
        "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"]


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else "profiles"
    os.makedirs(out, exist_ok=True)
    for rep in args:
        raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(raw)))
        if len(rows) < 3:
            print("no data in", rep)
            continue
        hdr = rows[0]
        cols = [i for i, h in enumerate(hdr) if h in ("Kernel Name", "ID") or any(h == k for k in KEYS)]
        name = os.path.join(out, "ncu_" + os.path.basename(rep).replace(".ncu-rep", "") + ".csv")
        with open(name, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow([hdr[i] for i in cols])
            w.writerow([rows[1][i] for i in cols])  # units
            for r in rows[2:]:
                w.writerow([r[i][:90] if hdr[i] == "Kernel Name" else r[i] for i in cols])
        print("wrote", name, len(rows) - 2, "launches")


if __name__ == "__main__":
    main()
