#!/usr/bin/env python3
"""Summarise an .ncu-rep (ncu -i ... --page raw --csv) into one CSV row per kernel launch (time, DRAM bytes, pipe
utilisation, stall reasons); tools/ncu_traffic_json.py condenses it per kernel family.  usage: ncu_summary.py <rep> [out.csv]"""
import csv
import subprocess
import sys

COLS = [
    ("gpu__time_duration.sum", "time_us"),
    ("dram__bytes_read.sum", "dram_rd"),
    ("dram__bytes_write.sum", "dram_wr"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pct"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue_pct"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu_pct"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma_pct"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu_pct"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "occ_pct"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("smsp__inst_executed.sum", "warp_inst"),
    ("smsp__warps_eligible.avg.per_cycle_active", "eligible"),
]
STALLS = ["long_scoreboard", "barrier", "short_scoreboard", "wait", "math_pipe_throttle", "not_selected", "sleeping", "no_instruction",
          "branch_resolving", "dispatch_stall", "mio_throttle", "lg_throttle", "membar"]


def main(rep, out=None):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    ix = {h: i for i, h in enumerate(hdr)}
    names = ["kernel"] + [c[1] for c in COLS] + ["stall_" + s for s in STALLS]
    res = []
    for r in rows[2:]:
        o = [r[ix["Kernel Name"]].split("(")[0][:60]]
        for m, _ in COLS:
            v = r[ix[m]] if m in ix else ""
            u = units[ix[m]] if m in ix else ""
            try:
                f = float(v.replace(",", ""))
                if u in ("ns", "nsecond"):
                    f /= 1000.0
                if u in ("ms", "msecond") and m == "gpu__time_duration.sum":
                    f *= 1000.0
                if u in ("s", "second") and m == "gpu__time_duration.sum":
                    f *= 1e6
                if u in ("Mbyte", "MB"):
                    f *= 1e6
                if u in ("Kbyte", "KB"):
                    f *= 1e3
                if u in ("Gbyte", "GB"):
                    f *= 1e9
                v = f"{f:.6g}"
            except ValueError:
                pass
            o.append(v)
        for s in STALLS:
            k = f"smsp__average_warps_issue_stalled_{s}_per_issue_active.ratio"
            o.append(r[ix[k]][:6] if k in ix else "")
        res.append(o)
    w = csv.writer(open(out, "w", newline="") if out else sys.stdout)
    w.writerow(names)
    w.writerows(res)


if __name__ == "__main__":
    main(*sys.argv[1:3])
