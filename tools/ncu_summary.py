#!/usr/bin/env python
"""Summarise an .ncu-rep (one kernel launch) into a small text file.

    python tools/ncu_summary.py k1_full.ncu-rep k1_full.txt [frames_in_launch]
"""
import csv
import json
import subprocess
import sys

WANT = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__warps_eligible.avg.per_cycle_active", "sm__cycles_elapsed.max",
    "smsp__warp_issue_stalled_barrier_per_warp_active.pct", "smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_math_pipe_throttle_per_warp_active.pct",
    "smsp__warp_issue_stalled_mio_throttle_per_warp_active.pct", "smsp__warp_issue_stalled_wait_per_warp_active.pct",
    "smsp__warp_issue_stalled_not_selected_per_warp_active.pct", "smsp__warp_issue_stalled_dispatch_stall_per_warp_active.pct",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    frames = float(sys.argv[3]) if len(sys.argv) > 3 else None
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units, vals = rows[0], rows[1], rows[2]
    d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
    lines = ["ncu --set full --clock-control none summary of %s" % rep, "kernel: %s" % d.get("Kernel Name", ("?",))[0], ""]
    for w in WANT:
        if w in d:
            lines.append("%-78s %18s %s" % (w, d[w][0], d[w][1]))
    if frames:
        def f(name):
            v, u = d[name]
            v = float(v.replace(",", ""))
            return v * {"Mbyte": 1e6, "Gbyte": 1e9, "Kbyte": 1e3, "byte": 1.0}.get(u, 1.0)
        rd, wr = f("dram__bytes_read.sum"), f("dram__bytes_write.sum")
        inst = float(d["smsp__inst_executed.sum"][0].replace(",", ""))
        lines += ["", "units (frames or model steps) in this launch: %d" % frames,
                  "dram bytes per unit: read %.1f  write %.1f  total %.1f" % (rd / frames, wr / frames, (rd + wr) / frames),
                  "thread-level instructions per unit (warp inst x 32): %.0f" % (inst * 32 / frames)]
        json.dump({"dram_bytes_per_launch": rd + wr, "units_in_launch": frames, "dram_bytes_per_unit": (rd + wr) / frames,
                   "thread_instr_per_unit": inst * 32 / frames, "source": rep}, open(out.replace(".txt", ".json"), "w"))
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
