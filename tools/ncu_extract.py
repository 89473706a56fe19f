"""Turns an ncu report into a small JSON summary of the per-kernel metrics.
    python tools/ncu_extract.py tool_out/r02_full.ncu-rep tool_out/r02_ncu_kernels_metrics.json"""
import csv
import json
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_uniform.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
        "launch__waves_per_multiprocessor", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum"]
STALLS = ["long_scoreboard", "short_scoreboard", "barrier", "membar", "math_pipe_throttle", "mio_throttle", "lg_throttle",
          "not_selected", "wait", "no_instruction", "dispatch_stall", "branch_resolving", "sleeping"]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    res = []
    for r in rows[2:]:
        m = {"kernel": r[idx["Kernel Name"]]}
        for k in KEYS:
            if k in idx:
                try:
                    m[k] = float(r[idx[k]].replace(",", ""))
                    m[k + ".unit"] = units[idx[k]]
                except ValueError:
                    pass
        for s in STALLS:
            k = f"smsp__average_warps_issue_stalled_{s}_per_issue_active.ratio"
            if k in idx:
                try:
                    m["stall_" + s] = float(r[idx[k]])
                except ValueError:
                    pass
        # normalise the byte counters to MB like the round-1 file
        for k in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
            if k in m:
                u = m.pop(k + ".unit", "byte")
                scale = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1e-6)
                m[k] = m[k] * scale
                m[k + ".unit"] = "MB"
        res.append(m)
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    for m in res:
        print(f"{m['kernel'][:60]:60s} {m.get('gpu__time_duration.sum', 0):8.1f} us  dram r/w {m.get('dram__bytes_read.sum', 0):7.1f}/{m.get('dram__bytes_write.sum', 0):6.1f} MB  "
              f"inst {m.get('smsp__inst_executed.sum', 0) / 1e6:6.2f} M  issue {m.get('smsp__issue_active.avg.pct_of_peak_sustained_active', 0):4.1f} %")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
