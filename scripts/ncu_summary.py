"""Summarise `ncu --set full` reports (read here, no GPU needed) into one JSON.
usage: ncu_summary.py out.json name=report.ncu-rep [name=report.ncu-rep ...]"""
import csv
import io
import json
import subprocess
import sys

WANT = {
    "gpu__time_duration.sum": "duration",
    "dram__bytes_read.sum": "dram_read",
    "dram__bytes_write.sum": "dram_write",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_throughput_pct",
    "gpu__compute_memory_throughput.avg.pct_of_peak_sustained_elapsed": "memory_throughput_pct",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "achieved_occupancy_pct",
    "sm__maximum_warps_per_active_cycle_pct": "theoretical_occupancy_pct",
    "launch__registers_per_thread": "registers_per_thread",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "launch__cluster_size": "cluster",
    "launch__shared_mem_per_block_dynamic": "dyn_smem",
    "launch__waves_per_multiprocessor": "waves_per_sm",
    "smsp__inst_executed.sum": "warp_instructions",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active": "pipe_fma_pct",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active": "pipe_xu_pct",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active": "pipe_alu_pct",
    "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active": "pipe_tensor_hmma_pct",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "pipe_tensor_pct",
    "sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active": "pipe_tensor_inst_pct",
    "smsp__issue_active.avg.pct_of_peak_sustained_active": "issue_active_pct",
    "smsp__cycles_active.avg": "smsp_cycles_active",
    "sm__cycles_elapsed.max": "sm_cycles_elapsed",
    "lts__t_sector_hit_rate.pct": "l2_hit_pct",
}


def read(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    head, units = rows[0], rows[1]
    res = []
    for r in rows[2:]:
        d = {"kernel": r[head.index("Kernel Name")][:160]}
        stalls = {}
        for i, h in enumerate(head):
            if h in WANT and r[i] != "":
                d[WANT[h]] = f"{r[i]} {units[i]}".strip()
            if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio") and r[i]:
                try:
                    stalls[h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]] = float(r[i].replace(",", ""))
                except ValueError:
                    pass
            if "tensor" in h and "pct" in h and r[i] not in ("", "0"):
                d.setdefault("tensor_metrics", {})[h] = r[i]
        d["top_stalls_warps_per_issue"] = dict(sorted(stalls.items(), key=lambda kv: -kv[1])[:6])
        res.append(d)
    return res


if __name__ == "__main__":
    out = {}
    for spec in sys.argv[2:]:
        name, rep = spec.split("=", 1)
        out[name] = read(rep)
    json.dump(out, open(sys.argv[1], "w"), indent=1)
    print(json.dumps(out, indent=1)[:6000])
