"""Condense ncu captures (ncu --set full) into a small JSON.
   python tools/ncu_summary.py capture.ncu-rep|capture_raw.csv [...]   -> JSON on stdout: {file: {metric: [value, unit]}}
A *_raw.csv is the output of `ncu -i x.ncu-rep --page raw --csv` (tools/gpu_job.sh exports it on the GPU box)."""
import csv
import io
import json
import os
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size", "launch__occupancy_limit_shared_mem",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "sm__cycles_elapsed.avg", "sm__cycles_active.avg", "sm__cycles_elapsed.max",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__ops_path_tensor_src_int8.avg.pct_of_peak_sustained_elapsed", "sm__ops_path_tensor_op_utcimma_src_int8_sparsity_off.avg.pct_of_peak_sustained_elapsed",
    "sm__ops_path_tensor_op_utchmma_src_bf16_dst_fp32_sparsity_off.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__mem_tensor_reads_op_ldt.sum.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
]


def read(path):
    if path.endswith(".csv"):
        out = open(path).read()
    else:
        out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    res = []
    for vals in rows[2:]:
        d = {"Kernel Name": [vals[hdr.index("Kernel Name")], ""]}
        for h, u, v in zip(hdr, units, vals):
            if h in KEYS:
                d[h] = [v, u]
        res.append(d)
    return res[0] if len(res) == 1 else res


if __name__ == "__main__":
    json.dump({os.path.basename(p): read(p) for p in sys.argv[1:]}, sys.stdout, indent=1)
    print()
