#!/usr/bin/env python
"""Turn an Nsight Compute report into a small JSON summary.

    ncu -i gpurun_out/decode_tc.ncu-rep --page raw --csv > /tmp/raw.csv     # done by this script
    python tools/ncu_summary.py decode_tc.ncu-rep decode_tc_summary.json
"""
import csv
import io
import json
import subprocess
import sys

WANT = [
    "Kernel Name", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__bytes_read.sum.per_second", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], check=True, capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    res = []
    for vals in rows[2:]:
        d = {}
        for name in WANT:
            if name in hdr:
                i = hdr.index(name)
                d[name] = f"{vals[i]} {units[i]}".strip()
        res.append(d)
    json.dump(res[0] if len(res) == 1 else res, open(out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
