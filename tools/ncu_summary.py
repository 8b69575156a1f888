#!/usr/bin/env python
"""Condenses an `ncu --set full` report into a per-kernel table and the per-launch DRAM traffic of each kernel.

  tools/ncu_summary.py probe_out/X.ncu-rep probe_out/name   -> probe_out/name_summary.csv
                                                               probe_out/name_traffic.json
"""
import csv
import io
import json
import re
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__waves_per_multiprocessor", "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__issue_active.avg.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__cycles_elapsed.max",
    "smsp__cycles_elapsed.avg.per_second",
]
UNIT_SCALE = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    header, units, body = rows[0], rows[1], rows[2:]
    cols = [header.index(m) for m in METRICS if m in header]
    ki = header.index("Kernel Name")
    traffic = {}
    with open(out + "_summary.csv", "w", newline="") as fh:
        w = csv.writer(fh)
        w.writerow(["kernel"] + [header[c] for c in cols])
        w.writerow(["unit"] + [units[c] for c in cols])
        for r in body:
            name = re.sub(r"\(.*", "", r[ki]).replace("void ", "").replace("unnamed>::", "")
            name = re.sub(r"<.*", "", name)
            w.writerow([name] + [r[c] for c in cols])
            rd, wr = header.index("dram__bytes_read.sum"), header.index("dram__bytes_write.sum")
            total = float(r[rd]) * UNIT_SCALE[units[rd]] + float(r[wr]) * UNIT_SCALE[units[wr]]
            traffic[name] = {"dram_bytes_per_launch": total,
                             "duration_us": float(r[header.index("gpu__time_duration.sum")]) *
                             {"us": 1, "ns": 1e-3, "ms": 1e3}[units[header.index("gpu__time_duration.sum")]]}
    json.dump({"source": rep.split("/")[-1], "note": "one launch per kernel of a late frame; ncu replays each kernel "
               "with caches flushed, so DRAM bytes are cold-cache upper bounds of the in-pipeline traffic",
               "kernels": traffic}, open(out + "_traffic.json", "w"), indent=1)
    for k, v in traffic.items():
        print(f"{k:28s} {v['duration_us']:8.2f} us  dram {v['dram_bytes_per_launch'] / 1e6:8.2f} MB")


if __name__ == "__main__":
    main()
