"""Condense `ncu --page raw --csv` into one line per kernel launch with the metrics the roofline needs.
usage: summarize_ncu_raw.py raw.csv [--traffic-json <out.json> workload source-file-name]
(the optional arguments also record dram read + write bytes summed over the listed launches for bench.py's roofline.traffic)"""
import csv
import sys

KEYS = [("gpu__time_duration.sum", "dur"), ("dram__bytes_read.sum", "dram_rd"), ("dram__bytes_write.sum", "dram_wr"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram%"),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm%"),
        ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "fma%"),
        ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma_inst%"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor%"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "occ%"),
        ("launch__registers_per_thread", "regs"), ("launch__occupancy_limit_shared_mem", "occ_lim_smem"),
        ("launch__grid_size", "grid"), ("launch__shared_mem_per_block_dynamic", "dsmem"),
        ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "bank_conf"),
        ("smsp__average_warp_latency_issue_stalled_short_scoreboard", "stall_short_sb"),
        ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "st_long"),
        ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "st_short"),
        ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "st_bar"),
        ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "st_mio"),
        ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "st_math"),
        ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "st_notsel"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue%")]
with open(sys.argv[1], newline="") as f:
    rd = list(csv.reader(f))
hdr = rd[0]
units = rd[1]
idx = {h: i for i, h in enumerate(hdr)}
print("columns:", " ".join(k for _, k in KEYS if _ in idx))
for row in rd[2:]:
    if len(row) < len(hdr):
        continue
    name = row[idx["Kernel Name"]].split("(")[0][-40:]
    out = [f"{row[idx['ID']]:>5s}", f"{name:40s}"]
    for key, short in KEYS:
        if key in idx:
            out.append(f"{short}={row[idx[key]]}{units[idx[key]] if short in ('dur', 'dram_rd', 'dram_wr') else ''}")
    for h_, i_ in idx.items():      # anything tensor-pipe related that is non-zero (the tensor pipe shows up under several names)
        if ("tensor" in h_ or "pipe_tc" in h_ or "tmem" in h_) and h_ not in dict(KEYS):
            v_ = row[i_]
            if v_ not in ("0", "0.000000", "", "n/a"):
                out.append(f"{h_}={v_}")
    print(" ".join(out))

if len(sys.argv) >= 6 and sys.argv[2] == "--traffic-json":
    import json
    import os
    path, workload, source = sys.argv[3], sys.argv[4], sys.argv[5]
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    total, n = 0.0, 0
    for row in rd[2:]:
        if len(row) < len(hdr):
            continue
        for key in ("dram__bytes_read.sum", "dram__bytes_write.sum"):
            if key in idx:
                total += float(row[idx[key]].replace(",", "")) * scale.get(units[idx[key]], 1.0)
        n += 1
    d = {}
    if os.path.exists(path):
        d = json.load(open(path))
    d[workload] = dict(bytes=total, launches=n, source=source)
    json.dump(d, open(path, "w"), indent=1)
