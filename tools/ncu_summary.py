"""Summarise an .ncu-rep (one kernel) as text: duration, throughput, stall mix, memory traffic.
usage: python tools/ncu_summary.py report.ncu-rep > summary.txt"""
import csv, io, subprocess, sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
h, u = rows[0], rows[1]
KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__waves_per_multiprocessor", "sm__cycles_elapsed.max",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__compute_memory_throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_bytes.sum", "l1tex__t_sector_hit_rate.pct",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__sass_inst_executed_op_local_ld.sum",
        "smsp__sass_inst_executed_op_local_st.sum", "smsp__average_warp_latency_per_inst_issued.ratio"]
for v in rows[2:]:
    d = dict(zip(h, v))
    print("kernel:", d.get("Kernel Name"), " id", d.get("ID"))
    for k in KEYS:
        if k in d:
            print("  %-72s %-12s %s" % (k, u[h.index(k)], d[k]))
    print("  warp stall reasons (average warps stalled per issue-active cycle):")
    st = [(float(d[k]), k) for k in h if "warps_issue_stalled" in k and k.endswith("per_issue_active.ratio") and d[k]]
    for val, k in sorted(st, reverse=True):
        print("    %-40s %.3f" % (k.split("issue_stalled_")[1].replace("_per_issue_active.ratio", ""), val))
    print()
