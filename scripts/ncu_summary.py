"""Summarise an .ncu-rep (read here, no GPU needed) into a small text file.

    python scripts/ncu_summary.py prof.ncu-rep summary.txt
"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
    "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tma_cycles_active.avg.pct_of_peak_sustained_active", "dram__cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "smsp__warps_eligible.avg.per_cycle_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_st.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_st.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum",
    "lts__t_sector_hit_rate.pct", "lts__t_bytes.sum", "sm__sass_inst_executed_op_shared_st.sum",
    "smsp__pcsamp_warps_issue_stalled_long_scoreboard", "smsp__pcsamp_warps_issue_stalled_barrier",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    lines = []
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        lines.append(f"== kernel: {name}")
        for i, h in enumerate(hdr):
            if h in KEYS or "issue_stalled" in h and h.endswith("_per_warp_active.pct"):
                lines.append(f"{h:90s} {units[i]:12s} {r[i]}")
        rd = float(r[hdr.index("dram__bytes_read.sum")]) if "dram__bytes_read.sum" in hdr else 0
        wr = float(r[hdr.index("dram__bytes_write.sum")]) if "dram__bytes_write.sum" in hdr else 0
        u = units[hdr.index("dram__bytes_read.sum")] if "dram__bytes_read.sum" in hdr else ""
        lines.append(f"traffic (dram read+write) = {rd + wr} {u}")
    open(out, "w").write(f"# summary of {rep} (ncu --set full --clock-control none)\n" + "\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
