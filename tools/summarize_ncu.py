"""Summarise an .ncu-rep (read here, no GPU needed) into the given .md file:
duration, DRAM bytes, throughput %, registers, occupancy, top stall reasons."""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "smsp__inst_executed.sum", "sm__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_xu.sum", "lts__t_bytes.sum",
    "l1tex__t_bytes_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_st.sum",
    "smsp__average_warp_latency_issue_stalled_long_scoreboard.pct", "smsp__average_warp_latency_issue_stalled_short_scoreboard.pct",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "launch__waves_per_multiprocessor",
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    if len(rows) < 3:
        print("no rows in", rep)
        return
    hdr, units = rows[0], rows[1]
    lines = [f"# ncu summary of `{rep}`", ""]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        lines.append(f"## {d.get('Kernel Name', '?')}  (launch id {d.get('ID', '?')})")
        lines.append("")
        lines.append("| metric | value | unit |")
        lines.append("|---|---|---|")
        for k in KEYS:
            if k in d:
                lines.append(f"| {k} | {d[k]} | {units[hdr.index(k)]} |")
        stalls = sorted(((float(d[k].replace(',', '')), k) for k in d if "issue_stalled" in k and k.endswith("_per_issue_active.ratio") and d[k]),
                        reverse=True)[:6]
        if stalls:
            lines.append("")
            lines.append("top stall reasons (warps stalled per issue-active cycle):")
            for v, k in stalls:
                lines.append(f"- {k.split('issue_stalled_')[1].split('_per_issue')[0]}: {v:.2f}")
        lines.append("")
    open(out, "w").write("\n".join(lines) + "\n")
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
