"""Summarise an .ncu-rep (ncu --set full) into a per-launch text block.
usage: python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv, io, subprocess, sys

METRICS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "smsp__inst_executed.sum",
           "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
           "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
           "l1tex__t_requests_pipe_lsu_mem_global_op_red.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum",
           "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
           "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
           "lts__t_sector_hit_rate.pct", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
           "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__thread_inst_executed_per_inst_executed.ratio"]

def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names, units = rows[hdr], rows[hdr + 1]
    col = {n: i for i, n in enumerate(names)}
    for r in rows[hdr + 2:]:
        if len(r) < len(names): continue
        print("-----")
        print("Kernel Name =", r[col["Kernel Name"]][:150])
        for m in METRICS:
            if m in col: print(f"{m} = {r[col[m]]} {units[col[m]]}")
        stalls = []
        for n, i in col.items():
            if n.startswith("smsp__pcsamp_warps_issue_stalled_") and not n.endswith("_not_issued"):
                try: stalls.append((float(r[i]), n[len("smsp__pcsamp_warps_issue_stalled_"):]))
                except ValueError: pass
        print("top stall samples =", sorted(stalls, reverse=True)[:6])

if __name__ == "__main__":
    main(sys.argv[1])
