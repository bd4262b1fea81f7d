"""Summarise an .ncu-rep (ncu --set full) into a small text table.
usage: python tools/ncu_summary.py prof.ncu-rep "<title>" > prof.txt"""
import csv
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram_read"),
    ("dram__bytes_write.sum", "dram_write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"),
    ("lts__t_bytes.sum", "l2_bytes"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_pct"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pct"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_active_pct"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__cluster_size", "cluster"),
    ("launch__shared_mem_per_block_dynamic", "dyn_smem"),
    ("smsp__inst_executed.sum", "warp_insts"),
    ("sm__inst_executed.avg.per_cycle_elapsed", "ipc_per_sm"),
    ("smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "stall_long_scoreboard"),
    ("smsp__average_warp_latency_issue_stalled_short_scoreboard.ratio", "stall_short_scoreboard"),
    ("smsp__average_warp_latency_issue_stalled_barrier.ratio", "stall_barrier"),
    ("smsp__average_warp_latency_issue_stalled_membar.ratio", "stall_membar"),
    ("smsp__average_warp_latency_issue_stalled_wait.ratio", "stall_wait"),
    ("smsp__average_warp_latency_issue_stalled_math_pipe_throttle.ratio", "stall_math_throttle"),
    ("smsp__average_warp_latency_issue_stalled_lg_throttle.ratio", "stall_lg_throttle"),
    ("smsp__average_warp_latency_issue_stalled_not_selected.ratio", "stall_not_selected"),
    ("smsp__average_warp_latency_issue_stalled_sleeping.ratio", "stall_sleeping"),
    ("smsp__average_warp_latency_issue_stalled_no_instruction.ratio", "stall_no_instruction"),
]


def main():
    rep, title = sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else ""
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(l for l in out.splitlines() if not l.startswith("==")))
    hdr, units = rows[0], rows[1]
    print("# " + title)
    print("# source: %s (ncu --set full --clock-control none; per-launch, cold-cache, serialised)" % rep)
    for row in rows[2:]:
        name = row[hdr.index("Kernel Name")]
        print("\n" + name[:150])
        for key, label in WANT:
            if key in hdr:
                i = hdr.index(key)
                print("    %-18s %s %s" % (label, row[i], units[i]))


if __name__ == "__main__":
    main()
