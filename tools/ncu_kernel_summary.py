"""Selected `ncu --set full` metrics of the kernels of a report, one block per launch.
Usage: python tools/ncu_kernel_summary.py report.ncu-rep [name-regex]"""
import csv
import io
import re
import subprocess
import sys

METRICS = [
    ("gpu__time_duration.sum", "duration"),
    ("sm__cycles_elapsed.max", "SM cycles"),
    ("launch__grid_size", "grid"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__shared_mem_per_block_dynamic", "dynamic smem / block"),
    ("launch__occupancy_limit_shared_mem", "occupancy limit (smem), blocks / SM"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU pipe"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "FMA pipe"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg", "tensor (HMMA sub-pipe) active cycles"),
    ("sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "tensor pipe active (of peak)"),
    ("smsp__inst_executed_op_shfl.sum", "shuffle instructions"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "shared-memory wavefronts"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared-memory bank conflicts"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("lts__t_sectors_srcunit_tex_op_read.sum", "L2 read sectors (from SMs)"),
    ("l1tex__m_xbar2l1tex_read_bytes.sum", "L2 -> SM bytes"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall: short scoreboard (per issue)"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall: long scoreboard"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall: barrier"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall: MIO throttle"),
    ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall: not selected"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall: wait"),
]


def main():
    rep = sys.argv[1]
    rx = re.compile(sys.argv[2]) if len(sys.argv) > 2 else None
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    print(f"# {rep}: ncu --set full --clock-control none (per-launch times are cold-cache and serialised)")
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")]
        if rx and not rx.search(name):
            continue
        print(f"\n## {name.split('(')[0]}")
        for key, label in METRICS:
            if key in hdr:
                i = hdr.index(key)
                v = r[i]
                try:
                    v = f"{float(v):,.3f}".rstrip("0").rstrip(".")
                except ValueError:
                    pass
                print(f"  {label:46s} {v} {units[i]}")


if __name__ == "__main__":
    main()
