"""Export the judged metrics of an .ncu-rep (ncu --set full) into a small text summary.
usage: python tools/ncu_export.py report.ncu-rep > <kernel>.txt"""
import csv
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "sm__cycles_elapsed.max", "launch__grid_size", "launch__block_size", "launch__cluster_size",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warp_latency_issue_stalled_barrier.ratio",
    "smsp__average_warp_latency_issue_stalled_membar.ratio", "smsp__average_warp_latency_issue_stalled_short_scoreboard.ratio",
    "smsp__average_warp_latency_issue_stalled_wait.ratio", "smsp__average_warp_latency_issue_stalled_math_pipe_throttle.ratio",
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for rec in rows[2:]:
        d = dict(zip(hdr, rec))
        print("kernel:", d.get("Kernel Name", "?"))
        for k in KEYS:
            for h in hdr:
                if h == k:
                    print("  %-75s %s %s" % (h, d[h], units[hdr.index(h)]))
        print()


if __name__ == "__main__":
    main(sys.argv[1])
