"""Summarise an .ncu-rep (read here, without a GPU) into a few headline metrics per kernel."""
import csv, subprocess, sys
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
r = list(csv.reader(out.splitlines()))
hdr, units = r[0], r[1]
want = ['Kernel Name', 'launch__grid_size', 'launch__block_size', 'launch__registers_per_thread',
        'gpu__time_duration.sum', 'sm__cycles_elapsed.avg.per_second', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'smsp__inst_executed.sum', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
        'smsp__average_warp_latency_issue_stalled_long_scoreboard.pct', 'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_wait_per_issue_active.ratio', 'smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio',
        'smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio',
        'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem', 'sm__maximum_warps_per_active_cycle_pct',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'smsp__inst_executed_op_shared_atom.sum', 'lts__t_sector_hit_rate.pct']
idx = [(w, hdr.index(w)) for w in want if w in hdr]
for row in r[2:]:
    for w, i in idx:
        print("%-80s %s %s" % (w, row[i], units[i]))
    print("---")
