"""dev tool: text summary of an .ncu-rep (raw page)"""
import csv, subprocess, sys
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
want = ['Kernel Name', 'Grid Size', 'Block Size', 'gpu__time_duration.sum', 'launch__registers_per_thread', 'launch__occupancy_limit_registers',
        'launch__occupancy_limit_shared_mem', 'launch__waves_per_multiprocessor', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'smsp__warps_active.avg.per_cycle_active', 'smsp__warps_eligible.avg.per_cycle_active', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed.avg.per_cycle_active', 'smsp__inst_executed.sum', 'smsp__thread_inst_executed_per_inst_executed.ratio',
        'sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active', 'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'l1tex__throughput.avg.pct_of_peak_sustained_active',
        'dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__t_bytes.sum',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'smsp__inst_executed_op_local_ld.sum', 'smsp__inst_executed_op_local_st.sum']
for r in rows[2:]:
    print("=" * 100)
    for w in want:
        if w in idx:
            print("%-72s %s %s" % (w, r[idx[w]], units[idx[w]]))
    print("-- warp stall reasons (warps stalled per issue-active cycle) --")
    st = []
    for h in hdr:
        if h.startswith('smsp__average_warps_issue_stalled') and h.endswith('_per_issue_active.ratio'):
            st.append((float(r[idx[h]]), h.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', '')))
    for v, n in sorted(st, reverse=True)[:8]:
        print("   %-28s %.2f" % (n, v))
