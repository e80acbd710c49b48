"""Summarise an `ncu --set full` report (.ncu-rep) per kernel launch: duration, occupancy limiters, pipe utilisation
(tensor, XU/MUFU, FMA), issue-slot utilisation, DRAM / L2 throughput, top warp-stall reasons.
usage: python tools/ncu_kernel_summary.py report.ncu-rep > summary.txt"""
import csv
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rd = list(csv.reader(raw.splitlines()))
hdr, units = rd[0], rd[1]
want = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"), ("launch__block_size", "block"), ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("launch__occupancy_limit_shared_mem", "CTAs/SM limit (smem)"), ("launch__occupancy_limit_registers", "CTAs/SM limit (regs)"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "tensor (hmma subpipe) active %"),
    ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "XU (MUFU) pipe %"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "FMA pipe %"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe %"),
    ("dram__bytes_read.sum", "DRAM read"), ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput %"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_active", "L1/TEX throughput %"),
    ("smsp__inst_executed.sum", "warp instructions"),
]
ik = hdr.index("Kernel Name")
for r in rd[2:]:
    print("=" * 110)
    print(r[ik][:200])
    for key, label in want:
        if key in hdr:
            i = hdr.index(key)
            print(f"  {label:34s} {r[i]:>16s} {units[i]}")
    stalls = []
    for i, h in enumerate(hdr):
        if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio"):
            try:
                stalls.append((float(r[i]), h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]))
            except ValueError:
                pass
    tot = sum(s for s, _ in stalls) or 1.0
    print("  warp stall reasons (share of warp-cycles): " + ", ".join(f"{n} {100*s/tot:.0f}%" for s, n in sorted(stalls, reverse=True)[:6]))
