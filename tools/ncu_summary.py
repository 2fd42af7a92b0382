"""Summarise an .ncu-rep (read here, no GPU): key raw metrics, stall mix, hottest source lines.
usage: python tools/ncu_summary.py prof.ncu-rep [selections_in_launch] [warps_per_cta]"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
nsel = float(sys.argv[2]) if len(sys.argv) > 2 else None
warps = int(sys.argv[3]) if len(sys.argv) > 3 else 8


def ncu(*args):
    return subprocess.run(["ncu", "-i", rep, *args], capture_output=True, text=True).stdout


rows = list(csv.reader(io.StringIO(ncu("--page", "raw", "--csv"))))
hdr, units, vals = rows[0], rows[1], rows[2]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "smsp__sass_inst_executed_op_local_ld.sum", "smsp__sass_inst_executed_op_local_st.sum",
        "sm__cycles_elapsed.avg", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "launch__shared_mem_per_block_dynamic",
        # shared-memory data pipe (LDS/STS wavefronts and tensor-core operand reads share it) and the tensor pipe
        "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active"]
print("== raw metrics")
for i, h in enumerate(hdr):
    if h in want:
        print(f"  {h:70s} {vals[i]:>16s} {units[i]}")
    if h == "smsp__inst_executed.sum":
        ninst = float(vals[i])
if nsel:
    print(f"  warp-instructions per selection: {ninst / nsel:.0f}  (per warp-step: {ninst / nsel / warps:.0f})")

rows = list(csv.reader(io.StringIO(ncu("--page", "source", "--csv", "--print-source", "cuda,sass"))))
cur, hdr, agg, stalls = None, None, [], {}
for r in rows:
    if len(r) == 2 and r[0] == "File Path":
        cur = r[1].split("/")[-1]
        continue
    if len(r) > 2 and r[0] == "Line No":
        hdr = r
        continue
    if hdr and len(r) == len(hdr):
        if r[0] != "":
            agg.append((int(r[hdr.index("# Samples")] or 0), int(r[hdr.index("Instructions Executed")] or 0), cur, r[0], r[1][:100]))
        else:
            for j, h in enumerate(hdr):
                if h.startswith("stall_") and "Not Issued" not in h:
                    try:
                        stalls[h] = stalls.get(h, 0) + int(r[j])
                    except ValueError:
                        pass
tot_s = sum(a[0] for a in agg) or 1
tot_i = sum(a[1] for a in agg) or 1
T = sum(stalls.values()) or 1
print("== stall mix (sampled)")
for k, v in sorted(stalls.items(), key=lambda x: -x[1])[:9]:
    print(f"  {k:26s} {100 * v / T:5.1f}%")
print("== hottest source lines (by samples)")
for a in sorted(agg, reverse=True)[:28]:
    per = f"{a[1] / nsel / warps:6.1f}" if nsel else ""
    print(f"  {100 * a[0] / tot_s:5.1f}%  inst {100 * a[1] / tot_i:5.1f}% {per}  {a[2]}:{a[3]}  {a[4]}")
