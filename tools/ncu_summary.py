"""Summarise an .ncu-rep (here, no GPU needed): key metrics + top stall sites per kernel.
usage: python tools/ncu_summary.py prof_out/prof.ncu-rep [kernel-regex] [top-n]"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
rx = sys.argv[2] if len(sys.argv) > 2 else "chunk_kernel"
topn = int(sys.argv[3]) if len(sys.argv) > 3 else 25
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
KEEP = ["gpu__time_duration.sum", "sm__cycles_elapsed.avg.per_second",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sectors_op_red.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        # the shared-memory data pipe (128 B wavefront per clk and SM) is shared by MMA operand fetch (tc) and
        # the LSU: their sum is the number to watch
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum", "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_st.sum.pct_of_peak_sustained_elapsed",
        "l1tex__m_l1tex2xbar_req_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_tmem.avg.pct_of_peak_sustained_active", "sm__cycles_elapsed.max",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size"]
for r in rows[2:]:
    print("==", r[hdr.index("Kernel Name")][:70])
    for k in KEEP:
        if k in hdr:
            i = hdr.index(k)
            print(f"   {k:75s} {r[i]} {units[i]}")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-name", "regex:" + rx],
                     capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
h = rows[1]
isrc, isamp, iex = h.index("Source"), h.index("# Samples"), h.index("Instructions Executed")
stall = [(i, x) for i, x in enumerate(h) if x.startswith("stall_") and "Not Issued" not in x]
data = rows[2:]
tot = sum(int(r[isamp]) for r in data)
print("total samples", tot)
for i in sorted(sorted(range(len(data)), key=lambda i: -int(data[i][isamp]))[:topn]):
    r = data[i]
    st = sorted(((int(r[c]), x[6:]) for c, x in stall if int(r[c]) > 0), reverse=True)[:2]
    print(f"{i:5d} {100 * int(r[isamp]) / tot:5.1f}% ex={r[iex]:>10s} {r[isrc].strip()[:58]:58s} {st}")
# shared-memory wavefronts by opcode (LSU-visible part; TMA / mbarrier traffic is only in the raw totals)
if "L1 Wavefronts Shared" in h:
    iw = h.index("L1 Wavefronts Shared")
    agg = {}
    for r in data:
        if r[iw].isdigit() and int(r[iw]) > 0:
            words = r[isrc].split()
            op = words[1] if words[0].startswith("@") else words[0]
            a = agg.setdefault(op, [0, 0])
            a[0] += int(r[iw])
            a[1] += int(r[iex])
    print("shared-memory wavefronts by opcode:")
    for op, (w, x) in sorted(agg.items(), key=lambda kv: -kv[1][0])[:8]:
        print(f"   {op:16s} wavefronts {w:14d}  instructions {x:12d}  ({w / max(x, 1):.1f} per instruction)")
