"""Summarise an .ncu-rep (read on the CPU box with `ncu -i`) into the handful of metrics DESIGN.md / bench.py cite.
usage: python scripts/ncu_summary.py prof.ncu-rep > summary.txt"""
import csv, subprocess, sys

WANT = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
    "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__inst_executed.sum", "sm__cycles_elapsed.avg", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
]
STALL = "smsp__average_warps_issue_stalled_"


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    for r in data:
        print("kernel:", r[ki][:100])
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                print(f"  {w:75s} {r[i]:>16s} {units[i]}")
        st = [(float(r[i]), h[len(STALL):].replace("_per_issue_active.ratio", "")) for i, h in enumerate(hdr)
              if h.startswith(STALL) and h.endswith("per_issue_active.ratio") and r[i] not in ("", "n/a")]
        st.sort(reverse=True)
        print("  warp stalls per issue (top):", ", ".join(f"{n}={v:.2f}" for v, n in st[:8]))
        print()


if __name__ == "__main__":
    main(sys.argv[1])
