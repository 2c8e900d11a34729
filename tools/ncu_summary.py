"""Summarise an .ncu-rep (read with `ncu -i`, no GPU needed) into a small markdown/CSV pair
<out_prefix>.md / <out_prefix>.csv.

    python tools/ncu_summary.py prof_gemm.ncu-rep prof_gemm_summary
"""
import csv
import io
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.max",
]


def main(rep, out_prefix):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True,
                         text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {m: hdr.index(m) for m in METRICS if m in hdr}
    name_i = hdr.index("Kernel Name")
    with open(out_prefix + ".csv", "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["kernel"] + [f"{m} [{units[i]}]" for m, i in idx.items()])
        for r in rows[2:]:
            w.writerow([r[name_i][:120]] + [r[i] for i in idx.values()])
    with open(out_prefix + ".md", "w") as f:
        f.write(f"# ncu summary of `{rep}`\n\n")
        f.write("| kernel | time [us] | DRAM rd+wr [MB] | tensor pipe active % | LTS % | DRAM % | regs |\n")
        f.write("|---|---|---|---|---|---|---|\n")
        for r in rows[2:]:
            g = lambda m: r[idx[m]] if m in idx else "?"
            rd, wr = float(g("dram__bytes_read.sum")), float(g("dram__bytes_write.sum"))
            f.write(f"| `{r[name_i][:90]}` | {float(g('gpu__time_duration.sum')):.1f} | "
                    f"{rd + wr:.1f} | "
                    f"{float(g('sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active')):.1f} | "
                    f"{float(g('lts__throughput.avg.pct_of_peak_sustained_elapsed')):.1f} | "
                    f"{float(g('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed')):.1f} | "
                    f"{g('launch__registers_per_thread')} |\n")
    print("wrote", out_prefix + ".md/.csv")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
