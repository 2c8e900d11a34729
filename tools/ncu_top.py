"""Digest an .ncu-rep on the machine that captured it (reports with --import-source are large):
per kernel the headline metrics plus the source/SASS lines with the most warp-stall samples.

    python tools/ncu_top.py x.ncu-rep x_top.txt [lines_per_kernel]
"""
import csv
import io
import subprocess
import sys

METRICS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
           "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
           "sm__inst_executed_pipe_tensor_op_umma.avg.pct_of_peak_sustained_active",
           "lts__throughput.avg.pct_of_peak_sustained_elapsed",
           "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
           "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
           "smsp__issue_active.avg.pct_of_peak_sustained_active",
           "launch__registers_per_thread", "launch__grid_size", "sm__cycles_elapsed.max",
           "lts__t_sectors_srcunit_tex_op_read.sum", "lts__t_bytes.sum"]


def run(args):
    return subprocess.run(["ncu"] + args, capture_output=True, text=True).stdout


def main(rep, out, topn):
    raw = list(csv.reader(io.StringIO(run(["-i", rep, "--page", "raw", "--csv"]))))
    hdr = raw[0]
    name_i = hdr.index("Kernel Name")
    with open(out, "w") as f:
        for kid, row in enumerate(raw[2:]):
            f.write(f"==== kernel {kid}: {row[name_i][:110]}\n")
            for m in METRICS:
                if m in hdr:
                    f.write(f"  {m} = {row[hdr.index(m)]} {raw[1][hdr.index(m)]}\n")
            src = list(csv.reader(io.StringIO(run(["-i", rep, "--page", "source", "--csv",
                                                   "--kernel-id", f":::{kid + 1}"]))))
            hi = next((i for i, r in enumerate(src) if "# Samples" in r), None)
            if hi is None:
                continue
            h = src[hi]
            si, so, ie = h.index("# Samples"), h.index("Source"), h.index("Instructions Executed")
            stalls = [i for i, c in enumerate(h) if c.startswith("stall_") and "Not Issued" not in c]
            data = [r for r in src[hi + 1:] if len(r) == len(h) and r[si].isdigit()]
            seen, uniq = set(), []
            for r in data:          # the page lists SASS and source views: keep one row per address
                key = (r[0], r[so])
                if key not in seen:
                    seen.add(key)
                    uniq.append(r)
            tot = sum(int(r[si]) for r in uniq) or 1
            agg = {}
            for r in uniq:
                for i in stalls:
                    agg[h[i]] = agg.get(h[i], 0) + int(r[i])
            f.write(f"  samples {tot}; warp instructions {sum(int(r[ie]) for r in uniq)}\n")
            f.write("  stalls: " + ", ".join(f"{k[6:]} {100 * v / tot:.1f}%" for k, v in
                                             sorted(agg.items(), key=lambda kv: -kv[1])[:9]) + "\n")
            for r in sorted(uniq, key=lambda r: -int(r[si]))[:topn]:
                st = sorted(((h[i][6:], int(r[i])) for i in stalls if int(r[i]) > 0),
                            key=lambda kv: -kv[1])[:3]
                f.write(f"  {100 * int(r[si]) / tot:5.1f}% x{r[ie]:>9} {r[so].strip()[:70]:70s} {st}\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else 22)
