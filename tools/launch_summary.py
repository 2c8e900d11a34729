"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel.

    python tools/launch_summary.py launches.csv [--step]

--step: keep exactly one training step = the launches from one zeroing of the flat gradient
buffer (the only > 30 us FillFunctor<float> of a step) up to the next one.
"""
import collections
import csv
import re
import sys


def main(path):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr, data = rows[hi], rows[hi + 1:]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    if "--step" in sys.argv:
        def dur(r):
            v = float(r[vi].replace(",", ""))
            return v / 1000.0 if r[ui] == "ns" else v
        marks = [i for i, r in enumerate(data) if len(r) > vi and "FillFunctor<float>" in r[ki]
                 and dur(r) > 30.0]
        if len(marks) >= 2:
            data = data[marks[0]:marks[1]]
    agg, tot = collections.defaultdict(lambda: [0, 0.0]), 0.0
    for r in data:
        if len(r) <= vi:
            continue
        v = float(r[vi].replace(",", ""))
        if r[ui] == "ns":
            v /= 1000.0
        name = re.sub(r"\(CUtensor.*", "", r[ki])
        name = re.sub(r"^void ", "", name)[:72]
        agg[name][0] += 1
        agg[name][1] += v
        tot += v
    print(f"| kernel | launches | total us | share |\n|---|---|---|---|")
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{k}` | {n} | {t:.1f} | {100 * t / tot:.1f} % |")
    print(f"\ntotal {tot:.0f} us over {len(data)} launches")


if __name__ == "__main__":
    main(sys.argv[1])
