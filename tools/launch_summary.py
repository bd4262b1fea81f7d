"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel name.
usage: python tools/launch_summary.py launches.csv "<title>" > launches.txt"""
import collections
import csv
import re
import sys


def main():
    path, title = sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else ""
    lines = [l for l in open(path) if not l.startswith("==")]
    agg, tot, n = collections.OrderedDict(), 0.0, 0
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", ""))
        unit = row["Metric Unit"]
        v = v / 1e3 if unit == "ns" else (v * 1e3 if unit == "ms" else v)
        short = re.sub(r"\(.*", "", row["Kernel Name"])[:96]
        a = agg.setdefault(short, [0, 0.0])
        a[0] += 1
        a[1] += v
        tot += v
        n += 1
    print("# " + title)
    print("# per-launch times are cold-cache and serialised under ncu: compare SHARES, not absolutes")
    print("# total %.1f us over %d launches" % (tot, n))
    print("%-98s %6s %12s %7s" % ("kernel", "count", "total_us", "share"))
    mine = 0.0
    for k, (c, v) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-98s %6d %12.1f %6.1f%%" % (k, c, v, 100 * v / tot))
        if "dp::" in k or "expand_kernel" in k or "reduce_kernel" in k or "stem_" in k or "_kernel" in k and "cutlass" not in k and "nvjet" not in k:
            mine += v
    print("# hand-written kernels (dp::*, expand/reduce/stem/...): %.1f%% of device time; the rest is cuDNN/cublasLt tensor-core kernels" % (100 * mine / tot))


if __name__ == "__main__":
    main()
