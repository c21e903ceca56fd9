"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel name.
Usage: python scripts/launch_summary.py launches.csv [header note] > summary.txt"""
import collections
import csv
import re
import sys


def main():
    path = sys.argv[1]
    note = sys.argv[2] if len(sys.argv) > 2 else ""
    with open(path) as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    r = csv.reader(lines)
    hdr = next(r)
    ix = {n: i for i, n in enumerate(hdr)}
    agg = collections.defaultdict(lambda: [0, 0.0])
    tot, n = 0.0, 0
    for row in r:
        if len(row) < len(hdr) or row[ix["Metric Name"]] != "gpu__time_duration.sum":
            continue
        v = float(row[ix["Metric Value"]].replace(",", ""))
        u = row[ix["Metric Unit"]]
        v = v / 1000 if u == "ns" else v * 1000 if u == "ms" else v
        key = re.sub(r"\(.*", "", row[ix["Kernel Name"]])[:78]
        agg[key][0] += 1
        agg[key][1] += v
        tot += v
        n += 1
    print("# %s" % note)
    print("# %d launches, %.1f ms of kernel time (per-launch times are cold-cache and serialised: compare SHARES)" % (n, tot / 1000))
    for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:40]:
        print("%-80s n=%5d  %9.2f ms  %5.1f%%  avg %8.1f us" % (k, c, t / 1000, 100 * t / tot, t / c))


if __name__ == "__main__":
    main()
