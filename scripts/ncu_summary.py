"""Summarise an .ncu-rep (one kernel) into a small text file: key raw metrics + the instructions that collect
the most warp-stall samples.  Usage: python scripts/ncu_summary.py x.ncu-rep x_summary.txt [note]"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__m_xbar2l1tex_read_bytes_mem_global_op_tma_ld.sum",
        "launch__registers_per_thread", "launch__grid_size", "launch__cluster_size", "sm__cycles_elapsed.max",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def run(rep, page):
    return subprocess.run(["ncu", "-i", rep, "--page", page, "--csv"], capture_output=True, text=True).stdout


def main():
    rep, out = sys.argv[1], sys.argv[2]
    note = sys.argv[3] if len(sys.argv) > 3 else ""
    raw = list(csv.reader(io.StringIO(run(rep, "raw"))))
    lines = ["ncu summary of %s" % rep, note, ""]
    hdr, units = raw[0], raw[1]
    for row in raw[2:]:
        d = dict(zip(hdr, row))
        lines.append("kernel: %s" % d.get("Kernel Name", "?")[:150])
        for k in KEYS:
            if k in d:
                lines.append("  %-75s %s %s" % (k, d[k], units[hdr.index(k)]))
    src = list(csv.reader(io.StringIO(run(rep, "source"))))
    if len(src) > 2:
        h = src[1]
        ix = {n: i for i, n in enumerate(h)}
        data = src[2:]
        tot = sum(int(r[ix["# Samples"]]) for r in data if r[ix["# Samples"]].isdigit())
        stalls = [n for n in h if n.startswith("stall_") and "Not Issued" not in n]
        lines += ["", "warp-stall samples: %d total; top instructions:" % tot]
        top = sorted(range(len(data)), key=lambda i: -int(data[i][ix["# Samples"]] or 0))[:25]
        for i in sorted(top):
            r = data[i]
            s = sorted(((n, int(r[ix[n]] or 0)) for n in stalls), key=lambda t: -t[1])[:2]
            lines.append("  [%4d] %-78s %6s (%4.1f%%) %s" % (i, r[ix["Source"]].strip()[:78], r[ix["# Samples"]],
                                                               100.0 * int(r[ix["# Samples"]]) / max(tot, 1),
                                                               ", ".join("%s %d" % t for t in s if t[1])))
        spins = [(i, r[ix["Source"]].strip()[:70], r[ix["Instructions Executed"]]) for i, r in enumerate(data)
                 if "TRYWAIT" in r[ix["Source"]]]
        lines += ["", "mbarrier try_wait instructions (executions = fast path + spin iterations):"]
        lines += ["  [%4d] %-70s executed %s" % t for t in spins]
    with open(out, "w") as fh:
        fh.write("\n".join(lines) + "\n")
    print("\n".join(lines[:30]))


if __name__ == "__main__":
    main()
