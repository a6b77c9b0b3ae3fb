"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list per kernel: launches, total ms, share, average us.
Usage: python tools/summarize_launches.py launches.csv > launch_summary.csv"""
import csv
import re
import sys
from collections import OrderedDict


def main(path):
    with open(path, newline="") as f:
        rows = list(csv.reader(l for l in f if l.startswith('"')))
    head = rows[0]
    i_name, i_metric, i_unit, i_val = head.index("Kernel Name"), head.index("Metric Name"), head.index("Metric Unit"), head.index("Metric Value")
    scale = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3}
    agg = OrderedDict()
    for r in rows[1:]:
        if r[i_metric] != "gpu__time_duration.sum":
            continue
        name = re.sub(r"^void ", "", r[i_name])
        name = re.sub(r"<unnamed>::", "", name)
        name = name.split("(")[0][:70]
        ms = float(r[i_val].replace(",", "")) * scale.get(r[i_unit], 1e-6)
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += ms
    total = sum(v[1] for v in agg.values())
    w = csv.writer(sys.stdout)
    w.writerow(["kernel", "launches", "total_ms", "share_pct", "avg_us"])
    for name, (n, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        w.writerow([name, n, f"{ms:.3f}", f"{100 * ms / total:.2f}", f"{1e3 * ms / n:.1f}"])
    w.writerow(["TOTAL", sum(v[0] for v in agg.values()), f"{total:.3f}", "100.00", ""])


if __name__ == "__main__":
    main(sys.argv[1])
