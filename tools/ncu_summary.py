#!/usr/bin/env python
"""Summarise an ncu launch list (`ncu --metrics gpu__time_duration.sum[,dram__bytes_read.sum,dram__bytes_write.sum] --csv --log-file X.csv ...`)
per kernel: launches, total and mean duration, share of the listed time, DRAM bytes per launch.

    python tools/ncu_summary.py results/launches.csv [skip_first_n_launches] > launches.summary.txt

Per-launch times under ncu are cold-cache and serialised (no PDL overlap): the kernel SHARES are what to compare with the bench, never the absolutes."""
import csv
import re
import sys
from collections import OrderedDict


def main():
    path = sys.argv[1]
    skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rows = list(csv.DictReader(lines))
    per_id = OrderedDict()
    for r in rows:
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except (ValueError, KeyError):
            continue
        unit = r.get("Metric Unit", "")
        name = re.sub(r"\(.*", "", r["Kernel Name"]).strip()
        d = per_id.setdefault(r["ID"], {"name": name})
        m = r["Metric Name"]
        if m.startswith("gpu__time_duration"):
            d["us"] = v * {"nsecond": 1e-3, "ns": 1e-3, "usecond": 1.0, "us": 1.0, "msecond": 1e3, "ms": 1e3, "second": 1e6}.get(unit, 1e-3)
        elif m.startswith("dram__bytes"):
            d["dram"] = d.get("dram", 0.0) + v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
    launches = [d for d in list(per_id.values())[skip:] if "us" in d]
    agg = OrderedDict()
    for d in launches:
        a = agg.setdefault(d["name"], [0, 0.0, 0.0])
        a[0] += 1
        a[1] += d["us"]
        a[2] += d.get("dram", 0.0)
    total = sum(a[1] for a in agg.values()) or 1.0
    print(f"{'kernel':58} {'launches':>8} {'total_us':>10} {'avg_us':>8} {'share':>6} {'dram_MB/launch':>14}")
    for name, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{name[:58]:58} {a[0]:8d} {a[1]:10.1f} {a[1] / a[0]:8.2f} {100 * a[1] / total:5.1f}% {a[2] / a[0] / 1e6:14.3f}")
    print(f"{'TOTAL':58} {sum(a[0] for a in agg.values()):8d} {total:10.1f} {'':8} {'':6} {sum(a[2] for a in agg.values()) / 1e6:14.1f} (MB, all launches)")


if __name__ == "__main__":
    main()
