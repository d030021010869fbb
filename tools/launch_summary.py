#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch log: time per kernel name.

    python tools/launch_summary.py results/launches.csv [--last N] [--top K]
"""
import csv
import io
import re
import sys
from collections import defaultdict


def short(name: str) -> str:
    name = re.sub(r"<.*", "", name)
    name = re.sub(r"\(.*", "", name)
    return name.split("::")[-1][:70] if "::" in name and not name.startswith("void") else name.replace("void ", "")[:70]


def main():
    path = sys.argv[1]
    last = int(sys.argv[sys.argv.index("--last") + 1]) if "--last" in sys.argv else None
    top = int(sys.argv[sys.argv.index("--top") + 1]) if "--top" in sys.argv else 40
    text = open(path, errors="replace").read()
    start = text.find('"ID"')
    rows = list(csv.DictReader(io.StringIO(text[start:])))
    rows = [r for r in rows if r.get("Metric Name") == "gpu__time_duration.sum"]
    if last:
        rows = rows[-last:]
    agg, cnt = defaultdict(float), defaultdict(int)
    for r in rows:
        v = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        ns = v * {"ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9, "nsecond": 1, "usecond": 1e3, "msecond": 1e6, "second": 1e9}.get(unit, 1)
        k = short(r["Kernel Name"])
        agg[k] += ns
        cnt[k] += 1
    tot = sum(agg.values())
    print(f"{len(rows)} launches, total {tot/1e6:.3f} ms")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:top]:
        print(f"{v/1e6:9.3f} ms  {100*v/tot:5.1f}%  x{cnt[k]:<5d} {k}")


if __name__ == "__main__":
    main()
