#!/usr/bin/env python
"""Per-kernel totals of an ncu launch list (`ncu --metrics gpu__time_duration.sum --csv --log-file X ...`).

    python tools/ncu_launches.py launches.csv [top_n]

Prints launches, total and average duration per kernel, longest first. The CSV's Metric Unit column decides the scale
(ncu writes ns, us or ms depending on the value)."""
import collections
import csv
import sys

UNIT_TO_MS = {"ns": 1e-6, "nsecond": 1e-6, "us": 1e-3, "usecond": 1e-3, "ms": 1.0, "msecond": 1.0, "s": 1e3, "second": 1e3}


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    top_n = int(sys.argv[2]) if len(sys.argv) > 2 else 16
    header, agg = None, collections.OrderedDict()
    with open(sys.argv[1], newline="") as f:
        for row in csv.reader(f):
            if header is None:
                if "Kernel Name" in row and "Metric Value" in row:   # ncu prints banner lines before the header
                    header = row
                    ki, vi = row.index("Kernel Name"), row.index("Metric Value")
                    ui = row.index("Metric Unit") if "Metric Unit" in row else None
                continue
            if len(row) <= max(ki, vi):
                continue
            try:
                value = float(row[vi].replace(",", ""))
            except ValueError:
                continue
            scale = UNIT_TO_MS.get(row[ui].strip(), 1e-6) if ui is not None else 1e-6
            entry = agg.setdefault(row[ki][:90], [0, 0.0])
            entry[0] += 1
            entry[1] += value * scale
    if header is None:
        raise SystemExit(f"{sys.argv[1]}: no ncu CSV header found (expected the columns 'Kernel Name' and 'Metric Value')")
    total = sum(t for _, t in agg.values())
    for name, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top_n]:
        print(f"{n:5d} launches {t:10.3f} ms total {1e3 * t / n:10.1f} us avg {100 * t / total:5.1f} %  {name}")
    print(f"{sum(n for n, _ in agg.values()):5d} launches {total:10.3f} ms in all")


if __name__ == "__main__":
    main()
