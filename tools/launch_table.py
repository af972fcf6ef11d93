"""ncu launch list (``--metrics gpu__time_duration.sum --csv``) -> markdown: per-kernel totals and the ordered kernel
sequence of one training step with its stream — what the F / L / B programs are made of.

    python tools/launch_table.py launches_tf32.csv --steps 3 > profiles/launches_tf32.md
"""
import argparse
import collections
import csv
import re
import sys


def short(name: str) -> str:
    name = re.sub(r"^void\s+", "", name)
    name = re.sub(r"\(.*$", "", name)
    return name.replace("slb::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--steps", type=int, default=3, help="training steps contained in the capture window")
    a = ap.parse_args()
    rows = list(csv.reader(open(a.csv)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr = rows[hi]
    ki, vi, si, gi, bi = (hdr.index(k) for k in ("Kernel Name", "Metric Value", "Stream", "Grid Size", "Block Size"))
    data = [r for r in rows[hi + 1:] if len(r) > vi]
    agg = collections.OrderedDict()
    for r in data:
        e = agg.setdefault(short(r[ki]), [0, 0.0])
        e[0] += 1
        e[1] += float(r[vi].replace(",", "")) / 1e3
    total = sum(e[1] for e in agg.values())
    print(f"# Launch list: {len(data)} kernels in {a.steps} steps, {total / a.steps:.0f} us of kernel time per step "
          f"(serialised under ncu, no overlap; durations include the launch ramp)\n")
    print("| kernel | launches / step | us / launch | us / step | share |")
    print("|---|---:|---:|---:|---:|")
    for n, (c, t) in sorted(agg.items(), key=lambda x: -x[1][1]):
        print(f"| `{n}` | {c / a.steps:.1f} | {t / c:.2f} | {t / a.steps:.1f} | {100 * t / total:.1f} % |")
    per = len(data) // a.steps
    print(f"\n## Kernel sequence of one step ({per} launches; stream column separates the stage programs and the side stream "
          "that carries weight gradients + optimizer)\n")
    print("| # | stream | kernel | grid | block | us |")
    print("|---:|---:|---|---|---|---:|")
    for i, r in enumerate(data[per:2 * per]):
        print(f"| {i} | {r[si]} | `{short(r[ki])}` | {r[gi]} | {r[bi]} | {float(r[vi].replace(',', '')) / 1e3:.2f} |")


if __name__ == "__main__":
    sys.exit(main())
