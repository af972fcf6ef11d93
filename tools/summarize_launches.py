"""ncu launch list (``--metrics gpu__time_duration.sum --csv``) → per-kernel markdown table.

    python tools/summarize_launches.py launches.csv profiles/launches.md "title"
"""
import collections
import csv
import sys


def main(src, dst, title="launch list"):
    with open(src) as f:
        lines = [l for l in f if l.startswith('"')]
    rows = list(csv.DictReader(lines))
    tot, cnt, grid = collections.Counter(), collections.Counter(), {}
    for r in rows:
        name = r["Kernel Name"].split("(")[0].replace("void ", "")
        v = float(r["Metric Value"].replace(",", ""))
        v = v / 1000 if r["Metric Unit"] == "ns" else (v * 1000 if r["Metric Unit"] == "ms" else v)
        tot[name] += v
        cnt[name] += 1
        grid.setdefault(name, set()).add(r["Grid Size"])
    total = sum(tot.values())
    with open(dst, "w") as f:
        f.write(f"# {title}\n\n{len(rows)} launches, {total:.1f} us total (ncu-serialised, cold caches: compare shares)\n\n")
        f.write("| kernel | launches | total us | avg us | share | grids |\n|---|---:|---:|---:|---:|---|\n")
        for k, v in tot.most_common():
            f.write(f"| `{k}` | {cnt[k]} | {v:.1f} | {v / cnt[k]:.1f} | {100 * v / total:.1f}% | {' '.join(sorted(grid[k]))[:60]} |\n")
    print(open(dst).read())


if __name__ == "__main__":
    main(*sys.argv[1:4])
