"""Summarise an .ncu-rep (read on the CPU box) into markdown: key raw metrics + top stall instructions.

    python tools/ncu_summary.py prof_fused.ncu-rep profiles/ncu_fused_cut7.md "title"
"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "sm__cycles_elapsed.max", "smsp__cycles_active.avg",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum"]


def run(args):
    return subprocess.run(["ncu", "-i"] + args, capture_output=True, text=True).stdout


def main(rep, dst, title):
    raw = list(csv.reader(io.StringIO(run([rep, "--page", "raw", "--csv"]))))
    hdr, units = raw[0], raw[1]
    out = [f"# {title}", "", f"source: `{rep}` (ncu --set full --clock-control none --import-source on)", ""]
    for r in raw[2:]:
        name = r[hdr.index("Kernel Name")]
        out += [f"## `{name[:110]}`", "", "| metric | value | unit |", "|---|---:|---|"]
        for k in KEYS:
            if k in hdr:
                out.append(f"| {k} | {r[hdr.index(k)]} | {units[hdr.index(k)]} |")
        out.append("")
    src = list(csv.reader(io.StringIO(run([rep, "--page", "source", "--csv"]))))
    h = next((i for i, r in enumerate(src) if "Source" in r and "Address" in r), None)
    if h is not None:
        hh = src[h]
        si, so = hh.index("Warp Stall Sampling (All Samples)"), hh.index("Source")
        rows = []
        for r in src[h + 1:]:
            if len(r) <= max(si, so) or r[0] == "Kernel Name":
                break
            try:
                rows.append((int(r[si]), r[so].strip()))
            except ValueError:
                pass
        tot = sum(n for n, _ in rows) or 1
        sass = " ".join(s for _, s in rows)
        out += ["## SASS evidence", "",
                f"HGMMA (wgmma): {sass.count('HGMMA')}  ·  UTMALDG (TMA load): {sass.count('UTMALDG')}  ·  "
                f"WARPGROUP.DEPBAR (wgmma.wait_group): {sass.count('WARPGROUP.DEPBAR')}  ·  SYNCS (mbarrier): {sass.count('SYNCS')}", "",
                "## top warp-stall sampling sites (first captured launch)", "", "| samples | share | SASS |", "|---:|---:|---|"]
        for n, s in sorted(rows, reverse=True)[:15]:
            out.append(f"| {n} | {100 * n / tot:.1f}% | `{s[:90]}` |")
    open(dst, "w").write("\n".join(out) + "\n")
    print("\n".join(out[:40]))


if __name__ == "__main__":
    main(*sys.argv[1:4])
