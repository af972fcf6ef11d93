"""Per-step stream timeline from an ncu launch list: which stream carries which kernels, in order, with running totals —
the dependent chain of the stage-2 program (main stream) against the forked weight-gradient / optimizer stream and the
stage-1 streams.  Durations are ncu's serialized per-kernel times (no overlap, launch ramp included), so the sums are an
upper bound of the in-graph time of each chain.

    python tools/critical_path.py launches_tf32.csv --per-step 117 > profiles/critical_path_tf32.md
"""
import argparse
import collections
import csv
import re


def short(name):
    return re.sub(r"\(.*$", "", re.sub(r"^void\s+", "", name)).replace("slb::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--per-step", type=int, default=117)
    a = ap.parse_args()
    rows = list(csv.reader(open(a.csv)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr = rows[hi]
    ki, vi, si = (hdr.index(k) for k in ("Kernel Name", "Metric Value", "Stream"))
    data = [(short(r[ki]), r[si], float(r[vi].replace(",", "")) / 1e3) for r in rows[hi + 1:] if len(r) > vi]
    # align the window to a step: a stage-2 pass starts with the scratch zeroing that follows the cross-entropy's predecessor;
    # use the first `ce_fwd_bwd_kernel` as the anchor and take one period of launches around it
    ce = [i for i, d in enumerate(data) if d[0] == "ce_fwd_bwd_kernel"]
    start = ce[0] if ce else 0
    end = ce[1] if len(ce) > 1 else start + a.per_step          # exactly one period: loss kernel to the next loss kernel
    step = data[start:end]
    by_stream = collections.OrderedDict()
    for k, s, us in step:
        by_stream.setdefault(s, []).append((k, us))
    tot = {s: sum(us for _, us in v) for s, v in by_stream.items()}
    main_stream = max(tot, key=tot.get)
    print(f"# Stream timeline of one training step (tf32 mode: the {len(step)} launches from one loss kernel to the next)\n")
    print("Durations: ncu `gpu__time_duration.sum` per kernel, serialized (upper bound of the in-graph time).  The step time of the")
    print("pipeline is set by the longest *dependent* chain — the stage-2 main stream; the other streams run concurrently.")
    print("(Stage 1 is phase-shifted by control-count microbatches and, in this eager capture, enqueues most of its launches")
    print("outside the window: its per-step total is F ~55 us + recompute/backward ~120 us, see `launches_tf32_final.md`.)\n")
    print("| stream | role | launches | sum of kernel times (us) |")
    print("|---:|---|---:|---:|")
    for s, v in by_stream.items():
        names = {k for k, _ in v}
        role = ("stage 2 main stream: backward chain (Linear dgrad, BN backward, conv dgrad) then next forward" if s == main_stream else
                "forked stream: weight gradients + SGD (joined at the end of the pass)" if "sgd_momentum_kernel" in names and "ce_fwd_bwd_kernel" not in names
                and not any(k.startswith("conv_bn_act") or k.startswith("conv3x3_small_fwd") for k in names) else "stage 1 stream")
        print(f"| {s} | {role} | {len(v)} | {tot[s]:.1f} |")
    print(f"\n## Stage-2 main stream ({main_stream}) in launch order\n")
    print("| # | kernel | us | running total (us) |")
    print("|---:|---|---:|---:|")
    run = 0.0
    cats = collections.Counter()
    for i, (k, us) in enumerate(by_stream[main_stream]):
        run += us
        cat = ("conv GEMM (wgmma)" if k.startswith("umma_gemm") else "Linear (fp32 CUDA cores)" if k.startswith("linear_") else
               "BatchNorm" if k.startswith("bn_") else "other")
        cats[cat] += us
        print(f"| {i} | `{k}` | {us:.2f} | {run:.1f} |")
    print("\n## What the stage-2 chain is made of\n")
    print("| category | us | share |")
    print("|---|---:|---:|")
    for c, us in cats.most_common():
        print(f"| {c} | {us:.1f} | {100 * us / run:.1f} % |")


if __name__ == "__main__":
    main()
