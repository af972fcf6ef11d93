"""Sweep (BLOCK_N, split-K) for every conv shape of the VGG16 stages at a given batch and write the best choices to
split_learning_b200/ops/conv_tuning.json (consumed by ``native.conv_tiling`` / ``native.wgrad_tiling``).

    python tools/tune_conv.py [--batch 32] [--iters 15]
Timing: CUDA events, median, L2 flushed before every iteration (in the training step the 470 MB working set evicts the
weights between uses, so cold-L2 is the representative condition).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from split_learning_b200.ops import native as N

SHAPES = [(32, 64, 64), (16, 64, 128), (16, 128, 128), (8, 128, 256), (8, 256, 256), (4, 256, 512), (4, 512, 512), (2, 512, 512)]
_flush = None


def flush():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def timeit(fn, iters, setup=None):
    for _ in range(2):
        if setup:
            setup()
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if setup:
            setup()
        flush()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--precision", default="tf32", choices=["tf32", "bf16"])
    a = ap.parse_args()
    B = a.batch
    dt = torch.float32 if a.precision == "tf32" else torch.bfloat16
    ke = 32 if a.precision == "tf32" else 64
    ckey, wkey = ("conv_f32", "wgrad_f32") if a.precision == "tf32" else ("conv", "wgrad")
    dst = os.path.join(ROOT, "gpurun_out", f"conv_tuning_b{B}.json")
    try:
        table = json.load(open(dst))
    except (OSError, ValueError):
        table = {"batch": B}
    table[ckey], table[wkey] = {}, {}
    ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
    for (HW, Cin, Cout) in SHAPES:
        M = B * HW * HW
        x = torch.randn(B, HW, HW, Cin, device="cuda").to(dt)
        dy = torch.randn(B, HW, HW, Cout, device="cuda").to(dt)
        w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05).to(dt)
        bias = torch.zeros(Cout, device="cuda")
        for flip in (0, 1):
            Nn, Ca = (Cout, Cin) if not flip else (Cin, Cout)
            out = torch.empty(B, HW, HW, Nn, device="cuda", dtype=dt)
            acc = torch.zeros(M, Nn, device="cuda")
            s1, s2 = torch.zeros(Nn, device="cuda"), torch.zeros(Nn, device="cuda")
            k_iters = 9 * (Ca // ke)
            best = None
            for bn in (64, 128, 256):
                if Nn % bn or (flip and bn > 128 and False):
                    continue
                for ks in (1, 2, 3, 4, 6, 8, 9, 12, 16, 18, 24):
                    if ks > max(1, k_iters // 2):
                        continue
                    tiles = ((M + 127) // 128) * (Nn // bn) * ks
                    if tiles > N.num_sms() * 4:
                        continue
                    if not flip:
                        fn = lambda: N.conv3x3_fwd(x, w, out, bias, s1, s2, acc=acc, tiling=(bn, ks), counters=ctr)
                    else:
                        fn = lambda: N.conv3x3_dgrad(dy, w, out, acc=acc, tiling=(bn, ks), counters=ctr)
                    t = timeit(fn, a.iters, (lambda: acc.zero_()) if ks > 1 else None)
                    if best is None or t < best[0]:
                        best = (t, bn, ks)
            key = f"{M},{Nn},{Ca},{flip}"
            table[ckey][key] = {"bn": best[1], "ks": best[2], "us": round(best[0], 2)}
            print("conv", "dgrad" if flip else "fwd", (HW, Cin, Cout), table[ckey][key], "default", N.conv_tiling(M, Nn, Ca, ke=ke), flush=True)
        dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
        k_iters = (M + ke - 1) // ke
        best = None
        for bn in (64, 128, 256):
            if Cin % bn:
                continue
            m_tiles = (9 * Cout + 127) // 128
            for ks in (1, 2, 3, 4, 6, 8, 12, 16, 24, 32):
                if ks > max(1, k_iters // 2) or m_tiles * (Cin // bn) * ks > N.num_sms() * 4:
                    continue
                t = timeit(lambda: N.conv3x3_wgrad(x, dy, dw, k_split=ks, block_n=bn), a.iters)
                if best is None or t < best[0]:
                    best = (t, bn, ks)
        key = f"{M},{Cin},{Cout}"
        table[wkey][key] = {"bn": best[1], "ks": best[2], "us": round(best[0], 2)}
        print("wgrad", (HW, Cin, Cout), table[wkey][key], flush=True)
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    json.dump(table, open(dst, "w"), indent=1)
    print("wrote", dst)


if __name__ == "__main__":
    main()
