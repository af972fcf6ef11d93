"""Run one conv shape at several (BLOCK_N, split-K) settings — meant to be wrapped in ncu to see where the time goes.

    ncu --metrics gpu__time_duration.sum,lts__t_bytes.sum,dram__bytes_read.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active \
        --clock-control none --csv --log-file gpurun_out/probe.csv python tools/probe_conv.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from split_learning_b200.ops import native as N

SHAPES = [(4, 512, 512), (16, 128, 128), (8, 256, 256)]
CONFIGS = [(64, 1), (64, 4), (128, 4), (128, 8), (256, 4), (256, 8), (256, 16)]


def main():
    dt = torch.float32 if (len(sys.argv) < 2 or sys.argv[1] == "tf32") else torch.bfloat16
    B = 32
    ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for (HW, Cin, Cout) in SHAPES:
        M = B * HW * HW
        x = torch.randn(B, HW, HW, Cin, device="cuda").to(dt)
        w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05).to(dt)
        bias = torch.zeros(Cout, device="cuda")
        out = torch.empty(B, HW, HW, Cout, device="cuda", dtype=dt)
        acc = torch.zeros(N.conv_partial_floats(M, Cout, max(k for _, k in CONFIGS)), device="cuda")
        s1, s2 = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
        for (bn, ks) in CONFIGS:
            if Cout % bn:
                continue
            for rep in range(2):
                acc.zero_()
                flush.zero_()
                torch.cuda.synchronize()
                N.conv3x3_fwd(x, w, out, bias, s1, s2, acc=acc, tiling=(bn, ks), counters=ctr)
                torch.cuda.synchronize()
    print("done")


if __name__ == "__main__":
    main()
