"""Cycle stamps of CTA (0,0,0) of the conv kernels: where does one launch spend its time?  (clock64 cycles at GHZ)

    python tools/trace_gemm.py [tf32|bf16]
stamps: 0 entry | 1 setup done (barriers) | 2 griddepcontrol.wait returned | 3 producer: ring of loads issued
        4, 5 unused | 6 accumulator complete | 7 accumulators drained, stores/reds issued
        8 reds visible (split-K) | 9 epilogue done | 10 CTA exit
"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from split_learning_b200.ops import native as N

GHZ = 1.98                       # H100 maximum SM clock (a power-capped card may run lower)


def main():
    dt = torch.float32 if (len(sys.argv) < 2 or sys.argv[1] == "tf32") else torch.bfloat16
    B = 32
    tr = torch.zeros(16, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    N.lib().slb_set_gemm_trace(ctypes.c_void_p(tr.data_ptr()))
    names = ["entry", "setup", "pdl", "ring", "first", "last", "accum", "drained", "redvis", "epi", "exit",
             "c0_ld", "c0_bias", "c0_store", "c0_reduce", "c0_end"]
    for (HW, Cin, Cout) in [(4, 512, 512), (16, 128, 128), (8, 256, 256), (32, 64, 64), (2, 512, 512)]:
        M = B * HW * HW
        x = torch.randn(B, HW, HW, Cin, device="cuda").to(dt)
        w = (torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05).to(dt)
        bias = torch.zeros(Cout, device="cuda")
        out = torch.empty(B, HW, HW, Cout, device="cuda", dtype=dt)
        acc = torch.zeros(N.conv_partial_floats(M, Cout, 4), device="cuda")
        s1, s2 = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
        for (bn, ks) in [(64, 1), (64, 4)]:
            if Cout % bn:
                continue
            for rep in range(3):
                acc.zero_(); tr.zero_(); flush.zero_()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                N.conv3x3_fwd(x, w, out, bias, s1, s2, acc=acc, tiling=(bn, ks), counters=ctr)
                e1.record()
                torch.cuda.synchronize()
            t = tr.tolist()
            base = t[0]
            rel = {n: round((v - base) / GHZ / 1e3, 2) for n, v in zip(names, t) if v}
            print(f"conv {HW}x{HW} {Cin}->{Cout} bn={bn} ks={ks}: event {e0.elapsed_time(e1) * 1e3:.1f} us | stamps(us) {rel}", flush=True)
    N.lib().slb_set_gemm_trace(ctypes.c_void_p(0))


if __name__ == "__main__":
    main()
