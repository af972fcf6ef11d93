"""Cycle stamps of CTA (0,0,0) of the conv kernels: where does one launch spend its time?  (clock64 cycles at GHZ)

    python tools/trace_gemm.py [tf32|bf16]     forward convs
    python tools/trace_gemm.py backward        tf32 input / weight gradients, per-K-step mainloop cost
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


def _wgrad_split(pixels, Cin, Cout, sms):
    """The automatic (block_n, k_split) of slb_conv3x3_wgrad for tf32 (32 pixels per K step)."""
    bn = min(128, Cin)
    k_iters = (pixels + 31) // 32
    tiles = ((9 * Cout + 127) // 128) * (Cin // bn)
    ks = min((sms + tiles - 1) // tiles, max(1, k_iters // 4))
    per = (k_iters + ks - 1) // ks
    return bn, (k_iters + per - 1) // per, k_iters


def backward(B=32):
    """tf32 dgrad / wgrad of every stage-2 conv at the executor's tiling: per-K-step mainloop cost of CTA (0,0,0) =
    (stamp 6 - stamp 2) / its K steps."""
    tr = torch.zeros(16, dtype=torch.int64, device="cuda")
    ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    N.lib().slb_set_gemm_trace(ctypes.c_void_p(tr.data_ptr()))
    for (HW, Cin, Cout) in [(32, 64, 64), (16, 64, 128), (16, 128, 128), (8, 128, 256), (8, 256, 256), (4, 256, 512),
                            (4, 512, 512), (2, 512, 512)]:
        M = B * HW * HW
        x = torch.randn(B, HW, HW, Cin, device="cuda")
        w = torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05
        dy = torch.randn(B, HW, HW, Cout, device="cuda")
        dx = torch.empty(B, HW, HW, Cin, device="cuda")
        dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
        bn, ks = N.conv_tiling(M, Cin, Cout, flip=1, ke=32)
        acc = torch.empty(max(1, N.conv_partial_floats(M, Cin, ks)), device="cuda")
        k_iters = 9 * Cout // 32
        dsteps = -(-k_iters // ks)
        wbn, wks, wk_iters = _wgrad_split(M, Cin, Cout, N.num_sms())
        wsteps = -(-wk_iters // wks)
        for op, fn, steps, tiling in [("dgrad", lambda: N.conv3x3_dgrad(dy, w, dx, acc=acc, counters=ctr), dsteps, (bn, ks)),
                                      ("wgrad", lambda: N.conv3x3_wgrad(x, dy, dw), wsteps, (wbn, wks))]:
            evs = []
            for rep in range(5):
                dw.zero_(); tr.zero_(); flush.zero_()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                evs.append(e0.elapsed_time(e1) * 1e3)
            t = tr.tolist()
            main_us = (t[6] - t[2]) / GHZ / 1e3
            print(f"{op} {HW}x{HW} {Cin}<->{Cout} bn={tiling[0]} ks={tiling[1]}: event {sorted(evs)[2]:.1f} us | "
                  f"mainloop {main_us:.2f} us over {steps} K steps = {main_us * 1e3 / steps:.0f} ns "
                  f"({(t[6] - t[2]) / steps:.0f} clk) per step | exit {(t[10] - t[0]) / GHZ / 1e3:.2f} us", flush=True)
    N.lib().slb_set_gemm_trace(ctypes.c_void_p(0))


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
    if len(sys.argv) > 1 and sys.argv[1] == "backward":
        backward()
    else:
        main()
