"""Isolated kernel timings + roofline fractions (CUDA events, warm-up, L2 flush between iterations).

    python tools/profile_kernels.py [--precision tf32|bf16] [--only NAME] [--iters 20] [--out gpurun_out/kernels.json]

``--precision tf32`` (default, the engine's default): fp32 tensors, wgmma tf32 convolutions (compute roofline =
half of the bf16 tensor throughput), fp32 CUDA-core Linear with the SGD update fused into the weight-gradient pass.

Roofline denominators: MEASURED_PEAKS.json (hbm_gbs, bf16_tflops) when present, else the H100 SXM data sheet (3.35 TB/s HBM3,
989 TFLOP/s dense bf16 at 700 W; a card with a lower power limit reaches less).  For the fused cut kernels the target time
is max(FLOPs / peak, link bytes / NVLINK_GBS).  Under ``ncu`` use ``--only`` + ``--iters 1``.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from split_learning_b200.ops import native as N

PEAKS = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "src": "H100 SXM data sheet"}
pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
if os.path.exists(pk):
    d = json.load(open(pk))
    PEAKS = {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "src": "measured"}
NVLINK_GBS = 450.0                  # NVLink 4, one direction (data sheet)

_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def timeit(fn, iters, setup=None):
    for _ in range(3):
        if setup:
            setup()
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if setup:
            setup()
        flush_l2()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


PREC = "tf32"


def ADT():
    return torch.float32 if PREC == "tf32" else torch.bfloat16


def ISZ():
    return 4 if PREC == "tf32" else 2


def bf(x):
    return x.to(ADT())


def conv_case(B, H, W, Cin, Cout):
    x = bf(torch.randn(B, H, W, Cin, device="cuda"))
    w = bf(torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.05)
    bias = torch.zeros(Cout, device="cuda")
    return x, w, bias


CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


def _conv_fwd(B, H, W, Cin, Cout, iters):
    x, w, bias = conv_case(B, H, W, Cin, Cout)
    y = torch.empty(B, H, W, Cout, device="cuda", dtype=ADT())
    s1, s2 = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    bn_, ks = N.conv_tiling(B * H * W, Cout, Cin)
    acc = torch.zeros(B * H * W, Cout, device="cuda") if ks > 1 else None
    med, best = timeit(lambda: N.conv3x3_fwd(x, w, y, bias, s1, s2, acc=acc), iters, (lambda: acc.zero_()) if acc is not None else None)
    flops = 2.0 * B * H * W * Cout * 9 * Cin
    byts = (x.numel() + w.numel() + y.numel()) * ISZ()
    return {"us": med, "best_us": best, "flops": flops, "bytes": byts, "tiling": [bn_, ks]}


@case
def conv4_fwd(iters):
    return _conv_fwd(32, 32, 32, 64, 64, iters)


@case
def conv11_fwd(iters):
    return _conv_fwd(32, 16, 16, 128, 128, iters)


@case
def conv18_fwd(iters):
    return _conv_fwd(32, 8, 8, 256, 256, iters)


@case
def conv28_fwd(iters):
    return _conv_fwd(32, 4, 4, 512, 512, iters)


@case
def conv38_fwd(iters):
    return _conv_fwd(32, 2, 2, 512, 512, iters)


@case
def conv4_fwd_b256(iters):
    return _conv_fwd(256, 32, 32, 64, 64, iters)


@case
def conv18_fwd_b512(iters):
    return _conv_fwd(512, 8, 8, 256, 256, iters)


@case
def conv4_wgrad(iters):
    B, H, W, Cin, Cout = 32, 32, 32, 64, 64
    x, w, _ = conv_case(B, H, W, Cin, Cout)
    dy = bf(torch.randn(B, H, W, Cout, device="cuda"))
    dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
    med, best = timeit(lambda: N.conv3x3_wgrad(x, dy, dw), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * B * H * W * Cout * 9 * Cin, "bytes": (x.numel() + dy.numel()) * ISZ() + dw.numel() * 4}


@case
def conv28_wgrad(iters):
    B, H, W, Cin, Cout = 32, 4, 4, 512, 512
    x, w, _ = conv_case(B, H, W, Cin, Cout)
    dy = bf(torch.randn(B, H, W, Cout, device="cuda"))
    dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
    med, best = timeit(lambda: N.conv3x3_wgrad(x, dy, dw), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * B * H * W * Cout * 9 * Cin, "bytes": (x.numel() + dy.numel()) * ISZ() + dw.numel() * 4}


@case
def conv8_dgrad_cut_head(iters):
    """dX of the first conv of stage 2 at cut 7 — the kernel whose epilogue stores into the upstream mailbox."""
    B, H, W, Cin, Cout = 32, 16, 16, 64, 128
    x, w, _ = conv_case(B, H, W, Cin, Cout)
    dy = bf(torch.randn(B, H, W, Cout, device="cuda"))
    dx = torch.empty(B, H, W, Cin, device="cuda", dtype=ADT())
    med, best = timeit(lambda: N.conv3x3_dgrad(dy, w, dx), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * B * H * W * Cout * 9 * Cin, "bytes": (dy.numel() + w.numel() + dx.numel()) * ISZ(),
            "link_bytes": dx.numel() * ISZ()}


def _fused(B, H, W, Cin, Cout, relu, pool, iters):
    x, w, bias = conv_case(B, H, W, Cin, Cout)
    gamma, beta = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    rm, rv = torch.zeros(Cout, device="cuda"), torch.ones(Cout, device="cuda")
    nbt = torch.zeros((), device="cuda", dtype=torch.int64)
    sm, si = torch.empty(Cout, device="cuda"), torch.empty(Cout, device="cuda")
    s = torch.zeros(2 * Cout, device="cuda")
    OH, OW = (H // 2, W // 2) if pool else (H, W)
    out = torch.zeros(B, OH, OW, Cout, device="cuda", dtype=ADT())
    bar = torch.zeros(4, device="cuda", dtype=torch.int32)
    flag = torch.zeros(4, device="cuda", dtype=torch.int32)

    def run():
        N.zero_(s)
        N.conv_bn_act_p2p(x, w, bias, gamma, beta, rm, rv, nbt, sm, si, s[:Cout], s[Cout:], None, out, relu, pool, bar,
                          flag=flag[0:1], seq=flag[1:2])
    med, best = timeit(run, iters)
    return {"us": med, "best_us": best, "flops": 2.0 * B * H * W * Cout * 9 * Cin, "bytes": (x.numel() + w.numel() + out.numel()) * ISZ(),
            "link_bytes": out.numel() * ISZ()}


@case
def fused_cut7(iters):
    return _fused(32, 32, 32, 64, 64, 1, 1, iters)


@case
def fused_cut14(iters):
    return _fused(32, 16, 16, 128, 128, 1, 1, iters)


@case
def fused_cut7_b128(iters):
    return _fused(128, 32, 32, 64, 64, 1, 1, iters)


@case
def linear50_fwd_f32(iters):
    """fp32 Linear 4096 -> 4096 at batch 32 (parity mode): IEEE fp32 FMAs on CUDA cores, weight streamed once."""
    x = torch.randn(32, 4096, device="cuda")
    w = torch.randn(4096, 4096, device="cuda") * 0.01
    acc = torch.zeros(32, 4096, device="cuda")
    med, best = timeit(lambda: N.linear_fwd_f32(x, w, acc), iters, lambda: acc.zero_())
    return {"us": med, "best_us": best, "flops": 2.0 * 32 * 4096 * 4096, "bytes": w.numel() * 4 + x.numel() * 4 + acc.numel() * 4, "fp32_cuda_cores": True}


@case
def linear50_dgrad_f32(iters):
    dz = torch.randn(32, 4096, device="cuda")
    w = torch.randn(4096, 4096, device="cuda") * 0.01
    dacc = torch.zeros(32, 4096, device="cuda")
    med, best = timeit(lambda: N.linear_dgrad_f32(dz, w, dacc), iters, lambda: dacc.zero_())
    return {"us": med, "best_us": best, "flops": 2.0 * 32 * 4096 * 4096, "bytes": w.numel() * 4 + dz.numel() * 4 + dacc.numel() * 4, "fp32_cuda_cores": True}


@case
def linear50_wgrad_sgd_f32(iters):
    """dW = dz^T x with the SGD-momentum update applied in the same pass: reads P, M once, writes P, M once; no G buffer."""
    x = torch.randn(32, 4096, device="cuda")
    dz = torch.randn(32, 4096, device="cuda")
    P, Mo = torch.randn(4096, 4096, device="cuda") * 0.01, torch.zeros(4096, 4096, device="cuda")
    bp, bm, bg = torch.zeros(4096, device="cuda"), torch.zeros(4096, device="cuda"), torch.zeros(4096, device="cuda")
    med, best = timeit(lambda: N.linear_wgrad_f32(dz, x, sgd=(P, Mo, bp, bm, bg, 5e-4, 0.5)), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * 32 * 4096 * 4096, "bytes": P.numel() * 16 + (x.numel() + dz.numel()) * 4, "fp32_cuda_cores": True}


@case
def linear50_fwd(iters):
    x = bf(torch.randn(32, 4096, device="cuda"))
    w = bf(torch.randn(4096, 4096, device="cuda") * 0.01)
    acc = torch.zeros(32, 4096, device="cuda")
    med, best = timeit(lambda: N.linear_fwd(x, w, acc, k_split=8), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * 32 * 4096 * 4096, "bytes": w.numel() * 2 + x.numel() * 2 + acc.numel() * 4}


@case
def linear50_wgrad(iters):
    x = bf(torch.randn(32, 4096, device="cuda"))
    dz = bf(torch.randn(32, 4096, device="cuda"))
    dw = torch.empty(4096, 4096, device="cuda")
    med, best = timeit(lambda: N.linear_wgrad(dz, x, dw), iters)
    return {"us": med, "best_us": best, "flops": 2.0 * 32 * 4096 * 4096, "bytes": dw.numel() * 4 + x.numel() * 2 + dz.numel() * 2}


@case
def sgd_stage2(iters):
    n = 33_600_000 // 128 * 128
    p, g, m = (torch.randn(n, device="cuda") for _ in range(3))
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    med, best = timeit(lambda: N.sgd_momentum(p, g, m, pb, 5e-4, 0.5), iters)
    return {"us": med, "best_us": best, "flops": 4.0 * n, "bytes": n * (12 + 12 + 2)}


@case
def bn_relu_pool_fwd_conv4(iters):
    B, H, W, C = 32, 32, 32, 64
    y = bf(torch.randn(B, H, W, C, device="cuda"))
    s1, s2 = y.float().reshape(-1, C).sum(0), (y.float() ** 2).reshape(-1, C).sum(0)
    gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    nbt = torch.zeros((), device="cuda", dtype=torch.int64)
    sm, si = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    out = torch.empty(B, H // 2, W // 2, C, device="cuda", dtype=ADT())
    med, best = timeit(lambda: N.bn_relu_pool_fwd(y, s1, s2, gamma, beta, rm, rv, nbt, sm, si, out, H, W, True, True), iters)
    return {"us": med, "best_us": best, "flops": 0.0, "bytes": (y.numel() + out.numel()) * ISZ()}


@case
def fedavg_4src_local(iters):
    n = 33_600_000 // 128 * 128
    srcs = [torch.randn(n, device="cuda") for _ in range(4)]
    out = torch.empty(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    med, best = timeit(lambda: N.fedavg(out, pb, [s.data_ptr() for s in srcs], [0.25] * 4, n), iters)
    return {"us": med, "best_us": best, "flops": 8.0 * n, "bytes": n * (16 + 4 + 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    ap.add_argument("--precision", default="tf32", choices=["tf32", "bf16"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "kernels.json"))
    a = ap.parse_args()
    global PREC
    PREC = a.precision
    res = {"peaks": PEAKS, "precision": PREC, "gpu": torch.cuda.get_device_name(0), "kernels": {}}
    fp32_cuda_tflops = N.num_sms() * 128 * 2 * 1.98e9 / 1e12   # FFMA peak of the CUDA cores (SMs x 128 lanes, 1980 MHz max clock)
    for name, fn in CASES.items():
        if a.only and a.only != name:
            continue
        bf16_only = name in ("linear50_fwd", "linear50_wgrad")
        f32_only = name.endswith("_f32")
        if (PREC == "tf32" and bf16_only) or (PREC == "bf16" and f32_only):
            continue
        r = fn(a.iters)
        tensor_peak = PEAKS["bf16_tflops"] * (0.5 if PREC == "tf32" else 1.0)
        peak = fp32_cuda_tflops if r.get("fp32_cuda_cores") else tensor_peak
        r["compute_peak_tflops"] = peak
        t_c = r["flops"] / (peak * 1e12) * 1e6
        t_m = r["bytes"] / (PEAKS["hbm_gbs"] * 1e9) * 1e6
        t_l = r.get("link_bytes", 0) / (NVLINK_GBS * 1e9) * 1e6
        roof = max(t_c, t_m, t_l)
        r.update({"roofline_us": roof, "bound": "compute" if roof == t_c else ("hbm" if roof == t_m else "nvlink"),
                  "frac_of_roofline": roof / r["us"], "tflops": r["flops"] / r["us"] / 1e6, "gbs": r["bytes"] / r["us"] / 1e3})
        res["kernels"][name] = r
        print(f"{name:26s} {r['us']:9.1f} us (best {r['best_us']:8.1f})  roofline {roof:7.2f} us [{r['bound']}]  "
              f"frac {r['frac_of_roofline']:.3f}  {r['tflops']:8.1f} TFLOP/s  {r['gbs']:8.1f} GB/s", flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
