"""Isolated timings + roofline fractions of the token-model kernels (wgmma GEMM epilogues, LayerNorm, attention).

    python tools/bench_token_kernels.py [--out profiles/kernels_tokens.json]

L2 is flushed between iterations (a 256 MB write); CUDA events; fractions are of MEASURED_PEAKS.json (cuBLAS bf16 burst,
HBM copy bandwidth).
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from split_learning_b200.ops import native as N  # noqa: E402

BF = torch.bfloat16


def timeit(fn, iters=20):
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    N.require()
    N.preload()
    peaks = {"bf16_tflops": 989.0, "hbm_gbs": 3350.0}          # H100 SXM data sheet unless MEASURED_PEAKS.json exists
    try:
        mp = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
        peaks["bf16_tflops"] = float(mp.get("bf16_tflops_burst", mp.get("bf16_tflops", peaks["bf16_tflops"])))
        peaks["hbm_gbs"] = float(mp.get("hbm_copy_gbs", mp.get("hbm_gbs", peaks["hbm_gbs"])))
    except (OSError, ValueError):
        pass
    rows = []
    for tokens in (1024, 4096, 16384):
        for (n, k, act, name) in ((3072, 768, "gelu", "ffn1 fwd (bias+GELU, keeps pre-act)"), (768, 3072, None, "ffn2 fwd (bias+residual)"),
                                  (768, 768, None, "proj fwd")):
            x = torch.randn(tokens, k, device="cuda").to(BF)
            w = torch.randn(n, k, device="cuda").to(BF)
            bias = torch.randn(n, device="cuda")
            out = torch.empty(tokens, n, device="cuda", dtype=BF)
            aux = torch.empty_like(out) if act else None
            res = torch.randn(tokens, n, device="cuda").to(BF) if "residual" in name else None
            us = timeit(lambda: N.gemm_act(x, w, out, tokens, n, k, bias=bias, act=act, aux=aux, residual=res))
            fl = 2.0 * tokens * n * k
            rows.append({"kernel": "umma_gemm<MODE_GEMM> " + name, "tokens": tokens, "N": n, "K": k, "us": round(us, 1),
                         "tflops": round(fl / us / 1e6, 1), "frac_bf16_peak": round(fl / us / 1e6 / peaks["bf16_tflops"], 3)})
        # dgrad / wgrad of the 768 -> 3072 layer
        n, k = 3072, 768
        dz = torch.randn(tokens, n, device="cuda").to(BF)
        w = torch.randn(n, k, device="cuda").to(BF)
        x = torch.randn(tokens, k, device="cuda").to(BF)
        dx = torch.empty(tokens, k, device="cuda", dtype=BF)
        us = timeit(lambda: N.gemm_act(dz, w, dx, tokens, k, n, b_mn=True, lda=n, ldb=k))
        fl = 2.0 * tokens * n * k
        rows.append({"kernel": "umma_gemm<MODE_GEMM> ffn1 dgrad (W read MN-major)", "tokens": tokens, "N": k, "K": n, "us": round(us, 1),
                     "tflops": round(fl / us / 1e6, 1), "frac_bf16_peak": round(fl / us / 1e6 / peaks["bf16_tflops"], 3)})
        dw = torch.zeros(n, k, device="cuda")
        tiles = ((n + 127) // 128) * ((k + 63) // 64)
        ks = max(1, min((tokens + 63) // 64, N.num_sms() // max(tiles, 1)))
        us = timeit(lambda: N.gemm_f32(dz, x, dw, n, k, tokens, a_mn=True, b_mn=True, lda=n, ldb=k, ldo=k, k_split=ks))
        rows.append({"kernel": "umma_gemm<MODE_GEMM> ffn1 wgrad (both MN-major, fp32 red.add)", "tokens": tokens, "N": k, "K": tokens,
                     "us": round(us, 1), "tflops": round(fl / us / 1e6, 1),
                     "frac_bf16_peak": round(fl / us / 1e6 / peaks["bf16_tflops"], 3)})
        # LayerNorm (fused dropout + residual) forward / backward: bytes moved
        d = 768
        xx = torch.randn(tokens, d, device="cuda").to(BF)
        rr = torch.randn(tokens, d, device="cuda").to(BF)
        g, b2 = torch.rand(d, device="cuda") + 0.5, torch.randn(d, device="cuda")
        y, pre = torch.empty_like(xx), torch.empty_like(xx)
        mean, rstd = torch.empty(tokens, device="cuda"), torch.empty(tokens, device="cuda")
        us = timeit(lambda: N.ln_fwd(xx, rr, g, b2, y, pre, mean, rstd, tokens, d, 1e-12, 0.1, 7))
        byt = tokens * d * 2 * 4
        rows.append({"kernel": "ln_fwd (dropout + residual + LN)", "tokens": tokens, "us": round(us, 1),
                     "gbs": round(byt / us / 1e3, 1), "frac_hbm": round(byt / us / 1e3 / peaks["hbm_gbs"], 3)})
        dy, dpre = torch.randn(tokens, d, device="cuda").to(BF), torch.empty_like(xx)
        dg, db = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
        us = timeit(lambda: N.ln_bwd(dy, pre, g, mean, rstd, dpre, dg, db, tokens, d))
        byt = tokens * d * 2 * 3
        rows.append({"kernel": "ln_bwd (dx + dgamma + dbeta)", "tokens": tokens, "us": round(us, 1),
                     "gbs": round(byt / us / 1e3, 1), "frac_hbm": round(byt / us / 1e3 / peaks["hbm_gbs"], 3)})
    for r in rows:
        print(json.dumps(r), flush=True)
    if a.out:
        json.dump({"peaks": peaks, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
