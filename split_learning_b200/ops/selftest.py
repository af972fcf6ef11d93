"""Numerics self-test of every sm_90a kernel against plain PyTorch fp32 references.

    python -m split_learning_b200.ops.selftest            # all checks, each in its own process
    python -m split_learning_b200.ops.selftest NAME ...   # selected checks, in-process

``tests/test_kernels_gpu.py`` runs the same functions under pytest.  Process isolation
matters while bringing kernels up: one illegal access poisons the CUDA context.
"""
from __future__ import annotations

import json
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

from . import native as N

CHECKS = {}


def check(fn):
    CHECKS[fn.__name__] = fn
    return fn


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _bf(x):
    return x.to(torch.bfloat16)


BF, F32 = torch.bfloat16, torch.float32
DTYPES = (F32, BF)          # fp32 tensors = wgmma tf32 (parity mode), bf16 = wgmma bf16 (fast mode)


def _exact():
    """The oracles are plain fp32 torch ops: no TF32 anywhere in the reference computation."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _tf32_rna(x):
    """fp32 -> nearest tf32 (10-bit mantissa, ties away from zero = cvt.rna.tf32.f32), kept in an fp32 container."""
    i = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    i = (i + 0x1000) & 0xFFFFE000
    i = torch.where(i >= 2 ** 31, i - 2 ** 32, i)
    return i.to(torch.int32).view(torch.float32).view(x.shape)


def _tol(dt, tf32=4e-3, bf16=1.5e-2):
    """Tolerance vs the exact fp32 oracle: tf32 operands carry 2^-11 relative rounding, bf16 2^-9."""
    return tf32 if dt == F32 else bf16


def _conv_case(B, H, W, Cin, Cout, seed=0, dt=BF):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g).to(dt)
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) * (1.0 / (9 * Cin) ** 0.5)).to(dt)
    bias = torch.randn(Cout, device="cuda", generator=g)
    return x, w, bias


def _ref_conv(x, w, bias=None):
    # NHWC -> NCHW fp32 reference
    _exact()
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), bias, padding=1)
    return y.permute(0, 2, 3, 1).contiguous()


CONV_SHAPES = [(32, 32, 32, 64, 64), (32, 16, 16, 64, 128), (32, 16, 16, 128, 128), (32, 8, 8, 128, 256),
               (32, 8, 8, 256, 256), (32, 4, 4, 256, 512), (32, 4, 4, 512, 512), (32, 2, 2, 512, 512), (8, 2, 2, 512, 512),
               (8, 32, 32, 64, 64)]


def _conv_fwd(dt):
    worst = 0.0
    for (B, H, W, Cin, Cout) in CONV_SHAPES:
        x, w, bias = _conv_case(B, H, W, Cin, Cout, dt=dt)
        y = torch.empty(B, H, W, Cout, device="cuda", dtype=dt)
        s1 = torch.zeros(Cout, device="cuda")
        s2 = torch.zeros(Cout, device="cuda")
        bn_, ks_ = N.conv_tiling(B * H * W, Cout, Cin, ke=32 if dt == F32 else 64)
        acc = torch.zeros(B * H * W, Cout, device="cuda") if ks_ > 1 else None
        ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
        N.conv3x3_fwd(x, w, y, bias, s1, s2, acc=acc, counters=ctr)          # in-kernel split-K finalisation
        if ks_ > 1:                                                           # ... and the two-kernel variant
            y2, t1, t2 = torch.empty_like(y), torch.zeros_like(s1), torch.zeros_like(s2)
            acc.zero_()
            N.conv3x3_fwd(x, w, y2, bias, t1, t2, acc=acc)
            torch.cuda.synchronize()
            assert int(ctr.abs().sum()) == 0, "tile semaphores must reset themselves"
            assert _rel(y2, y) < 1e-2 and _rel(t1, s1) < 1e-3
        torch.cuda.synchronize()
        ref = _ref_conv(x, w, bias)
        e = _rel(y, ref)
        yb = y.float().reshape(-1, Cout)
        e1 = _rel(s1, yb.sum(0))
        e2 = _rel(s2, (yb * yb).sum(0))
        extra = ""
        if dt == F32:       # against the same convolution on tf32-rounded operands: separates layout bugs from rounding
            extra = f" (vs tf32-rounded operands {_rel(y, _ref_conv(_tf32_rna(x), _tf32_rna(w), bias)):.2e})"
        print(f"  conv_fwd[{'tf32' if dt == F32 else 'bf16'}] {B}x{H}x{W} {Cin}->{Cout} bn={bn_} ksplit={ks_}: y {e:.2e} "
              f"sum {e1:.2e} sumsq {e2:.2e}{extra}")
        worst = max(worst, e, e1, e2)
    return worst, _tol(dt)


@check
def conv_fwd():
    return _conv_fwd(BF)


@check
def conv_fwd_tf32():
    return _conv_fwd(F32)


def _conv_dgrad(dt):
    worst = 0.0
    _exact()
    for (B, H, W, Cin, Cout) in CONV_SHAPES:
        x, w, _ = _conv_case(B, H, W, Cin, Cout, dt=dt)
        dy = torch.randn(B, H, W, Cout, device="cuda").to(dt)
        dx = torch.empty(B, H, W, Cin, device="cuda", dtype=dt)
        bn_, ks_ = N.conv_tiling(B * H * W, Cin, Cout, flip=1, ke=32 if dt == F32 else 64)
        acc = torch.zeros(B * H * W, Cin, device="cuda") if ks_ > 1 else None
        ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)       # must outlive the asynchronous kernel
        N.conv3x3_dgrad(dy, w, dx, acc=acc, counters=ctr)
        torch.cuda.synchronize()
        xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
        F.conv2d(xr, w.float().permute(0, 3, 1, 2), None, padding=1).backward(dy.float().permute(0, 3, 1, 2))
        e = _rel(dx, xr.grad.permute(0, 2, 3, 1))
        assert int(ctr.abs().sum()) == 0
        print(f"  conv_dgrad[{'tf32' if dt == F32 else 'bf16'}] {B}x{H}x{W} {Cin}<-{Cout}: {e:.2e}")
        worst = max(worst, e)
    return worst, _tol(dt)


@check
def conv_dgrad():
    return _conv_dgrad(BF)


@check
def conv_dgrad_tf32():
    return _conv_dgrad(F32)


@check
def conv_dgrad_bn_stats():
    """dgrad epilogue that also reduces the upstream block's BatchNorm-backward sums == the stand-alone reduce kernel
    (upstream block with and without MaxPool2)."""
    worst = 0.0
    for (B, H, W, Cin, Cout) in CONV_SHAPES:
        for pool in (False, True):
            x, w, _ = _conv_case(B, H, W, Cin, Cout)
            dy = _bf(torch.randn(B, H, W, Cout, device="cuda"))
            uh, uw = (2 * H, 2 * W) if pool else (H, W)
            up_y = _bf(torch.randn(B, uh, uw, Cin, device="cuda") * 1.5 + 0.2)       # saved conv output of the upstream block
            mean = up_y.float().mean((0, 1, 2))
            istd = (up_y.float().var((0, 1, 2), unbiased=False) + 1e-5).rsqrt()
            gamma = torch.rand(Cin, device="cuda") + 0.5
            beta = torch.randn(Cin, device="cuda") * 0.3
            bn_, ks_ = N.conv_tiling(B * H * W, Cin, Cout, flip=1)
            acc = torch.zeros(B * H * W, Cin, device="cuda") if ks_ > 1 else None
            ctr = torch.zeros(4096, device="cuda", dtype=torch.int32)
            dx = torch.empty(B, H, W, Cin, device="cuda", dtype=torch.bfloat16)
            dgamma, dbeta = torch.zeros(Cin, device="cuda"), torch.zeros(Cin, device="cuda")
            N.conv3x3_dgrad(dy, w, dx, acc=acc, counters=ctr,
                            bn_stats=(up_y, mean, istd, gamma, beta, True, pool, dgamma, dbeta))
            # oracle: plain dgrad + the two-kernel BN backward on its output
            dx2 = torch.empty_like(dx)
            acc2 = torch.zeros_like(acc) if acc is not None else None
            N.conv3x3_dgrad(dy, w, dx2, acc=acc2, counters=ctr)
            g2, b2 = torch.zeros(Cin, device="cuda"), torch.zeros(Cin, device="cuda")
            dyy = torch.empty_like(up_y)
            N.bn_relu_pool_bwd(dx2, up_y, gamma, beta, mean, istd, g2, b2, dyy, uh, uw, True, pool)
            dyy3 = torch.empty_like(up_y)
            N.bn_relu_pool_bwd(dx, up_y, gamma, beta, mean, istd, dgamma, dbeta, dyy3, uh, uw, True, pool, reduced=True)
            torch.cuda.synchronize()
            e = max(_rel(dx, dx2), _rel(dgamma, g2), _rel(dbeta, b2), _rel(dyy3, dyy))
            print(f"  conv_dgrad_bn_stats {B}x{H}x{W} {Cin}<-{Cout} pool={int(pool)}: {e:.2e}")
            worst = max(worst, e)
    return worst, 6e-3          # split-K red.add order differs between the two dgrad runs: dx may differ by one bf16 ulp


def _conv_wgrad(dt):
    worst = 0.0
    _exact()
    for (B, H, W, Cin, Cout) in CONV_SHAPES:
        x, w, _ = _conv_case(B, H, W, Cin, Cout, dt=dt)
        dy = torch.randn(B, H, W, Cout, device="cuda").to(dt)
        dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
        N.conv3x3_wgrad(x, dy, dw)
        torch.cuda.synchronize()
        wr = w.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        F.conv2d(x.float().permute(0, 3, 1, 2), wr, None, padding=1).backward(dy.float().permute(0, 3, 1, 2))
        e = _rel(dw, wr.grad.permute(0, 2, 3, 1))
        print(f"  conv_wgrad[{'tf32' if dt == F32 else 'bf16'}] {B}x{H}x{W} {Cin}x{Cout}: {e:.2e}")
        worst = max(worst, e)
    return worst, _tol(dt)


@check
def conv_wgrad():
    return _conv_wgrad(BF)


@check
def conv_wgrad_tf32():
    return _conv_wgrad(F32)


@check
def linear_f32():
    """fp32 CUDA-core Linear (parity mode) vs torch fp32: forward, input gradient, weight gradient (plain, accumulate,
    batch > 32) and the weight-gradient pass with the fused SGD-momentum update (two steps vs torch.optim.SGD)."""
    _exact()
    worst = 0.0
    for (Bn, inf, outf, pad) in [(32, 512, 4096, 0), (32, 4096, 4096, 0), (32, 4096, 10, 16), (8, 4096, 4096, 0), (48, 512, 256, 0)]:
        torch.manual_seed(7)
        x = torch.randn(Bn, inf, device="cuda")
        w = torch.randn(outf, inf, device="cuda") / inf ** 0.5
        acc = torch.zeros(Bn, outf, device="cuda")
        N.linear_fwd_f32(x, w, acc)
        torch.cuda.synchronize()
        e1 = _rel(acc, x @ w.t())
        ld = pad or outf
        dzp = torch.zeros(Bn, ld, device="cuda")
        dzp[:, :outf] = torch.randn(Bn, outf, device="cuda")
        dz = dzp[:, :outf]
        dacc = torch.zeros(Bn, inf, device="cuda")
        N.linear_dgrad_f32(dz, w, dacc)
        torch.cuda.synchronize()
        e2 = _rel(dacc, dz @ w)
        dw = torch.full((outf, inf), 7.0, device="cuda")
        N.linear_wgrad_f32(dz, x, g=dw)
        torch.cuda.synchronize()
        ref_dw = dz.t() @ x
        e3 = _rel(dw, ref_dw)
        N.linear_wgrad_f32(dz, x, g=dw, accumulate=True)
        torch.cuda.synchronize()
        e3 = max(e3, _rel(dw, 2 * ref_dw))
        e4 = 0.0
        if Bn <= 32:
            P, M = w.clone(), torch.zeros_like(w)
            bp, bm = torch.randn(outf, device="cuda"), torch.zeros(outf, device="cuda")
            rp, rb = torch.nn.Parameter(w.clone()), torch.nn.Parameter(bp.clone())
            opt = torch.optim.SGD([rp, rb], lr=0.05, momentum=0.5)
            for step in range(2):
                bg = dz.sum(0).contiguous() * (step + 1)
                rp.grad, rb.grad = ref_dw.clone(), bg.clone()
                opt.step()
                N.linear_wgrad_f32(dz, x, sgd=(P, M, bp, bm, bg, 0.05, 0.5))
                torch.cuda.synchronize()
                assert float(bg.abs().max()) == 0.0, "the fused update must zero the bias gradient"
            e4 = max(_rel(P, rp.data), _rel(bp, rb.data))
        print(f"  linear_f32 {Bn}x{inf}->{outf}: fwd {e1:.2e} dgrad {e2:.2e} wgrad {e3:.2e} wgrad+sgd {e4:.2e}")
        worst = max(worst, e1, e2, e3, e4)
    return worst, 2e-5


@check
def linear_all():
    worst = 0.0
    for (Bn, inf, outf, pad) in [(32, 512, 4096, 0), (32, 4096, 4096, 0), (32, 4096, 10, 16), (8, 4096, 4096, 0)]:
        x = _bf(torch.randn(Bn, inf, device="cuda"))
        w = _bf(torch.randn(outf, inf, device="cuda") / inf ** 0.5)
        acc = torch.zeros(Bn, outf, device="cuda")
        N.linear_fwd(x, w, acc)
        torch.cuda.synchronize()
        e1 = _rel(acc, x.float() @ w.float().t())
        ld = pad or outf
        dzp = torch.zeros(Bn, ld, device="cuda", dtype=torch.bfloat16)
        dzp[:, :outf] = _bf(torch.randn(Bn, outf, device="cuda"))
        dz = dzp[:, :outf]
        dacc = torch.zeros(Bn, inf, device="cuda")
        N.linear_dgrad(dz, w, dacc)
        torch.cuda.synchronize()
        e2 = _rel(dacc, dz.float() @ w.float())
        dw = torch.empty(outf, inf, device="cuda")
        N.linear_wgrad(dz, x, dw)
        torch.cuda.synchronize()
        e3 = _rel(dw, dz.float().t() @ x.float())
        print(f"  linear {Bn}x{inf}->{outf}: fwd {e1:.2e} dgrad {e2:.2e} wgrad {e3:.2e}")
        worst = max(worst, e1, e2, e3)
    return worst, 1e-2


def _bn_fwd_bwd(dt):
    worst = 0.0
    _exact()
    for (B, H, W, C, relu, pool) in [(32, 32, 32, 64, 1, 1), (32, 32, 32, 64, 1, 0), (32, 32, 32, 64, 0, 0),
                                     (32, 16, 16, 128, 1, 1), (32, 2, 2, 512, 1, 1), (8, 4, 4, 512, 1, 0)]:
        torch.manual_seed(1)
        y = (torch.randn(B, H, W, C, device="cuda") * 1.5 + 0.3).to(dt)
        gamma = torch.rand(C, device="cuda") + 0.5
        beta = torch.randn(C, device="cuda") * 0.1
        rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        nbt = torch.zeros((), device="cuda", dtype=torch.int64)
        s1 = torch.zeros(C, device="cuda")
        s2 = torch.zeros(C, device="cuda")
        N.col_stats(y.view(-1, C), s1, s2)
        sm, si = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        OH, OW = (H // 2, W // 2) if pool else (H, W)
        out = torch.empty(B, OH, OW, C, device="cuda", dtype=dt)
        N.bn_relu_pool_fwd(y, s1, s2, gamma, beta, rm, rv, nbt, sm, si, out, H, W, relu, pool)
        torch.cuda.synchronize()
        # reference
        yr = y.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        bn = torch.nn.BatchNorm2d(C).cuda().train()
        with torch.no_grad():
            bn.weight.copy_(gamma)
            bn.bias.copy_(beta)
        z = bn(yr)
        if relu:
            z = F.relu(z)
        if pool:
            z = F.max_pool2d(z, 2, 2)
        e1 = _rel(out, z.permute(0, 2, 3, 1))
        e2 = max(_rel(rm, bn.running_mean), _rel(rv, bn.running_var))
        dout = torch.randn_like(out.float()).to(dt)
        z.backward(dout.float().permute(0, 3, 1, 2))
        dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        dy = torch.empty_like(y)
        N.bn_relu_pool_bwd(dout, y, gamma, beta, sm, si, dg, db, dy, H, W, relu, pool)
        torch.cuda.synchronize()
        # single-launch variant (reduce -> grid barrier -> apply), twice on the same barrier words
        bar = torch.zeros(4, device="cuda", dtype=torch.int32)
        for _rep in range(2):
            dg2, db2, dy2 = torch.zeros_like(dg), torch.zeros_like(db), torch.empty_like(dy)
            N.bn_relu_pool_bwd(dout, y, gamma, beta, sm, si, dg2, db2, dy2, H, W, relu, pool, grid_bar=bar)
            torch.cuda.synchronize()
            assert _rel(dy2, dy) < 1e-2 and _rel(dg2, dg) < 2e-4 and _rel(db2, db) < 2e-4, "fused BN backward mismatch"
        assert bar.tolist()[1] == 2 and bar.tolist()[2] == 0
        e3 = _rel(dy, yr.grad.permute(0, 2, 3, 1))
        e4 = max(_rel(dg, bn.weight.grad), _rel(db, bn.bias.grad))
        print(f"  bn[{'fp32' if dt == F32 else 'bf16'}] {B}x{H}x{W}x{C} relu={relu} pool={pool}: out {e1:.2e} running {e2:.2e} "
              f"dy {e3:.2e} dgamma/dbeta {e4:.2e} nbt={int(nbt)}")
        worst = max(worst, e1, e2, e3, e4)
        assert int(nbt) == 1
    return worst, (2e-4 if dt == F32 else 2e-2)


@check
def bn_fwd_bwd():
    return _bn_fwd_bwd(BF)


@check
def bn_fwd_bwd_f32():
    return _bn_fwd_bwd(F32)


def _fused_cut_tail(dt):
    """conv+BN+ReLU+pool fused kernel vs torch (the cut blocks of cuts 7, 14, 10, 5)."""
    worst = 0.0
    ke = 32 if dt == F32 else 64
    for (B, H, W, Cin, Cout, relu, pool) in [(32, 32, 32, 64, 64, 1, 1), (32, 16, 16, 128, 128, 1, 1), (32, 16, 16, 64, 128, 1, 0),
                                             (32, 32, 32, 64, 64, 0, 0), (8, 32, 32, 64, 64, 1, 1), (32, 8, 8, 256, 256, 1, 1)]:
        assert N.fused_cut_supported(B, H, W, Cin, Cout, pool, ke=ke)
        x, w, bias = _conv_case(B, H, W, Cin, Cout, seed=5, dt=dt)
        gamma = torch.rand(Cout, device="cuda") + 0.5
        beta = torch.randn(Cout, device="cuda") * 0.1
        rm, rv = torch.zeros(Cout, device="cuda"), torch.ones(Cout, device="cuda")
        nbt = torch.zeros((), device="cuda", dtype=torch.int64)
        sm, si = torch.empty(Cout, device="cuda"), torch.empty(Cout, device="cuda")
        s1, s2 = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
        OH, OW = (H // 2, W // 2) if pool else (H, W)
        out = torch.zeros(B, OH, OW, Cout, device="cuda", dtype=dt)
        y = torch.zeros(B, H, W, Cout, device="cuda", dtype=dt)
        bar = torch.zeros(4, device="cuda", dtype=torch.int32)
        flag = torch.zeros(4, device="cuda", dtype=torch.int32)
        for rep in range(2):                      # second launch re-uses the barrier words (generation logic)
            s1.zero_(); s2.zero_()
            N.conv_bn_act_p2p(x, w, bias, gamma, beta, rm, rv, nbt, sm, si, s1, s2, y, out, relu, pool, bar,
                              flag=flag[0:1], seq=flag[1:2])
            torch.cuda.synchronize()
        bn = torch.nn.BatchNorm2d(Cout).cuda().train()
        with torch.no_grad():
            bn.weight.copy_(gamma); bn.bias.copy_(beta)
        conv = _ref_conv(x, w, bias).permute(0, 3, 1, 2)
        z = bn(conv); bn(conv)
        if relu:
            z = F.relu(z)
        if pool:
            z = F.max_pool2d(z, 2, 2)
        e1 = _rel(out, z.permute(0, 2, 3, 1))
        e2 = _rel(y, conv.permute(0, 2, 3, 1))
        e3 = max(_rel(rm, bn.running_mean), _rel(rv, bn.running_var))
        print(f"  fused cut[{'tf32' if dt == F32 else 'bf16'}] {B}x{H}x{W} {Cin}->{Cout} relu={relu} pool={pool}: out {e1:.2e} "
              f"y {e2:.2e} running {e3:.2e} flag={flag[:2].tolist()} nbt={int(nbt)}")
        assert flag[:2].tolist() == [2, 2] and int(nbt) == 2
        worst = max(worst, e1, e2, e3)
    return worst, (6e-3 if dt == F32 else 2e-2)


@check
def fused_cut_tail():
    return _fused_cut_tail(BF)


@check
def fused_cut_tail_tf32():
    return _fused_cut_tail(F32)


def _conv1_direct(dt):
    torch.manual_seed(2)
    _exact()
    B, Cin, H, W, Cout = 32, 3, 32, 32, 64
    x = torch.randn(B, Cin, H, W, device="cuda")
    w = torch.randn(Cout, 3, 3, Cin, device="cuda") * 0.2
    bias = torch.randn(Cout, device="cuda")
    y = torch.empty(B, H, W, Cout, device="cuda", dtype=dt)
    s1, s2 = torch.zeros(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    N.conv3x3_small_fwd(x, w, bias, y, s1, s2)
    torch.cuda.synchronize()
    wr = w.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ref = F.conv2d(x, wr, bias, padding=1)
    e1 = _rel(y, ref.permute(0, 2, 3, 1))
    e2 = _rel(s1, y.float().reshape(-1, Cout).sum(0))
    dy = torch.randn(B, H, W, Cout, device="cuda").to(dt)
    dw = torch.zeros(Cout, 3, 3, Cin, device="cuda")
    N.conv3x3_small_wgrad(x, dy, dw)
    torch.cuda.synchronize()
    ref.backward(dy.float().permute(0, 3, 1, 2))
    e3 = _rel(dw, wr.grad.permute(0, 2, 3, 1))
    print(f"  conv1 direct[{'fp32' if dt == F32 else 'bf16'}]: fwd {e1:.2e} stats {e2:.2e} wgrad {e3:.2e}")
    return max(e1, e2, e3), (1e-4 if dt == F32 else 1e-2)


@check
def conv1_direct():
    return _conv1_direct(BF)


@check
def conv1_direct_f32():
    return _conv1_direct(F32)


@check
def ce_and_linear_epilogues():
    torch.manual_seed(3)
    B, C = 32, 10
    logits = torch.randn(B, C, device="cuda") * 3
    labels = torch.randint(0, C, (B,), device="cuda")
    dl = torch.zeros(B, C, device="cuda")
    loss = torch.zeros(1, device="cuda")
    nan = torch.zeros(1, device="cuda", dtype=torch.int32)
    N.ce_fwd_bwd(logits, labels, dl, loss, nan)
    torch.cuda.synchronize()
    lr = logits.clone().requires_grad_(True)
    ref = F.cross_entropy(lr, labels)
    ref.backward()
    e1 = abs(float(loss) - float(ref)) / abs(float(ref))
    e2 = _rel(dl, lr.grad)
    assert int(nan) == 0
    # linear finalize / bwd prep / stand-alone dropout, both activation dtypes
    e3 = e4 = 0.0
    for dt in DTYPES:
        tol = 1e-5 if dt == F32 else 1e-2
        acc = torch.randn(B, 4096, device="cuda")
        bias = torch.randn(4096, device="cuda")
        out = torch.empty(B, 4096, device="cuda", dtype=dt)
        mask = torch.empty(B, 4096, device="cuda", dtype=torch.uint8)
        stepc = torch.full((1,), 7, device="cuda", dtype=torch.int32)
        N.linear_finalize(acc, bias, out, None, mask, True, 0.5, 123, stepc)
        torch.cuda.synchronize()
        ref_out = F.relu(acc + bias) * mask.float() * 2.0
        a3 = _rel(out, ref_out)
        keep = float(mask.float().mean())
        dacc = torch.randn(B, 4096, device="cuda")
        dz = torch.empty(B, 4096, device="cuda", dtype=dt)
        dbias = torch.empty(4096, device="cuda")
        N.linear_bwd_prep(dacc, out, mask, dz, dbias, True, 0.5)
        torch.cuda.synchronize()
        ref_dz = dacc * mask.float() * 2.0 * (out.float() > 0)
        a4 = max(_rel(dz, ref_dz), _rel(dbias, dz.float().sum(0)))
        xd = torch.randn(B, 512, device="cuda").to(dt)
        yd, md = torch.empty_like(xd), torch.empty(B, 512, device="cuda", dtype=torch.uint8)
        N.dropout_fwd(xd, yd, md, 0.5, 9, stepc)
        dxd = torch.empty_like(xd)
        N.dropout_bwd(dacc[:, :512].contiguous(), md, dxd, 0.5)
        torch.cuda.synchronize()
        a5 = max(_rel(yd, xd.float() * md.float() * 2.0), _rel(dxd, dacc[:, :512] * md.float() * 2.0))
        print(f"  [{'fp32' if dt == F32 else 'bf16'}] finalize {a3:.2e} keep={keep:.3f} bwd_prep {a4:.2e} dropout {a5:.2e}")
        assert 0.45 < keep < 0.55 and max(a3, a4, a5) < tol, (dt, a3, a4, a5)
        e3, e4 = max(e3, a3), max(e4, a4, a5)
    print(f"  ce loss {e1:.2e} dlogits {e2:.2e}")
    return max(e1, e2), 1e-5


@check
def optimizers_and_fedavg():
    torch.manual_seed(4)
    n = 1 << 20
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    ref_p = torch.nn.Parameter(p.clone())
    opt = torch.optim.SGD([ref_p], lr=0.01, momentum=0.5)
    m = torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    worst = 0.0
    for step in range(3):
        gi = g * (step + 1)
        ref_p.grad = gi.clone()
        opt.step()
        gg = gi.clone()
        N.sgd_momentum(p, gg, m, pb, 0.01, 0.5, step == 0)
        torch.cuda.synchronize()
        worst = max(worst, float((p - ref_p.data).abs().max()))
        assert float(gg.abs().max()) == 0.0
    sgd_bitwise = bool(torch.equal(p, ref_p.data))
    assert worst <= 2.4e-7, f"fp32 SGD-momentum deviates from torch.optim.SGD by {worst}"     # <= 1 ulp at |p| ~ 4
    e_shadow = _rel(pb, p)
    assert e_shadow < 8e-3, e_shadow                                                        # bf16 shadow: 2^-8 relative
    # AdamW
    p2 = torch.randn(n, device="cuda")
    ref2 = torch.nn.Parameter(p2.clone())
    o2 = torch.optim.AdamW([ref2], lr=1e-3, weight_decay=0.01)
    m2, v2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for step in range(1, 4):
        ref2.grad = g.clone() * step
        o2.step()
        N.adamw(p2, g.clone() * step, m2, v2, None, 1e-3, 0.9, 0.999, 1e-8, 0.01, step)
    torch.cuda.synchronize()
    e_adam = float((p2 - ref2.data).abs().max())
    # FedAvg
    srcs = [torch.randn(n, device="cuda") for _ in range(4)]
    srcs[1][5] = float("nan")
    coefs = [0.1, 0.2, 0.3, 0.4]
    out = torch.empty(n, device="cuda")
    N.fedavg(out, None, [s.data_ptr() for s in srcs], coefs, n)
    torch.cuda.synchronize()
    ref = sum(c * torch.nan_to_num(s) for c, s in zip(coefs, srcs))
    e_fa = float((out - ref).abs().max())
    # flat gradient-norm clipping (clip-grad-norm): sumsq + scale == torch.nn.utils.clip_grad_norm_
    gc = torch.randn(n, device="cuda")
    rg = torch.nn.Parameter(torch.zeros(n, device="cuda"))
    rg.grad = gc.clone()
    torch.nn.utils.clip_grad_norm_([rg], 5.0)
    acc = torch.zeros(4, device="cuda")
    N.sumsq(gc, acc)
    N.clip_scale(gc, acc, 5.0)
    torch.cuda.synchronize()
    e_clip = _rel(gc, rg.grad)
    print(f"  sgd max|diff| {worst:.2e} (bitwise equal to torch: {sgd_bitwise}) shadow {e_shadow:.2e} adamw {e_adam:.2e} "
          f"fedavg {e_fa:.2e} clip {e_clip:.2e}")
    return max(worst, e_adam, e_fa, e_clip * 1e-1), 1e-6


@check
def flags_and_peer():
    flag = torch.zeros(4, device="cuda", dtype=torch.int32)
    status = torch.zeros(1, device="cuda", dtype=torch.int32)
    side = torch.cuda.Stream()
    # load both kernels first: lazy module loading of a new kernel can wait for running kernels to finish
    N.set_flag(flag.data_ptr() + 12, 1)
    N.wait_flag(flag.data_ptr() + 12, 1, None, 1 << 10, status)
    torch.cuda.synchronize()
    N.wait_flag(flag.data_ptr(), 3, None, 1 << 22, status)          # waits on the main stream
    with torch.cuda.stream(side):
        N.set_flag(flag.data_ptr(), 3)
    torch.cuda.synchronize()
    assert int(flag[0]) == 3 and int(status) == 0
    ctr = torch.zeros(2, device="cuda", dtype=torch.int32)           # device-side sequence counters
    for it in range(1, 4):
        N.set_flag(flag.data_ptr() + 8, 0, ctr[0:1])
        N.wait_flag(flag.data_ptr() + 8, 0, ctr[1:2], 1 << 22, status)
    torch.cuda.synchronize()
    assert int(flag[2]) == 3 and ctr.tolist() == [3, 3] and int(status) == 0
    N.wait_flag(flag.data_ptr() + 4, 1, None, 1000, status)          # never set -> bounded timeout, no hang
    torch.cuda.synchronize()
    assert int(status) == 1
    return 0.0, 1.0


def run_one(name):
    t = time.time()
    err, tol = CHECKS[name]()
    ok = bool(err <= tol)
    print(json.dumps({"check": name, "err": err, "tol": tol, "ok": ok, "seconds": round(time.time() - t, 2)}))
    return ok


def main(argv):
    if argv:
        return 0 if all([run_one(n) for n in argv]) else 1
    results = {}
    for name in CHECKS:
        try:
            r = subprocess.run([sys.executable, "-m", "split_learning_b200.ops.selftest", name], capture_output=True,
                               text=True, timeout=300)
            tail = (r.stdout + r.stderr).strip().splitlines()[-25:]
            results[name] = r.returncode
        except subprocess.TimeoutExpired:
            tail, results[name] = ["TIMEOUT"], -9
        print(f"=== {name}: rc={results[name]}")
        print("\n".join(tail))
    print("SUMMARY", json.dumps(results))
    return 0 if all(v == 0 for v in results.values()) else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
