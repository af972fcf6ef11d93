"""Token-model kernels against the float64 references of ``token_oracles``, elementwise, at their edge shapes.

GEMM (every operand-major combination and every legal column-tile width, K tails, unaligned output pitches), the
autograd Linear, attention forward / backward (S from 1 to 128, both head widths, heads at box offset 32, packed and
column-sliced operands, key bias, exact dropout masks), LayerNorm (both backward variants, partial blocks, offset
inputs), the pointwise kernels, and the host-side argument checks."""
import json
import math
import os

import pytest
import torch

import token_oracles as O

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F64 = torch.float64
DEV = "cuda"
WORST = {}


def _need():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.ops import native as N
    N.require()
    N.preload()
    return N


def _check(family, got, ref, bound, what):
    r = O.check(got, ref, bound, f"{family} {what}")
    WORST[family] = max(WORST.get(family, 0.0), r)
    return r


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if WORST:
        print("\nworst error / bound per kernel family:", json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))
        out = os.environ.get("SLB200_BOUND_RATIOS")
        if out:
            with open(out, "w") as f:
                json.dump(WORST, f, indent=1, sort_keys=True)


def _r8(n):
    return (n + 7) // 8 * 8


def _bf(*shape, scale=1.0, offset=0.0, gen=None):
    return (torch.randn(*shape, device=DEV, generator=gen) * scale + offset).to(BF)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ GEMM
GEMM_M = (1, 8, 127, 128, 129, 792)
GEMM_N = (4, 10, 32, 36, 64, 100, 200, 768)
GEMM_K = (8, 40, 64, 72, 3072)
GEMM_TILES = [(a, b, bn) for a in (False, True) for b in (False, True) for bn in (32, 64, 128, 256) if not (b and bn == 32)]
ACTS = (None, "relu", "gelu", "tanh")


def _operands(M, N, K, a_mn, b_mn, gen):
    """A and B in the requested storage (padded 16-byte row pitches) and their float64 [M, K] / [N, K] views."""
    a = _bf(M, K, gen=gen)
    b = _bf(N, K, scale=1 / math.sqrt(K), gen=gen)
    if a_mn:
        sa = torch.zeros(K, _r8(M), dtype=BF, device=DEV)
        sa[:, :M] = a.T
        lda = _r8(M)
    else:
        sa, lda = a, K
    if b_mn:
        sb = torch.zeros(K, _r8(N), dtype=BF, device=DEV)
        sb[:, :N] = b.T
        ldb = _r8(N)
    else:
        sb, ldb = b, K
    return sa, lda, sb, ldb, a.to(F64), b.to(F64)


def _guarded(M, N, dtype, fill=float("nan")):
    """[M, N] output (pitch N) followed by 64 guard elements that must stay untouched."""
    buf = torch.full((M * N + 64,), fill, dtype=dtype, device=DEV)
    return buf, buf[:M * N].view(M, N)


@pytest.mark.parametrize("a_mn,b_mn,block_n", GEMM_TILES)
def test_gemm_act_all_shapes(a_mn, b_mn, block_n):
    N_ = _need()
    gen = _gen(100 + 8 * a_mn + 4 * b_mn + block_n)
    i = 0
    for M in GEMM_M:
        for Nn in GEMM_N:
            for K in GEMM_K:
                i += 1
                act = ACTS[i % 4]
                use_bias, use_res, use_aux = i % 2 == 0, (i // 2) % 2 == 0, i % 3 != 0
                sa, lda, sb, ldb, a, b = _operands(M, Nn, K, a_mn, b_mn, gen)
                bias = torch.randn(Nn, device=DEV, generator=gen) if use_bias else None
                res = _bf(M, Nn, gen=gen) if use_res else None
                obuf, out = _guarded(M, Nn, BF)
                abuf, aux = _guarded(M, Nn, BF) if use_aux else (None, None)
                N_.gemm_act(sa, sb, out, M, Nn, K, a_mn, b_mn, lda, ldb, Nn, bias=bias, act=act, aux=aux, residual=res,
                            block_n=block_n)
                y, yb, z, zb = O.gemm_ref(a, b, bias.to(F64) if use_bias else None, res.to(F64) if use_res else None, act)
                what = f"M={M} N={Nn} K={K} act={act} bias={use_bias} res={use_res}"
                _check("gemm_act", out, y, yb, what)
                assert torch.isnan(obuf[M * Nn:].float()).all(), f"{what}: wrote past the output"
                if use_aux:
                    _check("gemm_act", aux, z, zb, what + " aux")
                    assert torch.isnan(abuf[M * Nn:].float()).all(), f"{what}: wrote past aux"


@pytest.mark.parametrize("a_mn,b_mn,block_n", GEMM_TILES)
def test_gemm_f32_all_shapes(a_mn, b_mn, block_n):
    N_ = _need()
    gen = _gen(200 + 8 * a_mn + 4 * b_mn + block_n)
    i = 0
    for M in GEMM_M:
        for Nn in GEMM_N:
            for K in GEMM_K:
                i += 1
                ks = (1, 2, 3, 7)[i % 4]
                sa, lda, sb, ldb, a, b = _operands(M, Nn, K, a_mn, b_mn, gen)
                out0 = torch.randn(M, Nn, device=DEV, generator=gen)
                buf, out = _guarded(M, Nn, torch.float32)
                out.copy_(out0)
                N_.gemm_f32(sa, sb, out, M, Nn, K, a_mn, b_mn, lda, ldb, Nn, k_split=ks, block_n=block_n)
                ref, bound = O.gemm_f32_ref(a, b, out0.to(F64), ks)
                what = f"M={M} N={Nn} K={K} k_split={ks}"
                _check("gemm_f32", out, ref, bound, what)
                assert torch.isnan(buf[M * Nn:]).all(), f"{what}: wrote past the output"
                if i % 3 == 0:                           # the turn counter fixes the order of the K-slice additions
                    again = out0.clone()
                    N_.gemm_f32(sa, sb, again, M, Nn, K, a_mn, b_mn, lda, ldb, Nn, k_split=ks, block_n=block_n)
                    assert torch.equal(again, out), f"{what}: not bitwise reproducible"


@pytest.mark.parametrize("n_in,n_out,act", [(64, 36, None), (64, 36, "tanh"), (200, 100, None), (96, 100, "tanh"),
                                            (768, 8, None), (8, 768, None), (8, 768, "tanh")])
def test_linear_autograd(n_in, n_out, act):
    """``ops.nn.linear`` forward and backward: y, dx, dW and db accumulated into live gradients, and dres."""
    _need()
    from split_learning_b200.ops import nn as F
    gen = _gen(300 + n_out)
    m = 300
    x = _bf(m, n_in, gen=gen)
    w = torch.nn.Parameter(torch.randn(n_out, n_in, device=DEV, generator=gen) / math.sqrt(n_in))
    bias = torch.nn.Parameter(torch.randn(n_out, device=DEV, generator=gen) * 0.1)
    g0w, g0b = torch.randn_like(w), torch.randn_like(bias)
    w.grad, bias.grad = g0w.clone(), g0b.clone()
    res = _bf(m, n_out, gen=gen)
    dy = _bf(m, n_out, gen=gen)
    xn, rn = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
    y = F.linear(xn, w, bias, act, rn)
    y.backward(dy)
    wb = w.detach().to(BF).to(F64)
    yr, yb, _, _ = O.gemm_ref(x.to(F64), wb, bias.detach().to(F64), res.to(F64), act)
    _check("linear", y, yr, yb, "y")
    dz = rn.grad                                          # the residual's gradient is the GEMMs' dz
    if act is None:
        assert torch.equal(dz, dy)
    else:
        dzr, dzb = O.act_bwd_ref(dy.to(F64), y.to(F64), act)
        _check("linear", dz, dzr, dzb, "dz")
    dz64 = dz.to(F64)
    dxr, dxb, _, _ = O.gemm_ref(dz64, wb.T.contiguous())
    _check("linear", xn.grad, dxr, dxb, "dx")
    dwr, dwb = O.gemm_f32_ref(dz64.T, x.to(F64).T, g0w.to(F64), k_split=(m + 63) // 64)
    _check("linear", w.grad, dwr, dwb, "dW")
    dbr, dbb = O.colsum_ref(dz64, g0b.to(F64))
    _check("linear", bias.grad, dbr, dbb, "db")


# ------------------------------------------------------------------------------------------------ attention
ATT_S = (1, 2, 31, 63, 64, 65, 99, 127, 128)


def _attn_case(N_, B, S, H, Dh, packed, bias_kind, p=0.0, seed=0, seed_ofs=None, gen=None, repeat=False):
    E = H * Dh
    if packed:
        ld, cols = 3 * E, (0, E, 2 * E)
    else:
        ld, cols = 3 * E + 64, (64, 64 + E, 64 + 2 * E)     # column slices of one wider tensor
    qkv = _bf(B * S, ld, gen=gen)
    q, k, v = (O._heads(qkv, B, S, H, Dh, c, ld) for c in cols)
    kb = None
    if bias_kind == "bert":
        kb = torch.zeros(B, S, device=DEV)
        kb[:, S - max(1, S // 4):] = -10000.0
    elif bias_kind == "random":
        kb = torch.randn(B, S, device=DEV, generator=gen)
    ldo = E + 64
    out = torch.full((B * S, ldo), float("nan"), dtype=BF, device=DEV)
    lse = torch.empty(B * H * 128, device=DEV)
    N_.attn_fwd(qkv, qkv, qkv, ld, ld, ld, *cols, out, ldo, lse, kb, B, S, H, Dh, p, seed, seed_ofs)
    do_col = 0 if packed else 64
    lddo = E + do_col
    dO = _bf(B * S, lddo, gen=gen)
    dqkv = torch.full((B * S, ld), float("nan"), dtype=BF, device=DEV)
    N_.attn_bwd(qkv, qkv, qkv, dO, ld, ld, ld, lddo, *cols, do_col, dqkv, dqkv, dqkv, ld, ld, ld, *cols, lse, kb, B, S, H,
                Dh, p, seed, seed_ofs)
    if repeat:                                              # no atomics on this path: bitwise identical launches
        out2, lse2, dqkv2 = out.clone(), lse.clone(), dqkv.clone()
        N_.attn_fwd(qkv, qkv, qkv, ld, ld, ld, *cols, out2, ldo, lse2, kb, B, S, H, Dh, p, seed, seed_ofs)
        N_.attn_bwd(qkv, qkv, qkv, dO, ld, ld, ld, lddo, *cols, do_col, dqkv2, dqkv2, dqkv2, ld, ld, ld, *cols, lse2, kb, B,
                    S, H, Dh, p, seed, seed_ofs)
        rows = lambda t: t.view(B, H, 128)[:, :, :S]                      # rows >= S of lse are never written
        assert torch.equal(out2.view(torch.int16), out.view(torch.int16)) and torch.equal(rows(lse2), rows(lse))
        assert torch.equal(dqkv2.view(torch.int16), dqkv.view(torch.int16))
    drop = None
    if p > 0:
        ofs = int(seed_ofs.item()) if seed_ofs is not None else None
        drop = O.keep_scale(O.attn_drop_index(B, H, S, DEV), p, seed, ofs)
    fw = O.attention_fwd_ref(q, k, v, kb.to(F64) if kb is not None else None, drop)
    do = O._heads(dO, B, S, H, Dh, do_col, lddo)
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    what = f"B={B} S={S} H={H} Dh={Dh} packed={packed} bias={bias_kind} p={p}"
    _check("attn_fwd", O._heads(out, B, S, H, Dh, 0, ldo), fw["o"], fw["o_bound"], what + " O")
    assert torch.isnan(out[:, E:].float()).all(), what + ": wrote past the heads"
    got_lse = lse.view(B, H, 128)[:, :, :S]
    _check("attn_lse", got_lse, fw["lse"], fw["lse_bound"], what + " lse")
    for name, c in zip(("dq", "dk", "dv"), cols):
        _check("attn_bwd", O._heads(dqkv, B, S, H, Dh, c, ld), bw[name], bw[name + "_bound"], f"{what} {name}")
    if not packed:
        assert torch.isnan(dqkv[:, :64].float()).all(), what + ": wrote outside the gradient heads"


@pytest.mark.parametrize("Dh", [32, 64])
@pytest.mark.parametrize("S", ATT_S)
def test_attention_fwd_bwd(S, Dh):
    N_ = _need()
    gen = _gen(400 + S + Dh)
    for H in (1, 3, 4, 12):
        for packed in (True, False):
            for bias_kind in (None, "bert", "random"):
                for B in (1, 3):                            # 3 * S is not a multiple of 128 for S < 128
                    _attn_case(N_, B, S, H, Dh, packed, bias_kind, gen=gen, repeat=(B == 3 and bias_kind == "random"))


def test_attention_dropout_mask_is_the_ported_hash():
    """Recover the kernel's probability-dropout mask with V = I and compare it with the Python port, bit for bit."""
    N_ = _need()
    gen = _gen(500)
    B, S, H, Dh, p, seed = 3, 64, 2, 64, 0.1, 0xC0FFEE
    E = H * Dh
    for ofs in (None, 7):
        seed_ofs = torch.tensor([ofs], dtype=torch.int32, device=DEV) if ofs is not None else None
        q, k = _bf(B * S, E, gen=gen), _bf(B * S, E, gen=gen)
        eye = torch.eye(S, device=DEV).to(BF).repeat(B, H)                  # [B * S, H * Dh] with Dh == S
        out = torch.empty(B * S, E, dtype=BF, device=DEV)
        lse = torch.empty(B * H * 128, device=DEV)
        N_.attn_fwd(q, k, eye, E, E, E, 0, 0, 0, out, E, lse, None, B, S, H, Dh, p, seed, seed_ofs)
        got = out.view(B, S, H, Dh).transpose(1, 2) != 0                    # [B, H, query, key]
        want = O.keep_scale(O.attn_drop_index(B, H, S, DEV), p, seed, ofs) > 0
        assert torch.equal(got, want), f"ofs={ofs}: {int((got != want).sum())} mask elements differ"


@pytest.mark.parametrize("S,Dh,packed", [(31, 32, True), (99, 64, False), (128, 32, False), (65, 64, True)])
def test_attention_dropout_fwd_bwd(S, Dh, packed):
    N_ = _need()
    gen = _gen(600 + S)
    ofs = torch.tensor([3], dtype=torch.int32, device=DEV)
    for H in (3, 4):
        _attn_case(N_, 3, S, H, Dh, packed, "random", p=0.1, seed=1234 + S, gen=gen, repeat=True)
        _attn_case(N_, 3, S, H, Dh, packed, "bert", p=0.1, seed=99, seed_ofs=ofs, gen=gen)


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("D", [2, 64, 128, 768, 1024, 1026, 2048, 4096])
def test_layernorm_fwd_bwd(D):
    N_ = _need()
    gen = _gen(700 + D)
    eps = 1e-5
    gamma = torch.rand(D, device=DEV, generator=gen) + 0.5
    beta = torch.randn(D, device=DEV, generator=gen) * 0.1
    for rows in (1, 7, 8, 9, 4097):
        for use_res, p in ((False, 0.0), (True, 0.0), (False, 0.1), (True, 0.1)):
            for offset in (0.0, 32.0):                       # a common offset of 32 x the spread
                x = _bf(rows, D, offset=offset, gen=gen)
                res = _bf(rows, D, gen=gen) if use_res else None
                fused = use_res or p > 0
                seed = rows * 31 + D
                y = torch.empty(rows, D, dtype=BF, device=DEV)
                pre = torch.empty(rows, D, dtype=BF, device=DEV) if fused else None
                mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
                N_.ln_fwd(x, res, gamma, beta, y, pre, mean, rstd, rows, D, eps, p, seed)
                what = f"rows={rows} D={D} res={use_res} p={p} offset={offset}"
                drop = O.keep_scale(O.ln_drop_index(rows, D, DEV), p, seed) if p > 0 else None
                if fused:
                    pr, pb = O.ln_prologue_ref(x.to(F64), res.to(F64) if use_res else None, drop)
                    _check("ln_fwd", pre, pr, pb, what + " pre")
                pre_k = (pre if fused else x).to(F64)
                yr, yb, mu, rs = O.ln_fwd_ref(pre_k, gamma.to(F64), beta.to(F64), eps)
                _check("ln_fwd", y, yr, yb, what + " y")
                _, _, e_mu, eps_rs = O.ln_stats(pre_k, eps)
                _check("ln_fwd", mean, mu, e_mu.squeeze(-1) + O.U_32 * mu.abs(), what + " mean")
                _check("ln_fwd", rstd, rs, eps_rs.squeeze(-1) * rs, what + " rstd")
                dy = _bf(rows, D, gen=gen)
                dpre = torch.empty_like(dy)
                dg0, db0 = torch.randn(D, device=DEV, generator=gen), torch.randn(D, device=DEV, generator=gen)
                dg, db = dg0.clone(), db0.clone()
                N_.ln_bwd(dy, (pre if fused else x), gamma, mean, rstd, dpre, dg, db, rows, D)
                bw = O.ln_bwd_ref(dy.to(F64), pre_k, gamma.to(F64), eps, dg0.to(F64), db0.to(F64))
                _check("ln_bwd", dpre, bw["dpre"], bw["dpre_bound"], what + " dpre")
                _check("ln_bwd", dg, bw["dgamma"], bw["dgamma_bound"], what + " dgamma")
                _check("ln_bwd", db, bw["dbeta"], bw["dbeta_bound"], what + " dbeta")


# ------------------------------------------------------------------------------------------------ pointwise
@pytest.mark.parametrize("kind", ["relu", "gelu", "tanh"])
def test_act_bwd(kind):
    N_ = _need()
    gen = _gen(800)
    for n in (2, 4098, 300_002):
        z = _bf(n, scale=2.0, gen=gen)
        ref = torch.tanh(z.float()).to(BF) if kind == "tanh" else z
        dy = _bf(n, gen=gen)
        dz = torch.empty_like(dy)
        N_.act_bwd(dy, ref, dz, n, kind)
        r, b = O.act_bwd_ref(dy.to(F64), ref.to(F64), kind)
        _check("act_bwd", dz, r, b, f"{kind} n={n}")


def test_colsum_bf16():
    N_ = _need()
    gen = _gen(900)
    for rows in (1, 255, 257, 1000):
        for cols, ld in ((1, 8), (33, 40), (100, 136)):
            x = _bf(rows, ld, gen=gen)
            out0 = torch.randn(cols, device=DEV, generator=gen)
            out = out0.clone()
            N_.colsum_bf16(x, out, rows, cols, ld)
            r, b = O.colsum_ref(x[:, :cols].to(F64), out0.to(F64))
            _check("colsum", out, r, b, f"rows={rows} cols={cols} ld={ld}")


@pytest.mark.parametrize("with_types", [False, True])
def test_embed3(with_types):
    N_ = _need()
    gen = _gen(1000)
    vocab, npos, D, B, S, pad = 64, 128, 96, 3, 50, 0
    word = torch.randn(vocab, D, device=DEV, generator=gen)
    pos = torch.randn(npos, D, device=DEV, generator=gen)
    typ = torch.randn(2, D, device=DEV, generator=gen)
    ids = torch.randint(0, 5, (B, S), device=DEV, generator=gen)         # heavily repeated ids, the pad id among them
    ids[:, -4:] = pad
    tts = torch.randint(0, 2, (B, S), device=DEV, generator=gen) if with_types else None
    out = torch.empty(B * S, D, dtype=BF, device=DEV)
    N_.embed3_fwd(ids, tts, word, pos, typ, out, B * S, S, D)
    r, b = O.embed3_fwd_ref(ids.flatten(), tts.flatten() if with_types else None, word.to(F64), pos.to(F64),
                            typ.to(F64), S)
    _check("embed3", out, r, b, "fwd")
    g = _bf(B * S, D, gen=gen)
    dw0, dp0, dt0 = (torch.randn_like(t) for t in (word, pos, typ))
    dw, dp, dt = dw0.clone(), dp0.clone(), dt0.clone()
    N_.embed3_bwd(ids, tts, g, dw, dp, dt, B * S, S, D, pad)
    refs = O.embed3_bwd_ref(ids.flatten(), tts.flatten() if with_types else None, g.to(F64), S, dw0.to(F64),
                            dp0.to(F64), dt0.to(F64), pad)
    for name, got, (r, b) in (("dword", dw, refs[0:2]), ("dpos", dp, refs[2:4]), ("dtype", dt, refs[4:6])):
        _check("embed3", got, r, b, name)
    assert torch.equal(dw[pad], dw0[pad]), "the padding row received a gradient"
    assert torch.equal(dp[S:], dp0[S:]), "positions past S received a gradient"


def test_dropout_bf16_exact_mask():
    N_ = _need()
    gen = _gen(1100)
    n, p, seed = 3 * 4099 + 1, 0.1, 4242
    x = _bf(n, gen=gen)
    for ofs in (None, 9):
        so = torch.tensor([ofs], dtype=torch.int32, device=DEV) if ofs is not None else None
        y = torch.empty_like(x)
        N_.dropout_bf16(x, y, n, p, seed, so)
        ks = O.keep_scale(O.flat_drop_index(n, DEV), p, seed, ofs)
        _check("dropout", y, x.to(F64) * ks, O.U_BF * (x.to(F64) * ks).abs() + O.U_32 * (x.to(F64) * ks).abs(),
               f"ofs={ofs}")
        assert torch.equal(y != 0, (ks > 0) & (x != 0))
        dy = _bf(n, gen=gen)
        dx = torch.empty_like(dy)
        N_.dropout_bf16(dy, dx, n, p, seed, so)                              # backward re-applies the same mask
        assert torch.equal(dx != 0, (ks > 0) & (dy != 0))
    y0, y9 = torch.empty_like(x), torch.empty_like(x)
    N_.dropout_bf16(x, y0, n, p, seed)
    N_.dropout_bf16(x, y9, n, p, seed, torch.tensor([9], dtype=torch.int32, device=DEV))
    assert not torch.equal(y0, y9), "seed_ofs does not change the mask"
    # the LayerNorm prologue draws the same mask as dropout_bf16 over its [rows, D] block (nn.layer_norm's backward
    # relies on it)
    rows, D = 7, 130
    xl = _bf(rows, D, gen=gen)
    yl, pre = torch.empty_like(xl), torch.empty_like(xl)
    m, r = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    g1, b0 = torch.ones(D, device=DEV), torch.zeros(D, device=DEV)
    N_.ln_fwd(xl, None, g1, b0, yl, pre, m, r, rows, D, 1e-5, p, seed)
    yd = torch.empty_like(xl)
    N_.dropout_bf16(xl, yd, rows * D, p, seed)
    assert torch.equal(pre != 0, yd != 0)


# ------------------------------------------------------------------------------------------------ host checks
def _attn_args(S=16, H=2, Dh=32, ld=None, col=0):
    E = H * Dh
    ld = ld if ld is not None else 3 * E + 64
    rows = 2 * max(S, 1)
    t = torch.zeros(rows, max(ld, 8), dtype=BF, device=DEV)
    out = torch.zeros(rows, E + 64, dtype=BF, device=DEV)
    lse = torch.zeros(2 * H * 128, device=DEV)
    return t, ld, col, out, lse, E


@pytest.mark.parametrize("case", ["S=0", "S=129", "Dh=48", "Dh=64@col32", "ld%8", "past_ld", "bwd_Dh=64@col32",
                                  "bwd_past_ld", "bwd_dq_past_ld"])
def test_attention_host_checks(case):
    N_ = _need()
    S, H, Dh, ld, col = 16, 2, 32, None, 0
    if case == "S=0":
        S = 0
    elif case == "S=129":
        S = 129
    elif case == "Dh=48":
        Dh = 48
    elif case in ("Dh=64@col32", "bwd_Dh=64@col32"):
        Dh, col = 64, 32
    elif case == "ld%8":
        ld = 3 * H * Dh + 4
    elif case in ("past_ld", "bwd_past_ld"):
        ld, col = 3 * H * Dh, 2 * H * Dh + Dh              # the last head would read past the row pitch
    t, ld, col, out, lse, E = _attn_args(S, H, Dh, ld, col)
    torch.cuda.synchronize()
    before = out.clone()
    with pytest.raises(N_.NativeError):
        if case.startswith("bwd"):
            dq_ld = ld if case != "bwd_dq_past_ld" else E
            N_.attn_bwd(t, t, t, t, ld, ld, ld, ld, col, col, col, col, out, out, out, dq_ld, E + 64, E + 64, 8, 0, 0, lse,
                        None, 2, S, H, Dh)
        else:
            N_.attn_fwd(t, t, t, ld, ld, ld, col, col, col, out, E + 64, lse, None, 2, S, H, Dh)
    torch.cuda.synchronize()
    assert torch.equal(out, before), "a refused call still wrote its output"


def test_other_host_checks():
    N_ = _need()
    x = torch.zeros(4, 4100, dtype=BF, device=DEV)
    f = torch.zeros(4100, device=DEV)
    st = torch.zeros(4, device=DEV)
    with pytest.raises(N_.NativeError):
        N_.ln_fwd(x, None, f, f, x, None, st, st, 4, 63, 1e-5)             # odd D
    with pytest.raises(N_.NativeError):
        N_.ln_bwd(x, x, f, st, st, x, f, f, 4, 4098)                       # D > 4096
    with pytest.raises(N_.NativeError):
        N_.dropout_bf16(x, x, 7, 0.1, 1)                                   # odd n
    with pytest.raises(N_.NativeError):
        N_.act_bwd(x, x, x, 7, "gelu")                                     # odd n
    a = torch.zeros(128, 64, dtype=BF, device=DEV)
    out = torch.zeros(128, 64, dtype=BF, device=DEV)
    with pytest.raises(N_.NativeError):
        N_.gemm_act(a, a, out, 128, 64, 64, b_mn=True, block_n=32)         # MN-major B needs 64-wide groups
    with pytest.raises(N_.NativeError):
        N_.gemm_f32(a, a, st, 128, 64, 64, b_mn=True, block_n=32)
    torch.cuda.synchronize()
