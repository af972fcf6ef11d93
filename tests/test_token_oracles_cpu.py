"""The float64 references of ``token_oracles`` against torch's own float64 modules, fp32 emulations of each kernel
inside their bounds, and the sensitivity of every bound: a plausibly wrong result, computed in float64, must fall
outside it.  Runs on the CPU."""
import math

import pytest
import torch
import torch.nn.functional as F

import token_oracles as O

F64 = torch.float64
TIGHT = dict(rtol=1e-12, atol=1e-12)


def _bf(*shape, scale=1.0, gen=None):
    return O.bf16(torch.randn(*shape, generator=gen, dtype=F64) * scale)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("act", [None, "relu", "gelu", "tanh"])
def test_gemm_ref_matches_torch(act):
    g = _gen(0)
    a, b = _bf(37, 72, gen=g), _bf(20, 72, gen=g)
    bias, res = _bf(20, gen=g), _bf(37, 20, gen=g)
    y, _, z, _ = O.gemm_ref(a, b, bias, res, act)
    zt = F.linear(a, b, bias) + res
    torch.testing.assert_close(z, zt, **TIGHT)
    yt = {None: lambda t: t, "relu": F.relu, "gelu": F.gelu, "tanh": torch.tanh}[act](zt)
    torch.testing.assert_close(y, yt, **TIGHT)


@pytest.mark.parametrize("act", [None, "relu", "gelu", "tanh"])
def test_gemm_bound_holds_for_fp32_emulation(act):
    """fp32 accumulation + fp32 activation + one bf16 rounding (what the kernel does) stays inside the bound."""
    g = _gen(1)
    a, b = _bf(64, 3072, gen=g), _bf(48, 3072, scale=1 / 55, gen=g)
    bias, res = _bf(48, gen=g), _bf(64, 48, gen=g)
    y, yb, z, zb = O.gemm_ref(a, b, bias, res, act)
    z32 = a.float() @ b.float().T + bias.float() + res.float()
    y32 = O.act_ref(z32.double(), act).float()
    assert O.check(O.bf16(z32.double()), z, zb, "pre") <= 1
    assert O.check(O.bf16(y32.double()), y, yb, "out") <= 1


def test_gemm_bound_rejects_missing_k_slice():
    g = _gen(2)
    for K in (72, 3072):
        a, b = _bf(33, K, gen=g), _bf(40, K, gen=g)
        y, yb, _, _ = O.gemm_ref(a, b)
        wrong = a[:, 64:] @ b[:, 64:].T if K > 64 else a[:, :64] @ b[:, :64].T
        assert O.excess(wrong, y, yb).any(), K
        wrong = a[:, :-8] @ b[:, :-8].T                     # a dropped K tail
        assert O.excess(wrong, y, yb).any(), K


def test_gemm_bound_rejects_gelu_tanh():
    """GELU-tanh differs from GELU-erf by up to 2.4 % at x around -2.5; the bound must see it at |x| ~ 2."""
    z = torch.cat([torch.linspace(-3, -1.75, 64, dtype=F64), torch.linspace(1.75, 3, 64, dtype=F64)])
    z = O.bf16(z)
    a = torch.zeros(z.numel(), 8, dtype=F64)
    a[:, 0] = z
    b = torch.zeros(1, 8, dtype=F64)
    b[0, 0] = 1
    y, yb, _, _ = O.gemm_ref(a, b, act="gelu")
    wrong = F.gelu(z, approximate="tanh")[:, None]
    assert O.excess(wrong, y, yb).any()
    dy = torch.ones_like(z)
    dz, dzb = O.act_bwd_ref(dy, z, "gelu")
    zt = z.clone().requires_grad_(True)
    F.gelu(zt, approximate="tanh").backward(dy)
    assert O.excess(zt.grad, dz, dzb).any()


def test_gemm_f32_and_colsum_refs():
    g = _gen(3)
    a, b = _bf(30, 136, gen=g), _bf(12, 136, gen=g)
    out0 = torch.randn(30, 12, generator=g, dtype=F64)
    ref, bound = O.gemm_f32_ref(a, b, out0, k_split=3)
    torch.testing.assert_close(ref, out0 + a @ b.T, **TIGHT)
    part = [a[:, i:i + 64].float() @ b[:, i:i + 64].float().T for i in range(0, 136, 64)]
    got = out0.float()
    for p in part:
        got = got + p
    assert O.check(got.double(), ref, bound, "gemm_f32") <= 1
    x = _bf(300, 50, gen=g)
    c0 = torch.randn(50, generator=g, dtype=F64)
    cs, cb = O.colsum_ref(x, c0)
    torch.testing.assert_close(cs, c0 + x.sum(0), **TIGHT)
    assert O.excess(cs - x[-1], cs, cb).any()                # one row short


# ------------------------------------------------------------------------------------------------ attention
def _attn_inputs(B, S, H, Dh, bias_kind, seed):
    g = _gen(seed)
    q, k, v, do = (_bf(B, H, S, Dh, gen=g) for _ in range(4))
    kb = None
    if bias_kind == "bert":
        kb = torch.zeros(B, S, dtype=F64)
        kb[:, S - max(1, S // 4):] = -10000.0
    elif bias_kind == "random":
        kb = torch.randn(B, S, generator=g, dtype=torch.float32).double()
    return q, k, v, do, kb


def _attn_torch(q, k, v, kb, drop=None):
    B, H, S, Dh = q.shape
    x = q @ k.transpose(-1, -2) / math.sqrt(Dh)
    if kb is not None:
        x = x + kb[:, None, None, :]
    p = torch.softmax(x, -1)
    if drop is not None:
        p = p * drop
    return p @ v


@pytest.mark.parametrize("bias_kind", [None, "bert", "random"])
def test_attention_ref_matches_sdpa(bias_kind):
    B, S, H, Dh = 2, 37, 3, 32
    q, k, v, do, kb = _attn_inputs(B, S, H, Dh, bias_kind, 4)
    fw = O.attention_fwd_ref(q, k, v, kb)
    qt, kt, vt = (t.clone().requires_grad_(True) for t in (q, k, v))
    mask = kb[:, None, None, :].expand(B, H, S, S) if kb is not None else None
    ot = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask)
    torch.testing.assert_close(fw["o"], ot.detach(), **TIGHT)
    x = q @ k.transpose(-1, -2) / math.sqrt(Dh) + (kb[:, None, None, :] if kb is not None else 0)
    torch.testing.assert_close(fw["lse"], torch.logsumexp(x, -1), **TIGHT)
    ot.backward(do)
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    for name, t in (("dq", qt), ("dk", kt), ("dv", vt)):
        torch.testing.assert_close(bw[name], t.grad, **TIGHT)


def test_attention_ref_matches_multi_head_attention_forward():
    """nn.MultiheadAttention's functional form with identity projections and a float key-padding mask."""
    B, S, H, Dh = 2, 20, 4, 32
    E = H * Dh
    q, k, v, do, kb = _attn_inputs(B, S, H, Dh, "random", 5)
    seq = lambda t: t.transpose(1, 2).reshape(B, S, E).transpose(0, 1)           # [S, B, E]
    eye = torch.eye(E, dtype=F64)
    qs, ks, vs = (seq(t).clone().requires_grad_(True) for t in (q, k, v))
    out, _ = F.multi_head_attention_forward(qs, ks, vs, E, H, None, torch.zeros(3 * E, dtype=F64), None, None, False, 0.0,
                                            eye, torch.zeros(E, dtype=F64), training=False, key_padding_mask=kb,
                                            need_weights=False, use_separate_proj_weight=True, q_proj_weight=eye,
                                            k_proj_weight=eye, v_proj_weight=eye)
    fw = O.attention_fwd_ref(q, k, v, kb)
    torch.testing.assert_close(seq(fw["o"]), out.detach(), **TIGHT)
    out.backward(seq(do))
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    for name, t in (("dq", qs), ("dk", ks), ("dv", vs)):
        torch.testing.assert_close(seq(bw[name]), t.grad, **TIGHT)


def test_attention_ref_with_dropout_matches_autograd():
    B, S, H, Dh = 2, 30, 2, 64
    q, k, v, do, kb = _attn_inputs(B, S, H, Dh, "bert", 6)
    drop = O.keep_scale(O.attn_drop_index(B, H, S), 0.1, 77)
    qt, kt, vt = (t.clone().requires_grad_(True) for t in (q, k, v))
    ot = _attn_torch(qt, kt, vt, kb, drop)
    ot.backward(do)
    fw = O.attention_fwd_ref(q, k, v, kb, drop)
    torch.testing.assert_close(fw["o"], ot.detach(), **TIGHT)
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    for name, t in (("dq", qt), ("dk", kt), ("dv", vt)):
        torch.testing.assert_close(bw[name], t.grad, **TIGHT)


def _attn_emulate(q, k, v, do, kb, drop):
    """fp32 / bf16 emulation of attn_fwd_kernel and attn_bwd_kernel's rounding steps."""
    B, H, S, Dh = q.shape
    f = lambda t: t.float()
    scale = torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(Dh)))
    x = (f(q) @ f(k).transpose(-1, -2)) * scale + (f(kb)[:, None, None, :] if kb is not None else 0)
    mx = x.amax(-1, keepdim=True)
    e = torch.exp(x - mx)
    sm = e.sum(-1, keepdim=True)
    pd = O.bf16((e * (f(drop) if drop is not None else 1)).double()).float()
    o = (pd @ f(v)) * (1 / sm)
    lse = mx + torch.log(sm)
    p = torch.exp(x - lse)
    g = (f(do) @ f(v).transpose(-1, -2)) * (f(drop) if drop is not None else 1)
    D = (p * g).sum(-1, keepdim=True)
    ds = O.bf16((p * (g - D) * scale).double()).float()
    pd2 = O.bf16((p * (f(drop) if drop is not None else 1)).double()).float()
    r = lambda t: O.bf16(t.double())
    return r(o), lse.squeeze(-1).double(), r(ds @ f(k)), r(ds.transpose(-1, -2) @ f(q)), r(pd2.transpose(-1, -2) @ f(do))


@pytest.mark.parametrize("S,Dh,bias_kind,p", [(1, 32, None, 0.0), (65, 64, "bert", 0.0), (128, 32, "random", 0.1),
                                             (99, 64, None, 0.1)])
def test_attention_bounds_hold_for_fp32_emulation(S, Dh, bias_kind, p):
    B, H = 2, 2
    q, k, v, do, kb = _attn_inputs(B, S, H, Dh, bias_kind, 7)
    drop = O.keep_scale(O.attn_drop_index(B, H, S), p, 5) if p else None
    fw = O.attention_fwd_ref(q, k, v, kb, drop)
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    o, lse, dq, dk, dv = _attn_emulate(q, k, v, do, kb, drop)
    assert O.check(o, fw["o"], fw["o_bound"], "o") <= 1
    assert O.check(lse, fw["lse"], fw["lse_bound"], "lse") <= 1
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        assert O.check(got, bw[name], bw[name + "_bound"], name) <= 1


def test_attention_bounds_reject_plausible_mistakes():
    B, S, H, Dh = 2, 64, 4, 32
    q, k, v, do, kb = _attn_inputs(B, S, H, Dh, "random", 8)
    fw = O.attention_fwd_ref(q, k, v, kb)
    o, ob = fw["o"], fw["o_bound"]
    bw = O.attention_bwd_ref(fw, q, k, v, do)
    # the last key dropped
    assert O.excess(_attn_torch(q[:, :, :, :], k[:, :, :-1], v[:, :, :-1], kb[:, :-1]), o, ob).any()
    # two adjacent heads swapped
    assert O.excess(o[:, [1, 0, 2, 3]], o, ob).any()
    # 1/sqrt(E) instead of 1/sqrt(Dh)
    wrong = _attn_torch(q * math.sqrt(Dh / (H * Dh)), k, v, kb)
    assert O.excess(wrong, o, ob).any()
    # key bias applied along the query axis
    x = q @ k.transpose(-1, -2) / math.sqrt(Dh) + kb[:, None, :, None]
    assert O.excess(torch.softmax(x, -1) @ v, o, ob).any()
    # the same mistakes in the backward
    qt, kt, vt = (t.clone().requires_grad_(True) for t in (q, k, v))
    _attn_torch(qt * math.sqrt(1 / H), kt, vt, kb).backward(do)
    assert O.excess(qt.grad * math.sqrt(1 / H), bw["dq"], bw["dq_bound"]).any()
    assert O.excess(kt.grad, bw["dk"], bw["dk_bound"]).any()
    qt, kt, vt = (t.clone().requires_grad_(True) for t in (q, k, v))
    _attn_torch(qt[:, :, :, :], kt[:, :, :-1], vt[:, :, :-1], kb[:, :-1]).backward(do)
    assert O.excess(qt.grad, bw["dq"], bw["dq_bound"]).any()
    # dropout: a mask drawn with the wrong seed, or without the seed offset
    drop = O.keep_scale(O.attn_drop_index(B, H, S), 0.1, 3, ofs=5)
    fwd = O.attention_fwd_ref(q, k, v, kb, drop)
    other = O.keep_scale(O.attn_drop_index(B, H, S), 0.1, 3)
    assert O.excess(_attn_torch(q, k, v, kb, other), fwd["o"], fwd["o_bound"]).any()
    # lse of the unscaled logits
    assert O.excess(torch.logsumexp(q @ k.transpose(-1, -2) + kb[:, None, None, :], -1), fw["lse"], fw["lse_bound"]).any()


# ------------------------------------------------------------------------------------------------ LayerNorm
def test_layernorm_ref_matches_torch():
    g = _gen(9)
    rows, D = 13, 96
    pre = _bf(rows, D, gen=g) * 3 + 1
    gamma = torch.rand(D, generator=g, dtype=F64) + 0.5
    beta = torch.randn(D, generator=g, dtype=F64)
    dy = _bf(rows, D, gen=g)
    y, _, mu, rs = O.ln_fwd_ref(pre, gamma, beta)
    pt, gt, bt = (t.clone().requires_grad_(True) for t in (pre, gamma, beta))
    yt = F.layer_norm(pt, (D,), gt, bt, 1e-5)
    torch.testing.assert_close(y, yt.detach(), **TIGHT)
    torch.testing.assert_close(rs, 1 / torch.sqrt(pre.var(-1, unbiased=False) + 1e-5), **TIGHT)
    yt.backward(dy)
    dg0, db0 = torch.randn(D, generator=g, dtype=F64), torch.randn(D, generator=g, dtype=F64)
    bw = O.ln_bwd_ref(dy, pre, gamma, 1e-5, dg0, db0)
    torch.testing.assert_close(bw["dpre"], pt.grad, **TIGHT)
    torch.testing.assert_close(bw["dgamma"], dg0 + gt.grad, **TIGHT)
    torch.testing.assert_close(bw["dbeta"], db0 + bt.grad, **TIGHT)


def _ln_emulate(pre, gamma, beta, dy, eps=1e-5):
    """fp32 single-pass statistics (E[x^2] - mu^2), as ln_fwd_kernel / ln_bwd_kernel compute them."""
    D = pre.shape[1]
    p = pre.float()
    mu = p.sum(1, keepdim=True) / D
    var = ((p * p).sum(1, keepdim=True) / D - mu * mu).clamp_min(0)
    rs = torch.rsqrt(var + eps)
    xh = (p - mu) * rs
    y = xh * gamma.float() + beta.float()
    gd = dy.float() * gamma.float()
    a = gd.sum(1, keepdim=True) / D
    b = (gd * xh).sum(1, keepdim=True) / D
    dpre = rs * (gd - a - xh * b)
    return O.bf16(y.double()), O.bf16(dpre.double()), (dy.float() * xh).sum(0).double(), dy.float().sum(0).double()


@pytest.mark.parametrize("D,offset", [(2, 0.0), (64, 0.0), (1026, 0.0), (4096, 32.0), (768, 32.0)])
def test_layernorm_bounds_hold_for_fp32_emulation(D, offset):
    g = _gen(10)
    pre = O.bf16(torch.randn(9, D, generator=g, dtype=F64) + offset)
    gamma = torch.rand(D, generator=g, dtype=torch.float32).double() + 0.5
    beta = torch.randn(D, generator=g, dtype=torch.float32).double() * 0.1
    dy = _bf(9, D, gen=g)
    y, yb, _, _ = O.ln_fwd_ref(pre, gamma, beta)
    bw = O.ln_bwd_ref(dy, pre, gamma)
    ye, dpe, dge, dbe = _ln_emulate(pre, gamma, beta, dy)
    assert O.check(ye, y, yb, "y") <= 1
    assert O.check(dpe, bw["dpre"], bw["dpre_bound"], "dpre") <= 1
    assert O.check(dge, bw["dgamma"], bw["dgamma_bound"], "dgamma") <= 1
    assert O.check(dbe, bw["dbeta"], bw["dbeta_bound"], "dbeta") <= 1


def test_layernorm_bounds_reject_plausible_mistakes():
    g = _gen(11)
    rows, D = 16, 64
    pre = _bf(rows, D, gen=g)
    gamma = torch.rand(D, generator=g, dtype=F64) + 0.5
    beta = torch.zeros(D, dtype=F64)
    dy = _bf(rows, D, gen=g)
    y, yb, _, _ = O.ln_fwd_ref(pre, gamma, beta)
    # unbiased instead of biased variance
    mu = pre.mean(1, keepdim=True)
    wrong = (pre - mu) / torch.sqrt(pre.var(1, unbiased=True, keepdim=True) + 1e-5) * gamma + beta
    assert O.excess(wrong, y, yb).any()
    # dgamma / dbeta overwritten instead of accumulated
    dg0 = torch.ones(D, dtype=F64)
    bw = O.ln_bwd_ref(dy, pre, gamma, 1e-5, dg0, dg0)
    assert O.excess(bw["dgamma"] - dg0, bw["dgamma"], bw["dgamma_bound"]).any()
    assert O.excess(bw["dbeta"] - dg0, bw["dbeta"], bw["dbeta_bound"]).any()
    # the mean(g dy xhat) term left out of dpre
    mu, rs = pre.mean(1, keepdim=True), 1 / torch.sqrt(pre.var(1, unbiased=False, keepdim=True) + 1e-5)
    gd = gamma * dy
    assert O.excess(rs * (gd - gd.mean(1, keepdim=True)), bw["dpre"], bw["dpre_bound"]).any()


def test_ln_prologue_ref():
    g = _gen(12)
    x, r = _bf(5, 40, gen=g), _bf(5, 40, gen=g)
    drop = O.keep_scale(O.ln_drop_index(5, 40), 0.1, 9)
    pre, pb = O.ln_prologue_ref(x, r, drop)
    torch.testing.assert_close(pre, x * drop + r, **TIGHT)
    emu = O.bf16((x.float() * drop.float() + r.float()).double())
    assert O.check(emu, pre, pb, "pre") <= 1
    assert O.excess(x + r, pre, pb).any()                               # dropout not applied


# ------------------------------------------------------------------------------------------------ pointwise
@pytest.mark.parametrize("kind", ["relu", "gelu", "tanh"])
def test_act_bwd_ref_matches_autograd(kind):
    g = _gen(13)
    z = _bf(4000, scale=2.0, gen=g)
    dy = _bf(4000, gen=g)
    zt = z.clone().requires_grad_(True)
    fn = {"relu": F.relu, "gelu": F.gelu, "tanh": torch.tanh}[kind]
    y = fn(zt)
    y.backward(dy)
    ref = y.detach() if kind == "tanh" else z
    dz, dzb = O.act_bwd_ref(dy, ref, kind)
    torch.testing.assert_close(dz, zt.grad, **TIGHT)
    # fp32 emulation inside the bound (tanh takes the bf16-rounded output, as the kernel does)
    refb = O.bf16(ref)
    dzr, dzbr = O.act_bwd_ref(dy, refb, kind)
    if kind == "gelu":
        zf = refb.float()
        d = 0.5 * (1 + torch.erf(zf * 0.70710678)) + zf * 0.3989422804 * torch.exp(-0.5 * zf * zf)
    elif kind == "tanh":
        d = 1 - refb.float() ** 2
    else:
        d = (refb > 0).float()
    assert O.check(O.bf16((dy.float() * d).double()), dzr, dzbr, kind) <= 1


def test_embed3_ref_matches_nn_embedding():
    g = _gen(14)
    vocab, npos, D, B, S, pad = 50, 40, 24, 3, 17, 0
    word = torch.randn(vocab, D, generator=g, dtype=torch.float32).double()
    pos = torch.randn(npos, D, generator=g, dtype=torch.float32).double()
    typ = torch.randn(2, D, generator=g, dtype=torch.float32).double()
    ids = torch.randint(0, 6, (B, S), generator=g)                     # heavily repeated ids
    ids[:, -3:] = pad
    tts = torch.randint(0, 2, (B, S), generator=g)
    ew = torch.nn.Embedding(vocab, D, padding_idx=pad).double()
    ep = torch.nn.Embedding(npos, D).double()
    et = torch.nn.Embedding(2, D).double()
    with torch.no_grad():
        ew.weight.copy_(word), ep.weight.copy_(pos), et.weight.copy_(typ)
    out_t = ew(ids) + ep(torch.arange(S))[None] + et(tts)
    out, ob = O.embed3_fwd_ref(ids.flatten(), tts.flatten(), word, pos, typ, S)
    torch.testing.assert_close(out, out_t.detach().reshape(B * S, D), **TIGHT)
    gr = _bf(B, S, D, gen=g)
    out_t.backward(gr)
    z = lambda t: torch.zeros_like(t)
    dw, dwb, dp, dpb, dt, dtb = O.embed3_bwd_ref(ids.flatten(), tts.flatten(), gr.reshape(B * S, D), S, z(word), z(pos),
                                                  z(typ), pad)
    torch.testing.assert_close(dw, ew.weight.grad, **TIGHT)
    torch.testing.assert_close(dp, ep.weight.grad, **TIGHT)
    torch.testing.assert_close(dt, et.weight.grad, **TIGHT)
    # the padding row receiving a gradient is outside the bound
    wrong = torch.zeros_like(word).index_add_(0, ids.flatten(), gr.reshape(B * S, D))
    assert O.excess(wrong, dw, dwb).any()
    assert not O.excess(out_t.detach().reshape(B * S, D), out, ob).any()


# ------------------------------------------------------------------------------------------------ dropout hash
def _fmix32_int(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    return h ^ (h >> 16)


def test_dropout_hash_port():
    idx = torch.tensor([0, 1, 2, 12345, 2 ** 31 - 1, 2 ** 32 - 1, 2 ** 32 + 5], dtype=torch.int64)
    got = O.fmix32((O._mul32(idx & O.M32, O.GOLDEN) + 99) & O.M32)
    want = [_fmix32_int(((int(i) & 0xFFFFFFFF) * 0x9E3779B9 + 99) & 0xFFFFFFFF) for i in idx]
    assert got.tolist() == want
    assert O.mix_seed(7, None) == 7 and O.mix_seed(7, 3) == (7 + 3 * 0x9E3779B9) & 0xFFFFFFFF
    ks = O.keep_scale(O.flat_drop_index(1 << 16), 0.25, 11)
    assert set(ks.unique().tolist()) == {0.0, float(torch.tensor(1 / 0.75, dtype=torch.float32))}
    assert abs((ks > 0).double().mean().item() - 0.75) < 0.01
    assert not torch.equal(ks, O.keep_scale(O.flat_drop_index(1 << 16), 0.25, 11, ofs=1))
    assert not torch.equal(ks, O.keep_scale(O.flat_drop_index(1 << 16), 0.25, 12))
    # attention index layout: (blockIdx * 128 + row) * 128 + col with blockIdx = b * H + h
    ai = O.attn_drop_index(2, 3, 5)
    assert ai[1, 2, 4, 3].item() == ((1 * 3 + 2) * 128 + 4) * 128 + 3
