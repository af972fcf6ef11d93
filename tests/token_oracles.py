"""Float64 references of the token-model kernels, each with an elementwise error bound.

Every reference takes the bf16-rounded operands the kernel sees (as float64 tensors, on any device) and returns the
exact result together with a bound on how far the kernel may be from it.  The bounds follow the kernel's rounding
steps: fp32 accumulation (``(n + 2) * 2^-24`` of the sum of magnitudes), fp32 transcendental functions (a few ulp),
and a final rounding to bf16 (``2^-8`` of the magnitude: bf16 keeps 8 significand bits).  A kernel result passes when
``|got - ref| <= bound`` holds for every element; ``ratio()`` reports how much of the bound was used.

The dropout hash of ``transformer.cu`` is ported too (``keep_scale``), so that a kernel's exact mask can be rebuilt
for each of its index layouts.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

F64 = torch.float64
U_BF = 2.0 ** -8          # unit roundoff of bf16 (8 significand bits)
U_32 = 2.0 ** -24         # unit roundoff of fp32
M32 = 0xFFFFFFFF
GOLDEN = 0x9E3779B9       # the hash's multiplier, also the seed-offset multiplier


# ------------------------------------------------------------------------------------------------ comparison
def excess(got, ref, bound):
    """Elements where the kernel is outside the bound (``got`` any dtype)."""
    return (got.to(F64) - ref).abs() > bound


def ratio(got, ref, bound) -> float:
    """Worst |got - ref| / bound over all elements (0 where both are 0)."""
    err = (got.to(F64) - ref).abs()
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def check(got, ref, bound, what="") -> float:
    """Assert every element within its bound; return the worst ratio."""
    got = got.to(F64)
    bad = excess(got, ref, bound)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements outside the bound; first at flat index {i}: "
                             f"got {got.flatten()[i].item():.8g}, ref {ref.flatten()[i].item():.8g}, "
                             f"bound {bound.flatten()[i].item():.4g} (worst ratio {ratio(got, ref, bound):.3g})")
    return ratio(got, ref, bound)


def bf16(t):
    """Round to bf16 and back (the value a bf16 tensor holds)."""
    return t.to(torch.bfloat16).to(F64)


# ------------------------------------------------------------------------------------------------ dropout hash
def _mul32(a, b: int):
    """(a * b) mod 2^32 for int64 tensors a in [0, 2^32) without int64 overflow."""
    lo = (a * (b & 0xFFFF)) & M32
    hi = ((a * (b >> 16)) & 0xFFFF) << 16
    return (lo + hi) & M32


def fmix32(h):
    """MurmurHash3's 32-bit finaliser on int64 tensors holding uint32 values."""
    h = h ^ (h >> 16)
    h = _mul32(h, 0x85EBCA6B)
    h = h ^ (h >> 13)
    h = _mul32(h, 0xC2B2AE35)
    return h ^ (h >> 16)


def mix_seed(seed: int, ofs=None) -> int:
    """The launch seed after the optional device seed offset is mixed in: seed + ofs * 0x9E3779B9 (mod 2^32)."""
    seed &= M32
    return seed if ofs is None else (seed + (int(ofs) & M32) * GOLDEN) & M32


def keep_scale(idx, p: float, seed: int, ofs=None):
    """Per-element dropout scale the kernels apply: 1/(1-p) where kept, 0 where dropped.  ``idx``: int64 tensor of the
    kernel's element indices (taken mod 2^32, as the kernel's uint32 arithmetic does)."""
    s = mix_seed(seed, ofs)
    r = fmix32((_mul32(idx & M32, GOLDEN) + s) & M32) >> 8           # 24 random bits
    p32 = float(torch.tensor(p, dtype=torch.float32))                 # the kernel compares against fp32 p
    keep = r.to(F64) * 2.0 ** -24 >= p32
    inv_keep = float(torch.tensor(1.0, dtype=torch.float32) / (1.0 - torch.tensor(p, dtype=torch.float32)))
    return keep.to(F64) * inv_keep


def attn_drop_index(B, H, S, device=None):
    """[B, H, S, S] element indices of attention dropout: (blockIdx * 128 + query) * 128 + key, blockIdx = b * H + h."""
    blk = torch.arange(B * H, device=device, dtype=torch.int64).view(B, H, 1, 1)
    q = torch.arange(S, device=device, dtype=torch.int64).view(1, 1, S, 1)
    k = torch.arange(S, device=device, dtype=torch.int64).view(1, 1, 1, S)
    return (blk * 128 + q) * 128 + k


def ln_drop_index(rows, D, device=None):
    """[rows, D] element indices of the LayerNorm prologue's dropout: row * D + col."""
    return torch.arange(rows * D, device=device, dtype=torch.int64).view(rows, D)


def flat_drop_index(n, device=None):
    """Element indices of ``dropout_bf16``: the flat index."""
    return torch.arange(n, device=device, dtype=torch.int64)


# ------------------------------------------------------------------------------------------------ activations
def act_ref(z, act):
    if act in (None, "none"):
        return z
    if act == "relu":
        return z.clamp_min(0)
    if act == "gelu":
        return 0.5 * z * (1 + torch.erf(z / math.sqrt(2.0)))
    if act == "tanh":
        return torch.tanh(z)
    raise ValueError(act)


# Lipschitz constant of each activation, rounded up to a power of two (GELU-erf's slope peaks at 1.129)
_LIP = {None: 1.0, "none": 1.0, "relu": 1.0, "tanh": 1.0, "gelu": 2.0}


def _act_eval_err(z, y, act):
    """fp32 evaluation error of the epilogue's activation: erff / tanhf are within 2 ulp, GELU adds three roundings."""
    if act == "gelu":
        return 2.0 ** -21 * (y.abs() + z.abs())
    if act == "tanh":
        return 2.0 ** -22 * y.abs()
    return torch.zeros_like(z)


# ------------------------------------------------------------------------------------------------ GEMM
def gemm_ref(a, b, bias=None, residual=None, act=None):
    """Epilogue GEMM ``out = act(A B^T + bias + residual)`` of ``gemm_act``; A [M, K], B [N, K], float64.

    Returns ``(out, out_bound, pre, pre_bound)``: ``pre`` is the pre-activation ``aux`` receives."""
    K = a.shape[1]
    z = a @ b.T
    mag = a.abs() @ b.abs().T
    if bias is not None:
        z = z + bias
        mag = mag + bias.abs()
    if residual is not None:
        z = z + residual
        mag = mag + residual.abs()
    # fp32 accumulation of K products, then the bias and residual adds: (K + 2) roundings of at most 2^-24 of the sum
    e_z = (K + 2) * U_32 * mag
    y = act_ref(z, act)
    # bf16 rounding of the fp32 result, which is itself off by the (activated) accumulation error
    pre_bound = U_BF * z.abs() + (1 + U_BF) * e_z
    out_bound = U_BF * y.abs() + (1 + U_BF) * (_LIP[act] * e_z + _act_eval_err(z, y, act))
    return y, out_bound, z, pre_bound


def gemm_f32_ref(a, b, out0, k_split=1):
    """``gemm_f32``: out = out0 + A B^T with fp32 partial sums added into the live buffer, ``k_split`` slices."""
    K = a.shape[1]
    ref = out0 + a @ b.T
    # K products accumulated per slice, then one add per slice into the buffer
    bound = (K + k_split + 2) * U_32 * (out0.abs() + a.abs() @ b.abs().T)
    return ref, bound


def colsum_ref(x, out0):
    """``colsum_bf16``: out[c] = out0[c] + sum_r x[r][c], fp32 partial sums per block added with atomics."""
    rows = x.shape[0]
    return out0 + x.sum(0), (rows + 2) * U_32 * (out0.abs() + x.abs().sum(0))


# ------------------------------------------------------------------------------------------------ attention
def _heads(t, B, S, H, Dh, col, ld):
    """Head view [B, H, S, Dh] (float64) of head-packed columns [col, col + H * Dh) of a [B * S, ld] tensor."""
    return t.reshape(B * S, ld)[:, col:col + H * Dh].to(F64).reshape(B, S, H, Dh).transpose(1, 2)


def attention_fwd_ref(q, k, v, key_bias=None, drop=None):
    """Dense softmax attention per head.  q, k, v: [B, H, S, Dh] float64; key_bias: [B, S] (fp32 values) or None;
    drop: [B, H, S, S] keep-scale (0 or 1/(1-p)) or None.

    Returns a dict with ``o`` [B, H, S, Dh], ``lse`` [B, H, S] and their bounds, plus what the backward reference needs."""
    B, H, S, Dh = q.shape
    scale = 1.0 / math.sqrt(Dh)
    s = q @ k.transpose(-1, -2)
    x = s * scale
    if key_bias is not None:
        x = x + key_bias[:, None, None, :]
    lse = torch.logsumexp(x, -1)
    P = torch.exp(x - lse[..., None])
    Pd = P * drop if drop is not None else P
    o = Pd @ v
    # absolute error of a logit: fp32 accumulation of Dh products, the scale multiply and the bias add
    e_x = scale * (Dh + 2) * U_32 * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -22 * x.abs()
    if key_bias is not None:
        e_x = e_x + U_32 * key_bias.abs()[:, None, None, :]
    mx = x.amax(-1, keepdim=True)
    # relative error of exp((x - max) log2e): the logit error, rounding of the argument (2 ops) and exp2f (2 ulp)
    e_exp = e_x + 2.0 ** -22 * (x - mx).abs() + 2.0 ** -22
    # relative error of a normalised probability: its own exponent error, the P-weighted errors of the row sum (which
    # contributes log-derivative weights P) and the fp32 row sum (S adds) and reciprocal
    e_rowsum = (P * e_exp).sum(-1, keepdim=True)
    eps_p = e_exp + e_rowsum + (S + 4) * U_32
    # O = (sum_j bf16(p~_j) v_j) / sum: P~ rounded to bf16 (2^-8), fp32 P~ V over S keys, the 1/sum scale, bf16 store
    PdV = Pd.abs() @ v.abs()
    o_bound = U_BF * o.abs() + (1 + U_BF) * (((U_BF + eps_p) * Pd) @ v.abs() + (S + 4) * U_32 * PdV)
    # lse = max + logf(sum): the P-weighted logit error, the sum's roundings, logf (1 ulp) and the final add
    lse_bound = (P * e_x).sum(-1) + (S + 8) * U_32 + 2.0 ** -22 * lse.abs()
    return {"o": o, "o_bound": o_bound, "lse": lse, "lse_bound": lse_bound, "P": P, "Pd": Pd, "x": x, "e_x": e_x,
            "drop": drop, "scale": scale}


def attention_bwd_ref(fw, q, k, v, do):
    """Backward of ``attention_fwd_ref`` for output gradient ``do`` [B, H, S, Dh]: dq, dk, dv and their bounds.

    The kernel recomputes P from its own log-sum-exp, forms dP = dO V^T, D = rowsum(P * dP~), dS = P (dP~ - D) scale
    (rounded to bf16) and the three products dV = P~^T dO, dQ = dS K, dK = dS^T Q."""
    B, H, S, Dh = q.shape
    P, Pd, x, e_x, drop, scale = fw["P"], fw["Pd"], fw["x"], fw["e_x"], fw["drop"], fw["scale"]
    dP = do @ v.transpose(-1, -2)
    dPd = dP * drop if drop is not None else dP
    Dr = (P * dPd).sum(-1, keepdim=True)
    dS = P * (dPd - Dr) * scale
    dv = Pd.transpose(-1, -2) @ do
    dq = dS @ k
    dk = dS.transpose(-1, -2) @ q
    # relative error of the recomputed P: the logit error, the kernel's lse error, the argument's roundings, exp2f
    e_lse = fw["lse_bound"][..., None]
    eps_b = e_x + e_lse + 2.0 ** -22 * (x - fw["lse"][..., None]).abs() + 2.0 ** -22
    ks = drop if drop is not None else torch.ones_like(P)
    e_dP = (Dh + 2) * U_32 * (do.abs() @ v.abs().transpose(-1, -2)) * ks      # fp32 accumulation, then the keep-scale
    e_D = (P * (eps_b * dPd.abs() + e_dP)).sum(-1, keepdim=True) + (S + 2) * U_32 * (P * dPd.abs()).sum(-1, keepdim=True)
    # dS rounded to bf16 after three fp32 multiplies
    e_dS = U_BF * dS.abs() + (1 + U_BF) * (scale * P * (eps_b * (dPd - Dr).abs() + e_dP + e_D) + 2.0 ** -22 * dS.abs())
    dq_bound = U_BF * dq.abs() + (1 + U_BF) * (e_dS @ k.abs() + (S + 2) * U_32 * (dS.abs() @ k.abs()))
    dk_bound = U_BF * dk.abs() + (1 + U_BF) * (e_dS.transpose(-1, -2) @ q.abs() + (S + 2) * U_32 * (dS.abs().transpose(-1, -2) @ q.abs()))
    # P~ = bf16(P * keep-scale): the recomputation error plus the bf16 rounding
    e_Pd = (U_BF + (1 + U_BF) * (eps_b + U_32)) * Pd.abs()
    dv_bound = U_BF * dv.abs() + (1 + U_BF) * (e_Pd.transpose(-1, -2) @ do.abs()
                                                + (S + 2) * U_32 * (Pd.abs().transpose(-1, -2) @ do.abs()))
    return {"dq": dq, "dq_bound": dq_bound, "dk": dk, "dk_bound": dk_bound, "dv": dv, "dv_bound": dv_bound}


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_prologue_ref(x, res=None, drop=None):
    """pre = drop(x) + res in fp32, rounded to bf16 (the kernel normalises, and its backward re-reads, the bf16 values).
    Returns ``(pre, bound)`` where pre is the exact fp64 value before rounding."""
    t = x * drop if drop is not None else x
    pre = t + res if res is not None else t
    # fp32: the keep-scale multiply and the residual add, then the bf16 store
    e = 2 * U_32 * (t.abs() + (res.abs() if res is not None else 0))
    return pre, U_BF * pre.abs() + (1 + U_BF) * e


def ln_stats(pre, eps):
    D = pre.shape[-1]
    mu = pre.mean(-1, keepdim=True)
    var = ((pre - mu) ** 2).mean(-1, keepdim=True)           # biased, like the kernel and torch
    rs = 1.0 / torch.sqrt(var + eps)
    # single-pass fp32 statistics: each lane adds D / 32 values in sequence, then a 5-level shuffle tree
    depth = D / 32 + 8
    e_mu = depth * U_32 * pre.abs().mean(-1, keepdim=True)
    msq = (pre * pre).mean(-1, keepdim=True)
    # var = E[x^2] - mu^2: the error of E[x^2], of mu^2 and of the subtraction (cancels the offset: scales with E[x^2])
    e_var = (depth + 1) * U_32 * msq + 2 * mu.abs() * e_mu + 2 * U_32 * msq
    # relative error of rstd: half the relative error of var + eps, plus rsqrtf (2 ulp)
    eps_rs = e_var / (2 * (var + eps)) + 2.0 ** -22
    return mu, rs, e_mu, eps_rs


def ln_fwd_ref(pre, gamma, beta, eps=1e-5):
    """y = (pre - mean) * rstd * gamma + beta over the last axis; ``pre`` holds the bf16 values the kernel normalises.
    Returns ``(y, y_bound, mean, rstd)``."""
    mu, rs, e_mu, eps_rs = ln_stats(pre, eps)
    xh = (pre - mu) * rs
    y = xh * gamma + beta
    # error of xhat from the statistics, then three fp32 roundings (subtract, multiply twice) and the bf16 store
    e_xh = xh.abs() * eps_rs + rs * e_mu + 2.0 ** -22 * xh.abs()
    bound = U_BF * y.abs() + (1 + U_BF) * (gamma.abs() * e_xh + 2.0 ** -22 * (xh * gamma).abs() + U_32 * beta.abs())
    return y, bound, mu.squeeze(-1), rs.squeeze(-1)


def ln_bwd_ref(dy, pre, gamma, eps=1e-5, dgamma0=None, dbeta0=None):
    """LayerNorm backward: dpre = rstd (g dy - mean(g dy) - xhat mean(g dy xhat)), dgamma += sum dy xhat,
    dbeta += sum dy.  Returns a dict of values and bounds."""
    rows, D = pre.shape
    mu, rs, e_mu, eps_rs = ln_stats(pre, eps)
    xh = (pre - mu) * rs
    gd = gamma * dy
    a = gd.mean(-1, keepdim=True)
    bs = (gd * xh).mean(-1, keepdim=True)
    dpre = rs * (gd - a - xh * bs)
    e_xh = xh.abs() * eps_rs + rs * e_mu + 2.0 ** -22 * xh.abs()
    depth = D / 32 + 8
    e_a = depth * U_32 * gd.abs().mean(-1, keepdim=True)
    e_b = depth * U_32 * (gd * xh).abs().mean(-1, keepdim=True) + (gd.abs() * e_xh).mean(-1, keepdim=True)
    inner = (gd - a - xh * bs).abs()
    e_dpre = (rs * (e_a + xh.abs() * e_b + bs.abs() * e_xh) + eps_rs * (rs * inner)
              + 2.0 ** -22 * rs * (gd.abs() + a.abs() + (xh * bs).abs() + inner))
    dpre_bound = U_BF * dpre.abs() + (1 + U_BF) * e_dpre
    dg0 = dgamma0 if dgamma0 is not None else torch.zeros_like(gamma)
    db0 = dbeta0 if dbeta0 is not None else torch.zeros_like(gamma)
    dgamma = dg0 + (dy * xh).sum(0)
    dbeta = db0 + dy.sum(0)
    # fp32 sums over the rows (registers / shared memory / global atomics) plus the xhat error of every term
    dgamma_bound = (rows + 4) * U_32 * (dg0.abs() + (dy * xh).abs().sum(0)) + (dy.abs() * (e_xh + U_32 * xh.abs())).sum(0)
    dbeta_bound = (rows + 4) * U_32 * (db0.abs() + dy.abs().sum(0))
    return {"dpre": dpre, "dpre_bound": dpre_bound, "dgamma": dgamma, "dgamma_bound": dgamma_bound, "dbeta": dbeta,
            "dbeta_bound": dbeta_bound}


# ------------------------------------------------------------------------------------------------ pointwise
def act_bwd_ref(dy, ref, kind):
    """``act_bwd``: dz = dy * act'(.); ref = pre-activation (relu, gelu) or output (tanh).  Returns ``(dz, bound)``."""
    if kind == "relu":
        d = (ref > 0).to(F64)
        e = torch.zeros_like(dy)
    elif kind == "gelu":
        phi = torch.exp(-0.5 * ref * ref) / math.sqrt(2 * math.pi)
        d = 0.5 * (1 + torch.erf(ref / math.sqrt(2.0))) + ref * phi
        # erff (2 ulp) and the adds: 2^-21; __expf is within 2 + 1.16 x ulp (ulp = 2^-23) at x = z^2 / 2, at most
        # (2 + z^2) * 2^-23 of the |z| phi term, plus its three multiplies
        e = dy.abs() * (2.0 ** -21 + (8 + 2 * ref * ref) * U_32 * (ref * phi).abs())
    elif kind == "tanh":
        d = 1 - ref * ref
        e = dy.abs() * U_32 * (1 + ref * ref)                           # z^2 is exact in fp32, one subtract
    else:
        raise ValueError(kind)
    dz = dy * d
    return dz, U_BF * dz.abs() + (1 + U_BF) * (e + U_32 * dz.abs())


def embed3_fwd_ref(ids, tts, word, pos, typ, S):
    """word[ids] + pos[t % S] + type[tt or 0] (fp32 tables, two fp32 adds, bf16 store).  ids / tts: [tokens]."""
    t = torch.arange(ids.numel(), device=ids.device) % S
    tt = tts if tts is not None else torch.zeros_like(ids)
    a, b, c = word[ids], pos[t], typ[tt]
    out = a + b + c
    return out, U_BF * out.abs() + (1 + U_BF) * 2 * U_32 * (a.abs() + b.abs() + c.abs())


def embed3_bwd_ref(ids, tts, g, S, dword0, dpos0, dtyp0, pad_id=-1):
    """Scatter-add of ``g`` [tokens, D] into the word / position / type gradients (the padding id's row gets none)."""
    tokens = ids.numel()
    t = torch.arange(tokens, device=ids.device) % S
    tt = tts if tts is not None else torch.zeros_like(ids)
    keep = (ids != pad_id).to(F64)[:, None]
    out = []
    for base, idx, w in ((dword0, ids, keep), (dpos0, t, None), (dtyp0, tt, None)):
        gg = g * w if w is not None else g
        ref = base.clone().index_add_(0, idx, gg)
        mag = base.abs().clone().index_add_(0, idx, gg.abs())
        # fp32 atomic adds, one per token that hits the row
        out += [ref, (tokens + 2) * U_32 * mag]
    return out
