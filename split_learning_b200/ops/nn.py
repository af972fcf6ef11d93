"""Autograd-visible wrappers of the token-model kernels (``csrc/transformer.cu`` + the wgmma GEMM).

Each ``torch.autograd.Function`` below is one fused native op — forward *and* backward are hand-written sm_90a
kernels; torch only keeps the tape.  Activations are bf16, parameters stay fp32 ``nn.Parameter``s (state-dict, FedAvg,
LoRA and the flat fused optimizer are unchanged) and are read through a bf16 shadow: the one the flat optimizer
refreshes inside its update kernel (``ops.optim``), or a cached cast for frozen parameters.  Weight / bias /
LayerNorm / embedding gradients are accumulated by the kernels straight into ``param.grad`` (fp32, the flat
gradient buffer), so the functions return ``None`` for them.

Covers SURVEY §2.7 G11: Linear (+bias +GELU/tanh/ReLU +residual epilogues), LayerNorm (+dropout+residual prologue),
dense softmax attention S <= 128 (+key-padding bias, +probability dropout), dropout, BERT embeddings.
"""
from __future__ import annotations

import random
import threading
from typing import Optional

import torch

from . import native as N

_BF = torch.bfloat16
_rng = random.Random(0x5EED)


def seed_all(seed: int) -> None:
    _rng.seed(seed)


def next_seed() -> int:
    return _rng.getrandbits(32)


_tls = threading.local()


def set_seed_offset(counter: Optional[torch.Tensor]) -> None:
    """Device uint32/int32 scalar mixed into every dropout seed issued from this thread (``None`` = off).  A
    graph-captured step points it at its replay counter so that masks differ between replays."""
    _tls.seed_ofs = counter


def _seed_ofs():
    return getattr(_tls, "seed_ofs", None)


def bf16_of(p: torch.Tensor) -> torch.Tensor:
    """bf16 view of a parameter: optimizer-maintained shadow when there is one, cached cast otherwise."""
    sh = getattr(p, "_slb_bf16", None)
    if sh is not None:
        if getattr(p, "_slb_ver", None) != p._version:       # a torch in-place write (load_state_dict, FedAvg, merge)
            with torch.no_grad():
                sh.copy_(p.detach())
            p._slb_ver = p._version
        return sh
    c = getattr(p, "_slb_cache", None)
    if c is None or c[0] != p._version or c[1].device != p.device:
        c = (p._version, p.detach().to(_BF).contiguous())
        p._slb_cache = c
    return c[1]


def _grad_buf(p: torch.Tensor) -> torch.Tensor:
    if p.grad is None:
        p.grad = torch.zeros_like(p, memory_format=torch.contiguous_format)
    return p.grad


def _as_bf16(x: torch.Tensor) -> torch.Tensor:
    return x if x.dtype == _BF else x.to(_BF)


def _pad8(t: torch.Tensor) -> torch.Tensor:
    """[M, n] bf16 -> [M, ceil8(n)] zero padded (TMA needs 16-byte row pitches)."""
    n = t.shape[1]
    if n % 8 == 0:
        return t
    out = torch.zeros(t.shape[0], (n + 7) // 8 * 8, dtype=t.dtype, device=t.device)
    out[:, :n] = t
    return out


# --------------------------------------------------------------------------------------------- Linear
class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual, act):
        n_out = weight.shape[0]                       # any trailing shape (conv patch-embedding weights) = [n_out, -1]
        k_in = weight.numel() // n_out
        lead = x.shape[:-1]
        if k_in % 8:
            raise N.NativeError("native linear: in_features must be a multiple of 8")
        x2 = _as_bf16(x).reshape(-1, k_in).contiguous()
        m = x2.shape[0]
        wb = bf16_of(weight).view(n_out, k_in)
        out = torch.empty(m, n_out, dtype=_BF, device=x.device)
        aux = torch.empty_like(out) if act in ("gelu", "relu") else None
        res2 = _as_bf16(residual).reshape(m, n_out).contiguous() if residual is not None else None
        N.gemm_act(x2, wb, out, m, n_out, k_in, bias=bias, act=act, aux=aux, residual=res2)
        ctx.act, ctx.has_res, ctx.lead = act, residual is not None, lead
        ctx.weight, ctx.bias = weight, bias
        ctx.save_for_backward(x2, aux if aux is not None else (out if act == "tanh" else None))
        return out.view(*lead, n_out)

    @staticmethod
    def backward(ctx, dy):
        x2, ref = ctx.saved_tensors
        weight, bias = ctx.weight, ctx.bias
        n_out = weight.shape[0]
        k_in = weight.numel() // n_out
        m = x2.shape[0]
        dy2 = _as_bf16(dy).reshape(m, n_out).contiguous()
        if ctx.act:
            dz = torch.empty_like(dy2)
            N.act_bwd(dy2, ref, dz, dy2.numel(), ctx.act)
        else:
            dz = dy2
        dzp = _pad8(dz)
        ldz = dzp.shape[1]
        if weight.requires_grad:
            tiles = ((n_out + 127) // 128) * ((k_in + 63) // 64)
            ks = max(1, min((m + 63) // 64, N.num_sms(dy.device) // max(tiles, 1)))
            # dW[n][k] += sum_t dz[t][n] x[t][k]     (both operands MN-major: token-major storage is the K axis)
            N.gemm_f32(dzp, x2, _grad_buf(weight).view(n_out, k_in), n_out, k_in, m, a_mn=True, b_mn=True, lda=ldz, ldb=k_in, ldo=k_in,
                       k_split=ks)
        if bias is not None and bias.requires_grad:
            N.colsum_bf16(dzp, _grad_buf(bias), m, n_out, ldz)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(m, k_in, dtype=_BF, device=dy.device)
            # dx[t][k] = sum_n dz[t][n] W[n][k]      (B = the [N][K] weight read MN-major, no transposed copy)
            N.gemm_act(dzp, bf16_of(weight).view(n_out, k_in), dx, m, k_in, n_out, b_mn=True, lda=ldz, ldb=k_in)
            dx = dx.view(*ctx.lead, k_in)
        dres = dz.view(*ctx.lead, n_out) if ctx.has_res else None
        return dx, None, None, dres, None


def linear(x, weight, bias=None, act: Optional[str] = None, residual=None):
    """act(x W^T + b + residual) -> bf16.  ``residual`` is added before the activation (fused in the GEMM epilogue)."""
    return _LinearFn.apply(x, weight, bias, residual, act)


# --------------------------------------------------------------------------------------------- LayerNorm
class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, residual, eps, p_drop, seed):
        d = x.shape[-1]
        x2 = _as_bf16(x).reshape(-1, d).contiguous()
        rows = x2.shape[0]
        fused = residual is not None or p_drop > 0.0
        res2 = _as_bf16(residual).reshape(rows, d).contiguous() if residual is not None else None
        y = torch.empty_like(x2)
        pre = torch.empty_like(x2) if fused else None
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        ofs = _seed_ofs() if p_drop > 0.0 else None
        N.ln_fwd(x2, res2, gamma, beta, y, pre, mean, rstd, rows, d, eps, p_drop, seed, ofs)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.cfg = (x.shape, residual is not None, p_drop, seed, ofs)
        ctx.save_for_backward(pre if fused else x2, mean, rstd)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        pre, mean, rstd = ctx.saved_tensors
        shape, has_res, p_drop, seed, ofs = ctx.cfg
        rows, d = pre.shape
        dy2 = _as_bf16(dy).reshape(rows, d).contiguous()
        dpre = torch.empty_like(dy2)
        train = ctx.gamma.requires_grad
        N.ln_bwd(dy2, pre, ctx.gamma, mean, rstd, dpre, _grad_buf(ctx.gamma) if train else None,
                 _grad_buf(ctx.beta) if train else None, rows, d)
        dx = dpre
        if p_drop > 0.0:
            dx = torch.empty_like(dpre)
            N.dropout_bf16(dpre, dx, dpre.numel(), p_drop, seed, ofs)
        return dx.view(shape), None, None, (dpre.view(shape) if has_res else None), None, None, None


def layer_norm(x, gamma, beta, eps: float = 1e-5, residual=None, p_drop: float = 0.0):
    """LN(dropout(x) + residual) * gamma + beta  (dropout / residual optional, fused into the statistics pass)."""
    return _LayerNormFn.apply(x, gamma, beta, residual, float(eps), float(p_drop), next_seed() if p_drop > 0 else 0)


# --------------------------------------------------------------------------------------------- attention
class _AttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, cols, heads, key_bias, p_drop, seed):
        """q/k/v: bf16 [B, S, ld]; ``cols`` = first column of head 0 in each (packed QKV: same tensor three times)."""
        b, s, _ = q.shape
        packed = (q.data_ptr() == k.data_ptr() == v.data_ptr())
        q, k, v = (_as_bf16(t).contiguous() for t in (q, k, v))
        if packed:
            k = v = q
        e = ctx_e = (q.shape[-1] // 3) if packed else q.shape[-1]
        dh = e // heads
        out = torch.empty(b, s, e, dtype=_BF, device=q.device)
        lse = torch.empty(b * heads * 128, dtype=torch.float32, device=q.device)
        kb = key_bias.float().contiguous() if key_bias is not None else None
        ofs = _seed_ofs() if p_drop > 0.0 else None
        N.attn_fwd(q, k, v, q.shape[-1], k.shape[-1], v.shape[-1], cols[0], cols[1], cols[2], out, e, lse, kb, b, s, heads, dh,
                   p_drop, seed, ofs)
        ctx.cfg = (cols, heads, dh, p_drop, seed, packed, ctx_e, ofs)
        ctx.save_for_backward(q, k, v, lse, kb if kb is not None else lse)
        ctx.has_kb = kb is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, lse, kb = ctx.saved_tensors
        cols, heads, dh, p_drop, seed, packed, e, ofs = ctx.cfg
        b, s, _ = q.shape
        do = _as_bf16(dout).contiguous()
        if packed:
            dqkv = torch.empty_like(q)
            dq = dk = dv = dqkv
            dcols = cols
        else:
            dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            dcols = (0, 0, 0)
        N.attn_bwd(q, k, v, do, q.shape[-1], k.shape[-1], v.shape[-1], e, cols[0], cols[1], cols[2], 0, dq, dk, dv,
                   dq.shape[-1], dk.shape[-1], dv.shape[-1], dcols[0], dcols[1], dcols[2], lse, kb if ctx.has_kb else None,
                   b, s, heads, dh, p_drop, seed, ofs)
        if packed:
            return dqkv, None, None, None, None, None, None, None
        return dq, dk, dv, None, None, None, None, None


def attention(q, k, v, heads: int, cols=(0, 0, 0), key_bias=None, p_drop: float = 0.0):
    """softmax(Q K^T / sqrt(d) + key_bias) V per head, S <= 128; ``key_bias``: [B, S] additive."""
    return _AttentionFn.apply(q, k, v, tuple(cols), heads, key_bias, float(p_drop), next_seed() if p_drop > 0 else 0)


def attention_packed(qkv, heads: int, p_drop: float = 0.0, key_bias=None):
    """``qkv``: [B, S, 3E] = the in-projection output; heads are read in place through TMA column offsets."""
    e = qkv.shape[-1] // 3
    return attention(qkv, qkv, qkv, heads, (0, e, 2 * e), key_bias, p_drop)


# --------------------------------------------------------------------------------------------- dropout / embeddings
class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p, seed):
        x2 = _as_bf16(x).contiguous()
        y = torch.empty_like(x2)
        ofs = _seed_ofs()
        N.dropout_bf16(x2, y, x2.numel(), p, seed, ofs)
        ctx.cfg = (p, seed, ofs)
        return y

    @staticmethod
    def backward(ctx, dy):
        p, seed, ofs = ctx.cfg
        d2 = _as_bf16(dy).contiguous()
        dx = torch.empty_like(d2)
        N.dropout_bf16(d2, dx, d2.numel(), p, seed, ofs)
        return dx, None, None


def dropout(x, p: float, training: bool = True):
    if not training or p <= 0.0 or x.numel() % 2:
        return x
    return _DropoutFn.apply(x, float(p), next_seed())


class _Embed3Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, tts, word, pos, typ, pad_id):
        b, s = ids.shape
        d = word.shape[1]
        ids = ids.long().contiguous()
        tts = tts.long().contiguous() if tts is not None else None
        out = torch.empty(b, s, d, dtype=_BF, device=word.device)
        N.embed3_fwd(ids, tts, word, pos, typ, out, b * s, s, d)
        ctx.tables = (word, pos, typ)
        ctx.pad_id = pad_id
        ctx.save_for_backward(ids, tts if tts is not None else ids)
        ctx.has_tts = tts is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        ids, tts = ctx.saved_tensors
        word, pos, typ = ctx.tables
        if word.requires_grad:
            b, s = ids.shape
            g = _as_bf16(dout).contiguous()
            N.embed3_bwd(ids, tts if ctx.has_tts else None, g, _grad_buf(word), _grad_buf(pos), _grad_buf(typ), b * s, s,
                         word.shape[1], ctx.pad_id)
        return None, None, None, None, None, None


def embed3(ids, tts, word, pos, typ, pad_id: int = -1):
    """word[ids] + pos[arange(S)] + type[tts or 0] -> bf16 [B, S, D]; gradients scatter-add into the fp32 tables."""
    return _Embed3Fn.apply(ids, tts, word, pos, typ, int(pad_id))
