"""Native execution of the conv / BN / ReLU tables that the compiled VGG plan (``b200_executor``) does not cover —
MobileNetv1_CIFAR10 / MobileNetv1_MNIST of the Vanilla_SL variant (other/Vanilla_SL/src/model/MobileNetv1_CIFAR10.py:5-185:
dense 3x3 convs with stride 1 or 2, 1x1 convs, 32-channel layers, one max-pool, one Linear).

Same scheme as ``token_native``: the module tree (parameter names, state-dict, checkpoints) is untouched, the stage's
``forward`` is re-bound to a small NHWC/bf16 program whose heavy ops are ``torch.autograd.Function``s over the
hand-written sm_90a kernels:

* 3x3 conv  -> the wgmma implicit-GEMM kernel (forward, dgrad with mirrored taps, split-K wgrad).  Channel counts
  that are not multiples of 64 are zero-padded in the bf16 weight view; stride 2 is computed at stride 1 and
  sub-sampled (4 of the 27 convs), its backward scatters into a zero tensor;
* 1x1 conv  -> the wgmma GEMM of ``ops.nn.linear`` on the NHWC view (no im2col, no layout change);
* first conv (Cin = 1 or 3, NCHW fp32 input) -> ``conv3x3_small_fwd_kernel`` / ``conv3x3_small_wgrad_kernel``;
* BatchNorm(train) + ReLU (+ MaxPool2) -> ``col_stats`` + ``bn_relu_pool_fwd`` / ``bn_relu_pool_bwd`` (running
  statistics and ``num_batches_tracked`` updated by the kernel);
* Linear -> ``ops.nn.linear``.
Stage boundaries stay NCHW fp32 (the reference's wire format).  ``TorchExecutor(native=True)`` captures whole steps of
this program into CUDA graphs exactly as for the token models.
"""
from __future__ import annotations

import types
from typing import List, Tuple

import torch
import torch.nn as nn

from ..models import mobilenet as M
from ..ops import native as N
from ..ops import nn as F

_BF = torch.bfloat16


def supports(model: nn.Module) -> bool:
    return isinstance(model, (M.MobileNetv1_CIFAR10, M.MobileNetv1_MNIST))


def _c64(c: int) -> int:
    return (c + 63) // 64 * 64


def _pad_last(t: torch.Tensor, c: int) -> torch.Tensor:
    if t.shape[-1] == c:
        return t.contiguous()
    out = torch.zeros(*t.shape[:-1], c, dtype=t.dtype, device=t.device)
    out[..., :t.shape[-1]] = t
    return out


# ------------------------------------------------------------------------------------------------ conv 3x3
class _Conv3x3Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride):
        """x: [B, H, W, Cin] bf16 (NHWC); weight: the nn.Conv2d parameter [Cout, Cin, 3, 3] fp32."""
        cout, cin = weight.shape[0], weight.shape[1]
        cin_p, cout_p = _c64(cin), _c64(cout)
        b, h, w, _ = x.shape
        wp = torch.zeros(cout_p, 3, 3, cin_p, dtype=_BF, device=x.device) if (cin_p != cin or cout_p != cout) else None
        w_ohwi = weight.detach().permute(0, 2, 3, 1)
        if wp is None:
            wp = w_ohwi.to(_BF).contiguous()
        else:
            wp[:cout, :, :, :cin] = w_ohwi
        xp = _pad_last(x if x.dtype == _BF else x.to(_BF), cin_p)
        bp = None
        if bias is not None:
            bp = _pad_last(bias.detach().float(), cout_p)
        y = torch.empty(b, h, w, cout_p, dtype=_BF, device=x.device)
        N.conv3x3_fwd(xp, wp, y, bp)
        out = y if cout_p == cout else y[..., :cout]
        if stride == 2:
            out = out[:, ::2, ::2, :]
        ctx.weight, ctx.bias, ctx.stride = weight, bias, stride
        ctx.save_for_backward(xp, wp)
        return out.contiguous()

    @staticmethod
    def backward(ctx, dout):
        xp, wp = ctx.saved_tensors
        weight, bias, stride = ctx.weight, ctx.bias, ctx.stride
        cout, cin = weight.shape[0], weight.shape[1]
        cout_p, cin_p = wp.shape[0], wp.shape[3]
        b, h, w, _ = xp.shape
        d = dout if dout.dtype == _BF else dout.to(_BF)
        if stride == 2 or cout_p != cout:
            dy = torch.zeros(b, h, w, cout_p, dtype=_BF, device=d.device)
            if stride == 2:
                dy[:, ::2, ::2, :cout] = d
            else:
                dy[..., :cout] = d
        else:
            dy = d.contiguous()
        if weight.requires_grad:
            dw = torch.zeros(cout_p, 3, 3, cin_p, dtype=torch.float32, device=d.device)
            N.conv3x3_wgrad(xp, dy, dw)
            F._grad_buf(weight).add_(dw[:cout, :, :, :cin].permute(0, 3, 1, 2))
        if bias is not None and bias.requires_grad:
            db = torch.zeros(cout_p, dtype=torch.float32, device=d.device)
            N.colsum_bf16(dy, db, b * h * w, cout_p, cout_p)
            F._grad_buf(bias).add_(db[:cout])
        dx = None
        if ctx.needs_input_grad[0]:
            dxp = torch.empty(b, h, w, cin_p, dtype=_BF, device=d.device)
            N.conv3x3_dgrad(dy, wp, dxp)
            dx = dxp if cin_p == cin else dxp[..., :cin].contiguous()
        return dx, None, None, None


class _ConvStemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        """x: [B, Cin, H, W] fp32 (the stage input, Cin = 1 or 3) -> [B, H, W, Cout] bf16."""
        cout = weight.shape[0]
        b, _, h, w = x.shape
        x = x.float().contiguous()
        w_ohwi = weight.detach().permute(0, 2, 3, 1).contiguous()
        y = torch.empty(b, h, w, cout, dtype=_BF, device=x.device)
        N.conv3x3_small_fwd(x, w_ohwi, bias.detach() if bias is not None else None, y)
        ctx.weight, ctx.bias = weight, bias
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dout):
        x, = ctx.saved_tensors
        weight, bias = ctx.weight, ctx.bias
        cout, cin = weight.shape[0], weight.shape[1]
        d = (dout if dout.dtype == _BF else dout.to(_BF)).contiguous()
        if weight.requires_grad:
            dw = torch.zeros(cout, 3, 3, cin, dtype=torch.float32, device=d.device)
            N.conv3x3_small_wgrad(x, d, dw)
            F._grad_buf(weight).add_(dw.permute(0, 3, 1, 2))
        if bias is not None and bias.requires_grad:
            N.colsum_bf16(d, F._grad_buf(bias), d.numel() // cout, cout, cout)
        return None, None, None


# ------------------------------------------------------------------------------------------------ BN (+ReLU (+pool))
class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, bn, relu, pool):
        """y: [B, H, W, C] bf16 conv output; ``bn``: the nn.BatchNorm2d module (training mode: batch statistics)."""
        b, h, w, c = y.shape
        y = (y if y.dtype == _BF else y.to(_BF)).contiguous()
        stats = torch.zeros(2 * c, dtype=torch.float32, device=y.device)
        N.col_stats(y.view(-1, c), stats[:c], stats[c:])
        save = torch.empty(2 * c, dtype=torch.float32, device=y.device)
        out = torch.empty(b, h // 2 if pool else h, w // 2 if pool else w, c, dtype=_BF, device=y.device)
        N.bn_relu_pool_fwd(y, stats[:c], stats[c:], bn.weight, bn.bias, bn.running_mean, bn.running_var,
                           bn.num_batches_tracked, save[:c], save[c:], out, h, w, relu, pool,
                           momentum=bn.momentum if bn.momentum is not None else 0.1, eps=bn.eps,
                           update_running=bool(bn.track_running_stats))
        ctx.bn, ctx.cfg = bn, (relu, pool, h, w, c)
        ctx.save_for_backward(y, save)
        return out

    @staticmethod
    def backward(ctx, dout):
        y, save = ctx.saved_tensors
        bn = ctx.bn
        relu, pool, h, w, c = ctx.cfg
        d = (dout if dout.dtype == _BF else dout.to(_BF)).contiguous()
        tmp = torch.zeros(2 * c, dtype=torch.float32, device=d.device)      # the apply pass reads the totals: own buffer
        dy = torch.empty_like(y)
        N.bn_relu_pool_bwd(d, y, bn.weight, bn.bias, save[:c], save[c:], tmp[:c], tmp[c:], dy, h, w, relu, pool)
        if bn.weight.requires_grad:
            F._grad_buf(bn.weight).add_(tmp[:c])
            F._grad_buf(bn.bias).add_(tmp[c:])
        return dy, None, None, None


# ------------------------------------------------------------------------------------------------ stage program
def _program(model) -> List[Tuple]:
    """Group the owned layer indices into fused ops: ('stem'|'conv3'|'conv1', i) ('bn', i, relu, pool)
    ('relu',) ('pool',) ('flatten',) ('linear', i)."""
    idx = list(model.owned_indices())
    kinds = {i: model.LAYERS[i - 1].kind for i in idx}
    ops, k = [], 0
    while k < len(idx):
        i = idx[k]
        kind = kinds[i]
        if kind == "conv":
            mod = getattr(model, f"layer{i}")
            if mod.kernel_size == (1, 1):
                ops.append(("conv1", i))
            elif mod.in_channels <= 3:
                ops.append(("stem", i))
            else:
                ops.append(("conv3", i))
            k += 1
        elif kind == "bn2d":
            relu = k + 1 < len(idx) and kinds[idx[k + 1]] == "relu"
            pool = relu and k + 2 < len(idx) and kinds[idx[k + 2]] == "maxpool2"
            ops.append(("bn", i, relu, pool))
            k += 1 + int(relu) + int(pool)
        elif kind in ("relu", "maxpool2", "flatten"):
            ops.append(({"relu": "relu", "maxpool2": "pool", "flatten": "flatten"}[kind],))
            k += 1
        elif kind == "linear":
            ops.append(("linear", i))
            k += 1
        else:
            raise N.NativeError(f"no native op for layer kind {kind!r}")
    return ops


def _forward(self, x, **_):
    ops = self._slb_program
    nhwc = False                                   # stage input is NCHW fp32 (or [B, F] after a flatten)
    for op in ops:
        name = op[0]
        if name in ("conv3", "conv1", "bn", "relu", "pool") and not nhwc and x.dim() == 4:
            x = x.permute(0, 2, 3, 1).contiguous().to(_BF)
            nhwc = True
        if name == "stem":
            mod = getattr(self, f"layer{op[1]}")
            x = _ConvStemFn.apply(x, mod.weight, mod.bias)
            nhwc = True
        elif name == "conv3":
            mod = getattr(self, f"layer{op[1]}")
            x = _Conv3x3Fn.apply(x, mod.weight, mod.bias, mod.stride[0])
        elif name == "conv1":
            mod = getattr(self, f"layer{op[1]}")
            if mod.stride[0] != 1:
                x = x[:, ::mod.stride[0], ::mod.stride[0], :].contiguous()
            x = F.linear(x, mod.weight, mod.bias)
        elif name == "bn":
            mod = getattr(self, f"layer{op[1]}")
            if mod.training:
                x = _BnActFn.apply(x, mod, op[2], op[3])
            else:                                  # eval: running statistics, plain torch on the NHWC view
                y = nn.functional.batch_norm(x.float(), mod.running_mean, mod.running_var, mod.weight, mod.bias, False, 0.0,
                                             mod.eps)
                y = torch.relu(y) if op[2] else y
                if op[3]:
                    y = nn.functional.max_pool2d(y.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
                x = y.to(_BF)
        elif name == "relu":
            x = torch.relu(x)
        elif name == "pool":
            x = nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous()
        elif name == "flatten":
            if nhwc:
                x = x.permute(0, 3, 1, 2)
                nhwc = False
            x = x.reshape(x.shape[0], -1)
        elif name == "linear":
            mod = getattr(self, f"layer{op[1]}")
            x = F.linear(x, mod.weight, mod.bias)
    if nhwc:
        x = x.permute(0, 3, 1, 2)
    return x


def nativize(model: nn.Module) -> nn.Module:
    model._slb_program = _program(model)
    model.forward = types.MethodType(_forward, model)
    model._slb_native = True
    return model
