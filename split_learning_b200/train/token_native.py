"""Native execution of the token-model families (KWT / ViT / BERT_AGNEWS / BERT_EMOTION, with or without LoRA).

``nativize(model)`` re-binds the ``forward`` of every block of a stage to the fused sm_90a ops of ``ops.nn``
(wgmma GEMMs with bias / GELU / tanh / residual epilogues, wgmma attention, LayerNorm with fused
dropout+residual, hash dropout, embedding gather) while leaving the module tree — and therefore parameter names,
state-dicts, checkpoints, LoRA wrapping / merging and FedAvg — untouched.  The reference runs these layers through
stock ``torch.nn`` (src/model/BERT_AGNEWS.py:56-165, src/model/KWT_SPEECHCOMMANDS.py:5-109,
other/Vanilla_SL/src/model/ViT_CIFAR10.py:27-116, other/Vanilla_SL/src/model/BERT_EMOTION.py:183-428).

Activations between native ops are bf16; the stage boundary is fp32 (the wire format of the cut).  There is no
silent fallback: a shape the kernels do not cover raises.
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn

from ..models import bert as B
from ..models import transformer as T
from ..models.lora import LoRALinear
from ..ops import nn as F

TOKEN_FAMILIES = ("BERT", "KWT", "VIT")


def supports(model: nn.Module) -> bool:
    return isinstance(model, (T._TokenModel, B.BERT_AGNEWS, B.BERT_EMOTION))


# ------------------------------------------------------------------------------------------------ leaf helpers
def _lin(mod, x, act=None, residual=None):
    """nn.Linear or LoRALinear through the native GEMM (LoRA: frozen base + two skinny GEMMs)."""
    if isinstance(mod, LoRALinear):
        base = F.linear(x, mod.base.weight, mod.base.bias, None, residual)
        h = F.dropout(x, mod.drop.p, mod.training)
        low = F.linear(F.linear(h, mod.lora_A), mod.lora_B)
        out = base + low * mod.scaling
        if act == "gelu":
            return torch.nn.functional.gelu(out)
        if act == "tanh":
            return torch.tanh(out)
        return out
    return F.linear(x, mod.weight, mod.bias, act, residual)


def _ln(mod: nn.LayerNorm, x, residual=None, p_drop=0.0):
    return F.layer_norm(x, mod.weight, mod.bias, mod.eps, residual, p_drop)


# ------------------------------------------------------------------------------------------------ forwards
def _linear_forward(self, x):
    return _lin(self, x)


def _layernorm_forward(self, x):
    return _ln(self, x)


def _dropout_forward(self, x):
    if not x.is_cuda or x.numel() % 2:
        return nn.functional.dropout(x, self.p, self.training)
    return F.dropout(x, self.p, self.training)


def _encoder_block_forward(self, x):
    """Pre-LN block of KWT / ViT: x + MHA(LN(x)); x + MLP(LN(x))  (models/transformer.py:EncoderBlock)."""
    mha = self.mha
    h = _ln(self.ln1, x)
    qkv = F.linear(h, mha.in_proj_weight, mha.in_proj_bias)
    ctx = F.attention_packed(qkv, mha.num_heads, mha.dropout if self.training else 0.0)
    x = F.linear(ctx, mha.out_proj.weight, mha.out_proj.bias, None, x)
    m = _lin(self.mlp[0], _ln(self.ln2, x), act="gelu")
    return _lin(self.mlp[2], m, residual=x)


def _self_attention_forward(self, x, attention_mask=None):
    q, k, v = _lin(self.query, x), _lin(self.key, x), _lin(self.value, x)
    bias = None
    if attention_mask is not None:
        bias = (1.0 - attention_mask.to(torch.float32)) * -10000.0
    return F.attention(q, k, v, self.heads, (0, 0, 0), bias, self.dropout.p if self.training else 0.0)


def _residual_dense_norm_forward(self, h, residual):
    return _ln(self.LayerNorm, _lin(self.dense, h), residual, self.dropout.p if self.training else 0.0)


def _intermediate_forward(self, x):
    return _lin(self.dense, x, act="gelu")


def _pooler_forward(self, x):
    return _lin(self.dense, x[:, 0].contiguous(), act="tanh")


def _embeddings_forward(self, input_ids, token_type_ids=None):
    e = F.embed3(input_ids, token_type_ids, self.word_embeddings.weight, self.position_embeddings.weight,
                 self.token_type_embeddings.weight, self.word_embeddings.padding_idx if self.word_embeddings.padding_idx
                 is not None else -1)
    return F.dropout(_ln(self.LayerNorm, e), self.dropout.p, self.training)


def _patch_conv_forward(self, x):
    """ViT patch embedding: Conv2d(kernel == stride) == one GEMM over unfolded patches
    (other/Vanilla_SL/src/model/ViT_CIFAR10.py:41)."""
    p = self.kernel_size[0]
    b, c, hh, ww = x.shape
    gh, gw = hh // p, ww // p
    patches = x.reshape(b, c, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(b, gh * gw, c * p * p)
    y = F.linear(patches, self.weight, self.bias)
    return y.view(b, gh, gw, self.out_channels).permute(0, 3, 1, 2)


_FORWARDS = {
    T.EncoderBlock: _encoder_block_forward,
    B.SelfAttention: _self_attention_forward,
    B.ResidualDenseNorm: _residual_dense_norm_forward,
    B.Intermediate: _intermediate_forward,
    B.Pooler: _pooler_forward,
    B.Embeddings: _embeddings_forward,
    nn.LayerNorm: _layernorm_forward,
    nn.Dropout: _dropout_forward,
    nn.Linear: _linear_forward,
    LoRALinear: _linear_forward,
}


def nativize(model: nn.Module) -> nn.Module:
    """Bind the native forwards (idempotent).  Call after LoRA wrapping; ``merge_lora`` keeps working because only
    ``forward`` attributes are touched."""
    for mod in model.modules():
        fn = _FORWARDS.get(type(mod))
        if fn is None and isinstance(mod, nn.Conv2d) and mod.kernel_size == mod.stride and mod.padding == (0, 0):
            if (mod.in_channels * mod.kernel_size[0] * mod.kernel_size[1]) % 8 == 0:
                fn = _patch_conv_forward
        if fn is not None:
            mod.forward = types.MethodType(fn, mod)
    model._slb_native = True
    return model


def denativize(model: nn.Module) -> nn.Module:
    for mod in model.modules():
        if "forward" in mod.__dict__:
            del mod.__dict__["forward"]
    model._slb_native = False
    return model
