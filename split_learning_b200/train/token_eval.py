"""Native full-model evaluation of the token models: ViT_CIFAR10, BERT_AGNEWS and BERT_EMOTION (server-side validation on
the sm_90a kernels).

``NativeTokenEvaluator`` holds the merged model (``token_native.nativize``, ``eval()``: no dropout anywhere) and runs its
eval-mode forward as a fixed kernel sequence over static per-batch-size buffers: the wgmma GEMMs with bias / GELU / tanh /
residual epilogues, wgmma attention, LayerNorm and ``embed3`` that training uses, plus the eval-only kernels that replace
the torch glue of the module forwards: ViT patch rows and CLS + position assembly, the head LayerNorm read straight from
the CLS rows, the BERT pooler reading the CLS rows as a strided GEMM operand, and fp32 logits from the head GEMM.  Then
``eval_metrics`` adds the batch's fp64 loss, correct predictions and sample count to device totals.  Per batch size the
forward and the metrics are one CUDA graph on the evaluator's own stream; the host reads the totals once, after the last
batch.  Like the module forwards, BERT runs without an attention mask (``validation.evaluate`` calls
``model(input_ids=x)``).

Nothing for training is allocated: no optimizer, flat gradient or AdamW state.  The bf16 copies of the GEMM weights are
persistent buffers, refreshed in place on every ``load_state_dict``, so captured graphs stay valid across rounds.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
import torch.nn as nn

from ..models import bert as B
from ..models import transformer as T
from ..ops import native as N
from . import token_native

EVAL_FAMILIES = (T.ViT_CIFAR10, B.BERT_AGNEWS, B.BERT_EMOTION)
_BF = torch.bfloat16


def token_eval_supported(model_cls) -> bool:
    """Whether ``model_cls()`` has a native token eval program — decided on the meta device."""
    try:
        with torch.device("meta"):
            model = model_cls()
    except Exception:
        return False
    return type(model) in EVAL_FAMILIES and token_native.supports(model)


class _Plan:
    """Static buffers of one input shape, and the CUDA graphs captured over them."""

    def __init__(self, shape, device):
        self.shape = shape
        self.device = device
        self.graphs: Dict[bool, torch.cuda.CUDAGraph] = {}
        self.warm = set()

    def buf(self, *shape, dtype=_BF):
        return torch.empty(*shape, dtype=dtype, device=self.device)


class NativeTokenEvaluator:
    def __init__(self, model_cls, state_dict: Dict[str, torch.Tensor], device, use_graphs: bool = True):
        dev = torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device, self.use_graphs = dev, use_graphs
        N.preload(dev)
        self.stream = N.new_stream(dev)
        with torch.device(dev):
            model = model_cls()
        if type(model) not in EVAL_FAMILIES:
            raise N.NativeError(f"{type(model).__name__} has no native token eval program")
        model.requires_grad_(False)
        self.model = token_native.nativize(model).eval()
        self.vit = isinstance(model, T._ViT)
        if self.vit:
            self.blocks = [m for m in model.modules() if isinstance(m, T.EncoderBlock)]
            self.patch = model.layer1
            self.head_norm = getattr(model, f"layer{model.HEAD_NORM_LAYER}")
            self.head = getattr(model, f"layer{model.HEAD_NORM_LAYER + 1}")
            weights = [self.patch.weight] + [b.mha.in_proj_weight for b in self.blocks]
        else:
            rdn = [m for m in model.modules() if isinstance(m, B.ResidualDenseNorm)]
            attn = [m for m in model.modules() if isinstance(m, B.SelfAttention)]
            inter = [m for m in model.modules() if isinstance(m, B.Intermediate)]
            self.blocks = [(attn[i], rdn[2 * i], inter[i], rdn[2 * i + 1]) for i in range(len(attn))]
            self.embeddings = next(m for m in model.modules() if isinstance(m, B.Embeddings))
            self.pooler = next(m for m in model.modules() if isinstance(m, B.Pooler))
            self.head = next(m for m in model.modules() if isinstance(m, B.Classifier)).classifier
            weights = []
        weights += [m.weight for m in model.modules() if isinstance(m, nn.Linear)]
        # bf16 GEMM operands [out, in], one persistent buffer per weight (the pointers the graphs capture)
        self._bf = {id(w): torch.empty(w.shape[0], w.numel() // w.shape[0], dtype=_BF, device=dev) for w in weights}
        self._weights = weights
        self.plans: Dict[tuple, _Plan] = {}
        # [0] loss total (fp64), [1] correct, [2] samples (int64 views of the same words)
        self.acc = torch.zeros(4, dtype=torch.float64, device=dev)
        ints = self.acc.view(torch.int64)
        self.metrics = (self.acc[0:1], ints[1:2], ints[2:3])
        self.host = torch.zeros(4, dtype=torch.float64).pin_memory()
        self.load_state_dict(state_dict)

    # ------------------------------------------------------------------ parameters
    @torch.no_grad()
    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        """Copy a full state-dict into the model and refresh the bf16 GEMM weights in place."""
        self.stream.synchronize()
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.model.load_state_dict(sd)
            for w in self._weights:
                N.cast_f32_bf16(w, self._bf[id(w)])
        self.stream.synchronize()

    def _w(self, w: torch.Tensor) -> torch.Tensor:
        return self._bf[id(w)]

    # ------------------------------------------------------------------ programs
    def plan(self, shape) -> _Plan:
        shape = tuple(int(s) for s in shape)
        pl = self.plans.get(shape)
        if pl is None:
            pl = self.plans[shape] = self._vit_plan(shape) if self.vit else self._bert_plan(shape)
        return pl

    def _vit_plan(self, shape) -> _Plan:
        m = self.model
        if len(shape) != 4 or shape[1:] != (m.IN_CH, m.IMG, m.IMG):
            raise N.NativeError(f"{type(m).__name__} eval takes [B, {m.IN_CH}, {m.IMG}, {m.IMG}] images, got {list(shape)}")
        b, p, e = shape[0], self.patch.kernel_size[0], m.EMBED
        pl = _Plan(shape, self.device)
        pl.P = (m.IMG // p) ** 2
        pl.S = pl.P + 1
        t = b * pl.S
        pl.x_in = pl.buf(*shape, dtype=torch.float32)
        pl.labels = pl.buf(b, dtype=torch.int64)
        pl.pt = pl.buf(b * pl.P, m.IN_CH * p * p)
        pl.pe = pl.buf(b * pl.P, e)
        pl.x, pl.x2, pl.h, pl.ctx = (pl.buf(t, e) for _ in range(4))
        pl.qkv = pl.buf(t, 3 * e)
        pl.mid = pl.buf(t, self.blocks[0].mlp[0].out_features)
        pl.mean, pl.rstd = pl.buf(t, dtype=torch.float32), pl.buf(t, dtype=torch.float32)
        pl.lse = pl.buf(b * self.blocks[0].mha.num_heads * 128, dtype=torch.float32)
        pl.hn = pl.buf(b, e)
        pl.logits = pl.buf(b, self.head.out_features, dtype=torch.float32)
        return pl

    def _bert_plan(self, shape) -> _Plan:
        if len(shape) != 2:
            raise N.NativeError(f"BERT eval takes [B, S] token ids, got {list(shape)}")
        b, s = shape
        hid = self.embeddings.word_embeddings.weight.shape[1]
        pl = _Plan(shape, self.device)
        pl.S = s
        t = b * s
        pl.x_in = pl.buf(b, s, dtype=torch.int64)
        pl.labels = pl.buf(b, dtype=torch.int64)
        pl.x, pl.q, pl.k, pl.v, pl.ctx, pl.d, pl.a, pl.pre = (pl.buf(t, hid) for _ in range(8))
        pl.mid = pl.buf(t, self.blocks[0][2].dense.out_features)
        pl.mean, pl.rstd = pl.buf(t, dtype=torch.float32), pl.buf(t, dtype=torch.float32)
        pl.lse = pl.buf(b * self.blocks[0][0].heads * 128, dtype=torch.float32)
        pl.pooled = pl.buf(b, hid)
        pl.logits = pl.buf(b, self.head.out_features, dtype=torch.float32)
        return pl

    def _lin(self, x, mod, out, rows, act=None, residual=None):
        n_out, k_in = self._w(mod.weight).shape
        N.gemm_act(x, self._w(mod.weight), out, rows, n_out, k_in, bias=mod.bias, act=act, residual=residual)

    def _vit_forward(self, pl: _Plan) -> None:
        m, b = self.model, pl.shape[0]
        e, p = m.EMBED, self.patch.kernel_size[0]
        t = b * pl.S
        N.patch_rows(pl.x_in, pl.pt, p)
        wp = self._w(self.patch.weight)
        N.gemm_act(pl.pt, wp, pl.pe, b * pl.P, e, wp.shape[1], bias=self.patch.bias)
        N.vit_tokens(pl.pe, m.cls_token, m.pos_embed, pl.x, b, pl.P, e)
        for blk in self.blocks:
            mha = blk.mha
            N.ln_fwd(pl.x, None, blk.ln1.weight, blk.ln1.bias, pl.h, None, pl.mean, pl.rstd, t, e, blk.ln1.eps)
            N.gemm_act(pl.h, self._w(mha.in_proj_weight), pl.qkv, t, 3 * e, e, bias=mha.in_proj_bias)
            N.attn_fwd(pl.qkv, pl.qkv, pl.qkv, 3 * e, 3 * e, 3 * e, 0, e, 2 * e, pl.ctx, e, pl.lse, None, b, pl.S,
                       mha.num_heads, e // mha.num_heads)
            self._lin(pl.ctx, mha.out_proj, pl.x2, t, residual=pl.x)
            N.ln_fwd(pl.x2, None, blk.ln2.weight, blk.ln2.bias, pl.h, None, pl.mean, pl.rstd, t, e, blk.ln2.eps)
            self._lin(pl.h, blk.mlp[0], pl.mid, t, act="gelu")
            self._lin(pl.mid, blk.mlp[2], pl.x, t, residual=pl.x2)
        hn = self.head_norm
        N.ln_rows_fwd(pl.x, pl.S * e, hn.weight, hn.bias, pl.hn, b, e, hn.eps)      # x[:, 0] -> LayerNorm
        N.gemm_bias_f32(pl.hn, self._w(self.head.weight), pl.logits, self.head.bias, b, self.head.out_features, e)

    def _bert_forward(self, pl: _Plan) -> None:
        b, s = pl.shape
        t = b * s
        emb = self.embeddings
        hid = emb.word_embeddings.weight.shape[1]
        N.embed3_fwd(pl.x_in, None, emb.word_embeddings.weight, emb.position_embeddings.weight,
                     emb.token_type_embeddings.weight, pl.d, t, s, hid)
        ln = emb.LayerNorm
        N.ln_fwd(pl.d, None, ln.weight, ln.bias, pl.x, None, pl.mean, pl.rstd, t, hid, ln.eps)
        for sa, ao, it, oo in self.blocks:
            self._lin(pl.x, sa.query, pl.q, t)
            self._lin(pl.x, sa.key, pl.k, t)
            self._lin(pl.x, sa.value, pl.v, t)
            N.attn_fwd(pl.q, pl.k, pl.v, hid, hid, hid, 0, 0, 0, pl.ctx, hid, pl.lse, None, b, s, sa.heads, hid // sa.heads)
            self._lin(pl.ctx, ao.dense, pl.d, t)
            n = ao.LayerNorm
            N.ln_fwd(pl.d, pl.x, n.weight, n.bias, pl.a, pl.pre, pl.mean, pl.rstd, t, hid, n.eps)
            self._lin(pl.a, it.dense, pl.mid, t, act="gelu")
            self._lin(pl.mid, oo.dense, pl.d, t)
            n = oo.LayerNorm
            N.ln_fwd(pl.d, pl.a, n.weight, n.bias, pl.x, pl.pre, pl.mean, pl.rstd, t, hid, n.eps)
        # pooler: tanh(x[:, 0] W^T + b) with the CLS rows read in place (row pitch S * hidden)
        dense = self.pooler.dense
        N.gemm_act(pl.x, self._w(dense.weight), pl.pooled, b, hid, hid, lda=s * hid, bias=dense.bias, act="tanh")
        N.gemm_bias_f32(pl.pooled, self._w(self.head.weight), pl.logits, self.head.bias, b, self.head.out_features, hid)

    def _run(self, pl: _Plan, with_metrics: bool) -> None:
        def body():
            (self._vit_forward if self.vit else self._bert_forward)(pl)
            if with_metrics:
                N.eval_metrics(pl.logits, pl.labels, *self.metrics)
        if not self.use_graphs:
            body()
            return
        g = pl.graphs.get(with_metrics)
        if g is not None:
            g.replay()
            return
        if with_metrics not in pl.warm:
            body()                                     # first call of this program: eager (loads kernels, sets attributes)
            pl.warm.add(with_metrics)
            return
        from ..utils.timing import capture_graph
        g = pl.graphs[with_metrics] = capture_graph(torch.cuda.current_stream(), body)
        g.replay()

    # ------------------------------------------------------------------ public
    @torch.no_grad()
    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """Eval-mode fp32 logits of one batch (the kernel sequence ``evaluate`` runs)."""
        pl = self.plan(x.shape)
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            pl.x_in.copy_(x, non_blocking=True)
            self._run(pl, False)
            out = pl.logits.clone()
        self.stream.synchronize()
        return out

    @torch.no_grad()
    def evaluate(self, source, pump: Optional[Callable[[], None]] = None) -> Dict[str, float]:
        """Same result dict as ``validation.evaluate``: loss = mean of the per-batch mean losses, accuracy in percent.
        ``source`` yields (x, labels) — images [B, C, H, W] or token ids [B, S] — or dicts with input_ids / labels."""
        batches = 0
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            N.zero_(self.acc)
            for i, batch in enumerate(source):
                x, y = (batch["input_ids"], batch["labels"]) if isinstance(batch, dict) else batch
                pl = self.plan(x.shape)
                pl.x_in.copy_(x, non_blocking=True)
                pl.labels.copy_(torch.as_tensor(y), non_blocking=True)
                self._run(pl, True)
                batches += 1
                if pump is not None and i % 5 == 4:
                    pump()
            self.host.copy_(self.acc, non_blocking=True)
        self.stream.synchronize()
        ints = self.host.view(torch.int64)
        loss, correct, total = float(self.host[0]), int(ints[1]), int(ints[2])
        return {"val_loss": loss / max(batches, 1), "val_acc": 100.0 * correct / max(total, 1),
                "val_correct": correct, "val_total": total}
