"""Native sm_90a stage executor for VGG-family layer tables.

A stage's ``LayerSpec`` slice is compiled into a static plan of fused blocks

    ConvBlock   = [conv3x3] [BatchNorm2d(train)] [ReLU] [MaxPool2]     (wgmma implicit GEMM
                  + fused BN-stat epilogue; BN/ReLU/pool apply kernel writes the block output —
                  for the last block of a non-last stage that output pointer *is* the next
                  stage's mailbox slot, local or NVLink-peer, and the kernel publishes the flag)
    Dropout     = standalone dropout on a dense activation (VGG layer 46)
    LinearBlock = Linear [ReLU] [Dropout]   (swap-AB wgmma GEMM, split-K, fused finalisation)

over flat fp32 master / gradient / momentum buffers.  Forward, backward(+recompute) and the
optimizer step of one microbatch are captured once per batch size into CUDA graphs; the host
only copies the input in and replays.

The same block sequence also runs in eval mode (``eval_forward``, ``train/b200_eval.py``): conv without BN statistics,
BatchNorm on the running statistics, dropout skipped, always the fp32 (tf32) flavour, forward buffers only, one CUDA
graph per batch size.  ``eval_only=True`` builds an executor for that alone (no gradient, momentum, bf16 shadow or
exportable memory).

Two compute precisions (``precision=`` / ``b200.precision`` / ``SLB200_PRECISION``):

* ``tf32`` (default, the reference's precision): fp32 activations and weights end to end,
  convolutions on ``wgmma`` tf32 with fp32 accumulation (what PyTorch/cuDNN does by
  default for the reference's ``nn.Conv2d``), Linear layers in IEEE fp32 on the CUDA cores (the
  reference's ``nn.Linear`` is an fp32 cuBLAS GEMM) with the SGD-momentum step fused into the
  weight-gradient pass; BN / ReLU / pool / CE / SGD in fp32.  No reduced-precision copy of
  anything exists in this mode.
* ``bf16`` (opt-in fast mode): bf16 activations and a bf16 weight shadow refreshed by the fused
  SGD kernel, bf16 wgmma GEMMs for convolutions and Linear layers.

Semantics follow the reference trainer (src/train/VGG16.py:61-190): SGD(lr, momentum) step per
microbatch, recompute-forward with *current* weights on non-last stages (BN running stats
advance twice, as in the reference), CE mean loss on the last stage, NaN flag kept on device.
Conv weights are stored [Cout][3][3][Cin]; ``state_dict()`` converts to torch's layout so
checkpoints stay loadable by the reference model classes.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import torch

from ..models import SplitModel
from ..ops import native as N
from .executor import StageExecutor


# ----------------------------------------------------------------------------- plan
@dataclass
class ConvBlock:
    conv: Optional[int] = None       # layer indices (1-based) or None
    bn: Optional[int] = None
    relu: bool = False
    pool: bool = False
    cin: int = 0
    cout: int = 0
    H: int = 0
    W: int = 0


@dataclass
class DropoutOp:
    idx: int
    p: float
    n: int = 0


@dataclass
class LinearBlock:
    lin: int
    fin: int
    fout: int
    relu: bool = False
    drop: float = 0.0


def _input_shape(model: SplitModel) -> Tuple[str, Tuple[int, ...]]:
    """Shape of the stage input (without batch): ('image', (C,H,W)) or ('flat', (F,))."""
    x = model.example_input(1)
    c, h, w = x.shape[1:]
    kind = "image"
    for i in range(1, model.start_layer + 1):
        s = model.LAYERS[i - 1]
        if s.kind == "conv3x3":
            c = s.args[1]
        elif s.kind == "maxpool2":
            h, w = h // 2, w // 2
        elif s.kind == "flatten":
            kind, c = "flat", c * h * w
        elif s.kind == "linear":
            c = s.args[1]
    return (kind, (c, h, w)) if kind == "image" else (kind, (c,))


def supports(model: SplitModel) -> bool:
    ok_kinds = {"conv3x3", "bn2d", "relu", "maxpool2", "flatten", "dropout", "linear"}
    if not all(s.kind in ok_kinds for _, s in model.owned_specs()):
        return False
    try:
        compile_plan(model)
        return True
    except (ValueError, NotImplementedError):
        return False


def compile_plan(model: SplitModel):
    kind, shp = _input_shape(model)
    specs = model.owned_specs()
    blocks: List[Any] = []
    if kind == "image":
        c, h, w = shp
    else:
        c, h, w = shp[0], 1, 1
    flat = kind == "flat"
    i = 0
    while i < len(specs):
        idx, s = specs[i]
        if s.kind in ("conv3x3", "bn2d", "relu", "maxpool2") and not flat:
            b = ConvBlock(H=h, W=w, cin=c)
            if s.kind == "conv3x3":
                if s.args[0] != c:
                    raise ValueError("channel mismatch")
                b.conv, c = idx, s.args[1]
                i += 1
            if i < len(specs) and specs[i][1].kind == "bn2d":
                b.bn = specs[i][0]
                i += 1
            if i < len(specs) and specs[i][1].kind == "relu":
                b.relu = True
                i += 1
            if i < len(specs) and specs[i][1].kind == "maxpool2":
                b.pool = True
                h, w = h // 2, w // 2
                i += 1
            b.cout = c
            if b.conv is not None and b.cin > 4 and (b.cin % 64 or b.cout % 64):
                raise NotImplementedError("wgmma conv path needs channels % 64 == 0")
            if b.conv is not None and b.bn is None and (b.relu or b.pool):
                raise NotImplementedError("conv+ReLU/pool without BatchNorm has no native plan yet")
            if b.conv is not None and b.bn is None and b.cin <= 4:
                raise NotImplementedError("first-layer conv must be followed by BatchNorm in the same stage")
            if b.W > 128 or (128 % b.W):
                raise NotImplementedError("image width must divide 128")
            blocks.append(b)
        elif s.kind == "flatten":
            if not flat and (h, w) != (1, 1):
                raise NotImplementedError("flatten of a spatial map > 1x1 (NHWC/NCHW order differs)")
            flat, c = True, c * h * w
            i += 1
        elif s.kind == "dropout" and flat:
            blocks.append(DropoutOp(idx, float(s.args[0]), c))
            i += 1
        elif s.kind == "linear" and flat:
            b = LinearBlock(idx, s.args[0], s.args[1])
            if s.args[0] != c:
                raise ValueError("feature mismatch")
            c = s.args[1]
            i += 1
            if i < len(specs) and specs[i][1].kind == "relu":
                b.relu = True
                i += 1
            if i < len(specs) and specs[i][1].kind == "dropout":
                b.drop = float(specs[i][1].args[0])
                i += 1
            if b.fin % 64:
                raise NotImplementedError("Linear in_features % 64")
            blocks.append(b)
        else:
            raise NotImplementedError(f"layer {idx}: {s.kind} in this position")
    out_shape = ("flat", (c,)) if flat else ("image", (c, h, w))
    return (kind, shp), blocks, out_shape


def _align(n: int, a: int = 128) -> int:
    return (n + a - 1) // a * a


def flat_layouts(model_cls, start_layer: int, end_layer: int):
    """Flat-buffer layouts of the stage ``model_cls(start, end)`` — exactly what ``B200Executor`` allocates — computed
    from the layer table alone (meta device, nothing is allocated): {"P": {key: (offset, numel)}, "S": ..., "I": ...}
    with 128-float aligned entries (4 floats per entry in "I").  Every replica derives every other replica's layout
    from (model, layers), which is how the FedAvg all-reduce finds the same layer inside stages cut at different points."""
    with torch.device("meta"):
        model = model_cls(start_layer, end_layer)
    _, blocks, _ = compile_plan(model)
    P: Dict[str, Tuple[int, int]] = {}
    S: Dict[str, Tuple[int, int]] = {}
    I: Dict[str, Tuple[int, int]] = {}
    off = so = io = 0
    for b in blocks:
        if isinstance(b, ConvBlock):
            if b.conv is not None:
                P[f"layer{b.conv}.weight"] = (off, _align(b.cout * 9 * b.cin)); off += _align(b.cout * 9 * b.cin)
                P[f"layer{b.conv}.bias"] = (off, _align(b.cout)); off += _align(b.cout)
            if b.bn is not None:
                P[f"layer{b.bn}.weight"] = (off, _align(b.cout)); off += _align(b.cout)
                P[f"layer{b.bn}.bias"] = (off, _align(b.cout)); off += _align(b.cout)
                S[f"layer{b.bn}.running_mean"] = (so, _align(b.cout)); so += _align(b.cout)
                S[f"layer{b.bn}.running_var"] = (so, _align(b.cout)); so += _align(b.cout)
                I[f"layer{b.bn}.num_batches_tracked"] = (io, 4); io += 4
        elif isinstance(b, LinearBlock):
            P[f"layer{b.lin}.weight"] = (off, _align(b.fout * b.fin)); off += _align(b.fout * b.fin)
            P[f"layer{b.lin}.bias"] = (off, _align(b.fout)); off += _align(b.fout)
    return {"P": P, "S": S, "I": I}


# ----------------------------------------------------------------------------- executor
class B200Executor(StageExecutor):
    def __init__(self, model: SplitModel, model_name: str, learning: dict, device, is_first=False, is_last=False,
                 recompute: bool = True, use_graphs: bool = True, seed: int = 1234, fused_cut: bool = True,
                 precision: Optional[str] = None, eval_only: bool = False, state_dict: Optional[Dict[str, torch.Tensor]] = None):
        N.require()
        import os
        self.eval_only = eval_only
        if eval_only:
            precision = "tf32"
        precision = (precision or learning.get("precision") or os.environ.get("SLB200_PRECISION") or "tf32").lower()
        if precision in ("fp32", "float32"):
            precision = "tf32"
        if precision not in ("tf32", "bf16"):
            raise ValueError(f"precision must be tf32 or bf16, got {precision!r}")
        self.precision = precision
        self.fp32 = precision == "tf32"
        self.act_dtype = torch.float32 if self.fp32 else torch.bfloat16
        self.ke = 32 if self.fp32 else 64                 # K elements per 128-byte MMA pipeline stage
        self.clip = float(learning.get("clip-grad-norm") or 0.0)
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        N.preload(self.device)
        self.model_cls = type(model)
        self._sd_keys = list(model.state_dict().keys())          # checkpoint key order of this stage (reference layout)
        self.start_layer, self.end_layer = model.start_layer, model.end_layer
        self.model_name = model_name
        self.is_first, self.is_last = is_first, is_last
        self.recompute = recompute
        self.use_graphs = use_graphs
        self.fused_cut = fused_cut and os.environ.get("SLB200_FUSED_CUT", "1") != "0"
        # single-launch BN backward (reduce -> grid barrier -> apply): measured SLOWER than two PDL-chained launches
        # (L pass 825 us vs 776 us) — a software grid barrier costs more than a kernel boundary here.  Off by default.
        self.fused_bn_bwd = os.environ.get("SLB200_FUSED_BN_BWD", "0") != "0"
        # BatchNorm-backward reduction of block k-1 folded into the dgrad epilogue of block k (one launch less per pair).
        # SLB200_FUSED_BNSTATS: 0 off (default), 1 upstream blocks without max-pool, 2 all.  Measured on one box (N = 1,
        # 400 steps): 36.47 k / 36.27 k / 35.83 k images/s — once the extra epilogue lives in its own kernel instantiation
        # (it cost every conv 1.8 % when it shared one), the 8 saved launches do not pay for the y / parameter loads the
        # fused epilogue adds to the dgrad's critical path.  Kept (tested in ops/selftest.py) as an option.
        self.fused_bn_stats = 0 if self.fused_bn_bwd else int(os.environ.get("SLB200_FUSED_BNSTATS", "0"))
        self.lr = float(learning.get("learning-rate", 0.01))
        self.mu = float(learning.get("momentum", 0.0))
        self.seed = seed
        (self.in_kind, self.in_shape), self.blocks, (self.out_kind, self.out_shape) = compile_plan(model)
        self.num_classes = model.num_classes() if is_last else None
        self._layout_params(model)
        self.load_state_dict(state_dict if state_dict is not None else model.state_dict())
        self.plans: Dict[int, "_Plan"] = {}
        self.eval_plans: Dict[int, "_Plan"] = {}
        self.step_ctr = torch.zeros(1, device=self.device, dtype=torch.int32)
        self.nan_flag = torch.zeros(1, device=self.device, dtype=torch.int32)
        self.loss_buf = torch.zeros(4, device=self.device)       # [0] = mean CE loss of the last microbatch
        self._store: Dict[Any, Tuple[int, int]] = {}      # data_id -> (batch, slot)
        self.slots = max(1, int(learning.get("control-count", 3))) if not is_last else 1
        # Stages sharing a GPU (N = 1: one stream per stage) compete for SMs.  SLB200_STAGE_PRIO = none (default) | last |
        # first raises the CUDA priority of that stage's streams (captured into its graph nodes).  Measured, same box:
        # "last" (the critical path) is 10 % SLOWER (32.6 k vs 36.3 k images/s: the first stage's persistent cut-tail kernel
        # then waits for SMs with part of its CTAs already spinning at their grid barrier) and "first" 4 % slower (35.1 k vs
        # 36.5 k) — equal priorities let the hardware interleave best.
        prio = os.environ.get("SLB200_STAGE_PRIO", "none")
        self.stream_priority = -1 if ((prio == "last" and is_last) or (prio == "first" and is_first)) else 0
        self.stream = N.new_stream(self.device, self.stream_priority)
        # device data plane hooks (set by parallel.mailbox): where the stage output / input gradient go
        self.out_target = None
        self.grad_target = None

    # ------------------------------------------------------------------ parameters
    def _layout_params(self, model: SplitModel) -> None:
        """Flat fp32 master layout; every tensor starts on a 128-element boundary."""
        self.entries: Dict[str, Tuple[int, Tuple[int, ...]]] = {}   # key -> (offset, stored shape)
        off = 0
        for b in self.blocks:
            if isinstance(b, ConvBlock):
                if b.conv is not None:
                    self.entries[f"layer{b.conv}.weight"] = (off, (b.cout, 3, 3, b.cin))
                    off += _align(b.cout * 9 * b.cin)
                    self.entries[f"layer{b.conv}.bias"] = (off, (b.cout,))
                    off += _align(b.cout)
                if b.bn is not None:
                    self.entries[f"layer{b.bn}.weight"] = (off, (b.cout,))
                    off += _align(b.cout)
                    self.entries[f"layer{b.bn}.bias"] = (off, (b.cout,))
                    off += _align(b.cout)
            elif isinstance(b, LinearBlock):
                self.entries[f"layer{b.lin}.weight"] = (off, (b.fout, b.fin))
                off += _align(b.fout * b.fin)
                self.entries[f"layer{b.lin}.bias"] = (off, (b.fout,))
                off += _align(b.fout)
        self.n_params = max(off, 128)
        # contiguous [start, end) of every block's parameters in the flat buffers (per-block optimizer launches)
        self.block_range: Dict[int, Tuple[int, int]] = {}
        for bi, b in enumerate(self.blocks):
            keys = []
            if isinstance(b, ConvBlock):
                keys = [f"layer{b.conv}.weight", f"layer{b.conv}.bias"] if b.conv is not None else []
                keys += [f"layer{b.bn}.weight", f"layer{b.bn}.bias"] if b.bn is not None else []
            elif isinstance(b, LinearBlock):
                keys = [f"layer{b.lin}.weight", f"layer{b.lin}.bias"]
            if keys:
                lo = min(self.entries[k][0] for k in keys)
                hi = max(_align(self.entries[k][0] + math.prod(self.entries[k][1])) for k in keys)
                self.block_range[bi] = (lo, hi)
        dev = self.device
        if self.eval_only:                               # inference: parameters and statistics only, process-private
            def alloc(n):
                return torch.zeros(n, device=dev), None
        else:
            # The fp32 master lives in an IPC-exportable allocation: the round-end FedAvg all-reduce (parallel/allreduce.py)
            # reads and writes the replicas' masters in place over NVLink — no staging copy, no START payload next round.
            from ..parallel.mailbox import alloc_exportable

            def alloc(n):
                raw, handle, _ = alloc_exportable(n * 4, dev)
                return raw.view(torch.float32)[:n], handle
        self.P, self.P_handle = alloc(self.n_params)
        self.G = None if self.eval_only else torch.zeros(self.n_params, device=dev)
        self.M = None if self.eval_only else torch.zeros(self.n_params, device=dev)
        self.PB = None if self.fp32 else torch.zeros(self.n_params, device=dev, dtype=torch.bfloat16)
        # BatchNorm running statistics: one flat exportable buffer S (mean | var per BN, 128-aligned entries) plus a float
        # mirror I of the integer counters (4 floats per BN) that the all-reduce averages-and-rounds (src/Utils.py:59-60)
        self.stat_entries: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        self.int_entries: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        so = io = 0
        for b in self.blocks:
            if isinstance(b, ConvBlock) and b.bn is not None:
                self.stat_entries[f"layer{b.bn}.running_mean"] = (so, (b.cout,))
                so += _align(b.cout)
                self.stat_entries[f"layer{b.bn}.running_var"] = (so, (b.cout,))
                so += _align(b.cout)
                self.int_entries[f"layer{b.bn}.num_batches_tracked"] = (io, (1,))
                io += 4
        self.n_stats, self.n_ints = max(so, 128), max(io, 4)
        self.S, self.S_handle = alloc(self.n_stats)
        self.I, self.I_handle = alloc(self.n_ints)
        self.bn_state: Dict[int, Dict[str, torch.Tensor]] = {}
        for b in self.blocks:
            if isinstance(b, ConvBlock) and b.bn is not None:
                om = self.stat_entries[f"layer{b.bn}.running_mean"][0]
                ov = self.stat_entries[f"layer{b.bn}.running_var"][0]
                self.bn_state[b.bn] = {"running_mean": self.S[om:om + b.cout], "running_var": self.S[ov:ov + b.cout],
                                       "num_batches_tracked": torch.zeros((), device=dev, dtype=torch.int64)}
                self.bn_state[b.bn]["running_var"].fill_(1.0)

    def view(self, buf: torch.Tensor, key: str) -> torch.Tensor:
        off, shape = self.entries[key]
        return buf[off:off + math.prod(shape)].view(shape)

    def W(self, key: str) -> torch.Tensor:
        """The tensor the GEMMs read: the fp32 master itself (tf32 mode) or its bf16 shadow."""
        return self.view(self.P if self.fp32 else self.PB, key)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        with torch.no_grad():
            for key, (off, shape) in self.entries.items():
                t = sd[key].to(self.device, torch.float32)
                if len(shape) == 4:                      # torch [Cout,Cin,3,3] -> stored [Cout,3,3,Cin]
                    t = t.permute(0, 2, 3, 1).contiguous()
                self.P[off:off + t.numel()].copy_(t.reshape(-1))
            for bn, st in self.bn_state.items():
                for k in st:
                    if f"layer{bn}.{k}" in sd:
                        st[k].copy_(sd[f"layer{bn}.{k}"].to(self.device))
            if self.PB is not None:
                self.PB.copy_(self.P)
        # stream-level, never device-wide: a device synchronize would also wait for kernels of *other* clients sharing the
        # GPU — including flag waits only this thread's next launch can release — and is not permitted while a sibling
        # thread captures a CUDA graph
        torch.cuda.current_stream(self.device).synchronize()

    def state_dict(self) -> Dict[str, torch.Tensor]:
        if getattr(self, "stream", None) is not None:
            self.stream.synchronize()                    # the stage's own work (side streams are joined into it per pass)
        torch.cuda.current_stream(self.device).synchronize()
        out = {}
        for key in self._sd_keys:
            if key in self.entries:
                t = self.view(self.P, key).detach().clone()
                if t.dim() == 4:
                    t = t.permute(0, 3, 1, 2).contiguous()
                out[key] = t
            else:
                layer, name = key.split(".", 1)
                out[key] = self.bn_state[int(layer[5:])][name].detach().clone()
        return out

    # ------------------------------------------------------------------ plans
    def plan(self, batch: int) -> "_Plan":
        if self.eval_only:
            raise RuntimeError("this executor was built with eval_only=True: it has no training plan")
        p = self.plans.get(batch)
        if p is None:
            p = self.plans[batch] = _Plan(self, batch)
        return p

    def eval_plan(self, batch: int) -> "_Plan":
        p = self.eval_plans.get(batch)
        if p is None:
            p = self.eval_plans[batch] = _Plan(self, batch, eval_mode=True)
        return p

    def eval_forward(self, x: torch.Tensor) -> torch.Tensor:
        """Eval-mode output of this stage (BatchNorm on running statistics, no dropout, fp32 numerics) in the wire layout of
        ``forward_only``.  Touches no training state: slots, stored microbatches, step counter, BN statistics, NaN flag."""
        xi = self._to_internal(x, torch.float32)
        pl = self.eval_plan(xi.shape[0])
        self._enter()
        with torch.cuda.stream(self.stream):
            pl.x_in[0].copy_(xi, non_blocking=True)
            pl.run_eval()
            out = self._from_internal_out(pl.final_out()).clone()
        self.stream.synchronize()
        return out

    # ------------------------------------------------------------------ StageExecutor API (tensor in / tensor out)
    def _to_internal(self, x: torch.Tensor, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        dtype = dtype or self.act_dtype
        x = x.to(self.device, non_blocking=True)
        if self.is_first:
            return x.float().contiguous()
        if self.in_kind == "image":
            if x.dim() == 4 and x.shape[1] == self.in_shape[0] and x.shape[-1] != self.in_shape[0]:
                x = x.permute(0, 2, 3, 1)                # NCHW wire -> NHWC
            return x.to(dtype).contiguous()
        return x.to(dtype).contiguous()

    def _from_internal_out(self, t: torch.Tensor) -> torch.Tensor:
        if self.out_kind == "image":
            return t.permute(0, 3, 1, 2).float().contiguous()       # NCHW fp32 on the compat wire
        return t.float()

    def _enter(self) -> None:
        """Tensor-API calls may hand us tensors produced on the caller's stream."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))

    def _grad_to_wire(self, gi: torch.Tensor) -> torch.Tensor:
        if self.in_kind == "image":
            c, h, w = self.in_shape
            return gi.reshape(gi.shape[0], h, w, c).permute(0, 3, 1, 2).float().contiguous()
        return gi.float()

    def forward_only(self, data_id, x) -> torch.Tensor:
        xi = self._to_internal(x)
        B = xi.shape[0]
        pl = self.plan(B)
        slot = pl.acquire_slot()
        self._enter()
        with torch.cuda.stream(self.stream):
            pl.x_in[slot].copy_(xi, non_blocking=True)
            pl.run_forward(slot)
            out = self._from_internal_out(pl.final_out())
        self.stream.synchronize()
        self._store[data_id] = (B, slot)
        return out

    def backward(self, data_id, grad) -> Optional[torch.Tensor]:
        B, slot = self._store.pop(data_id)
        pl = self.plan(B)
        g = grad.to(self.device)
        if self.out_kind == "image" and g.dim() == 4 and g.shape[1] == self.out_shape[0] and g.shape[-1] != self.out_shape[0]:
            g = g.permute(0, 2, 3, 1)
        g = g.to(self.act_dtype)
        self._enter()
        with torch.cuda.stream(self.stream):
            pl.dout_in.copy_(g, non_blocking=True)
            pl.run_backward(slot)
            res = None
            if not self.is_first:
                res = self._grad_to_wire(pl.input_grad())
        self.stream.synchronize()
        pl.release_slot(slot)
        return res

    def forward_backward_last(self, x, labels) -> Optional[torch.Tensor]:
        xi = self._to_internal(x)
        B = xi.shape[0]
        pl = self.plan(B)
        labels = labels.to(self.device)
        self._enter()
        with torch.cuda.stream(self.stream):
            pl.x_in[0].copy_(xi, non_blocking=True)
            pl.labels.copy_(labels, non_blocking=True)
            pl.run_last()
            res = None
            if not self.is_first:
                res = self._grad_to_wire(pl.input_grad())
        self.stream.synchronize()
        return res

    def nan_detected(self) -> bool:
        return bool(int(self.nan_flag.item()))

    def reset_epoch(self):
        self.nan_flag.zero_()
        self._store.clear()
        for p in self.plans.values():
            p.free = list(range(p.n_slots))

    def in_flight(self) -> int:
        return len(self._store)

    def last_loss(self):
        return float(self.loss_buf[0].item())


# ----------------------------------------------------------------------------- per-batch-size plan
class _Plan:
    """Static buffers + captured graphs for one batch size.  ``eval_mode``: the inference forward only (forward buffers,
    one input slot, fp32 activations and weights whatever the executor's precision)."""

    def __init__(self, ex: B200Executor, B: int, eval_mode: bool = False):
        self.ex, self.B = ex, B
        self.eval = eval_mode
        train = not eval_mode
        self.fp32 = ex.fp32 or eval_mode
        self.ke = 32 if self.fp32 else ex.ke
        dev = ex.device
        bf = torch.float32 if eval_mode else ex.act_dtype  # activation dtype of this plan (fp32 in tf32 mode)
        self.n_slots = 1 if eval_mode else ex.slots
        self.free = list(range(self.n_slots))
        # ---- stage input slots
        if ex.is_first:
            c, h, w = ex.in_shape
            self.x_in = [torch.zeros(B, c, h, w, device=dev) for _ in range(self.n_slots)]
        elif ex.in_kind == "image":
            c, h, w = ex.in_shape
            self.x_in = [torch.zeros(B, h, w, c, device=dev, dtype=bf) for _ in range(self.n_slots)]
        else:
            self.x_in = [torch.zeros(B, ex.in_shape[0], device=dev, dtype=bf) for _ in range(self.n_slots)]
        self.labels = torch.zeros(B, device=dev, dtype=torch.int64)
        # ---- zero-scratch (BN sums, split-K accumulators of the bf16 Linear GEMMs): one contiguous region, one zero kernel
        # per pass
        scratch = 0
        self.soff: Dict[Tuple[int, str], Tuple[int, int]] = {}
        # ---- split-K / slice partials of the conv kernels (in-kernel finalisation) and the fp32 Linear kernels: every
        # element is stored before it is read, so they need no zeroing.  One region serves every such launch of the plan:
        # all of them run on the plan's stream, a conv launch adds up its own partials before it completes, and the kernel
        # that adds up a Linear launch's partials (linear_finalize / linear_bwd_prep / dropout_bwd) precedes the next
        # launch that writes the region.
        part = 0

        def reserve(key, n):
            nonlocal scratch
            self.soff[key] = (scratch, n)
            scratch += _align(n, 4)
        for bi, b in enumerate(ex.blocks):
            if isinstance(b, ConvBlock):
                if b.bn is not None and train:
                    reserve((bi, "sum"), b.cout)
                    reserve((bi, "sumsq"), b.cout)
                if b.conv is not None and b.cin > 4:
                    M = B * b.H * b.W
                    part = max(part, N.conv_partial_floats(M, b.cout, N.conv_tiling(M, b.cout, b.cin, ke=self.ke)[1]))
                    if train and not (bi == 0 and ex.is_first):
                        part = max(part, N.conv_partial_floats(M, b.cin, N.conv_tiling(M, b.cin, b.cout, flip=1, ke=ex.ke)[1]))
            elif isinstance(b, LinearBlock) and self.fp32:
                part = max(part, N.linear_f32_slices(False, b.fout, b.fin) * B * b.fout)
                if train:
                    part = max(part, N.linear_f32_slices(True, b.fout, b.fin) * B * b.fin)
            elif isinstance(b, LinearBlock):
                reserve((bi, "acc"), B * b.fout)
                if train:
                    reserve((bi, "dacc_in"), B * b.fin)
        self.scratch = torch.zeros(max(scratch, 4), device=dev)
        self.part = torch.zeros(part, device=dev) if part else None
        # ---- activations
        self.act: List[Dict[str, torch.Tensor]] = []
        for bi, b in enumerate(ex.blocks):
            d: Dict[str, torch.Tensor] = {}
            if isinstance(b, ConvBlock):
                OH, OW = (b.H // 2, b.W // 2) if b.pool else (b.H, b.W)
                if b.conv is not None:
                    d["y"] = torch.zeros(B, b.H, b.W, b.cout, device=dev, dtype=bf)
                    if train:
                        d["dy"] = torch.zeros(B, b.H, b.W, b.cout, device=dev, dtype=bf)
                d["out"] = d["y"] if (b.conv is not None and b.bn is None) else torch.zeros(B, OH, OW, b.cout, device=dev, dtype=bf)
                if train:
                    d["bwd_bar"] = torch.zeros(4, device=dev, dtype=torch.int32)     # grid-barrier words of the fused BN backward
                    d["save_mean"] = torch.zeros(b.cout, device=dev)
                    d["save_invstd"] = torch.ones(b.cout, device=dev)
                    d["dx"] = torch.zeros(B, b.H, b.W, b.cin, device=dev, dtype=bf) if (b.cin > 4 and b.conv is not None) else None
                    if b.conv is None:
                        d["dx_orphan"] = torch.zeros(B, b.H, b.W, b.cout, device=dev, dtype=bf)
                    d["dout_bf16"] = torch.zeros(B, OH, OW, b.cout, device=dev, dtype=bf)
            elif isinstance(b, DropoutOp):
                if train:
                    d["out"] = torch.zeros(B, b.n, device=dev, dtype=bf)
                    d["mask"] = torch.zeros(B, b.n, device=dev, dtype=torch.uint8)
                    d["dx"] = torch.zeros(B, b.n, device=dev, dtype=bf)
            else:
                ld = _align(b.fout, 16)
                final_logits = bi == len(ex.blocks) - 1 and ex.is_last
                d["logits"] = torch.zeros(B, b.fout, device=dev) if final_logits else None
                if train:
                    d["out"] = torch.zeros(B, ld, device=dev, dtype=bf)[:, :b.fout]
                    d["dz"] = torch.zeros(B, ld, device=dev, dtype=bf)[:, :b.fout]
                    d["mask"] = torch.zeros(B, b.fout, device=dev, dtype=torch.uint8) if b.drop > 0 else None
                    d["dx_bf16"] = torch.zeros(B, b.fin, device=dev, dtype=bf)
                else:                                      # the final Linear of the model writes the fp32 logits only
                    d["out"] = d["logits"] if final_logits else torch.zeros(B, ld, device=dev, dtype=bf)[:, :b.fout]
            self.act.append(d)
        self.ticket = torch.zeros(4, device=dev, dtype=torch.int32)
        self.tile_counters = torch.zeros(4096, device=dev, dtype=torch.int32)   # split-K tile semaphores (self-resetting)
        if train:
            # gradient w.r.t. the stage output (arrives from the next stage)
            last = self.act[-1]["out"]
            self.dout_in = torch.zeros(last.shape, device=dev, dtype=bf)
            self.dlogits = torch.zeros(B, ex.num_classes, device=dev) if ex.is_last else None
            self.gnorm = torch.zeros(4, device=dev)                             # clip-grad-norm: sum of squared gradients
            # weight-gradient kernels run on a forked stream: they only feed the optimizer, so they overlap with the
            # dY -> dX critical path of the layers below (captured as parallel branches of the CUDA graph)
            self.side = N.new_stream(dev, ex.stream_priority)
        self.graphs: Dict[Tuple[str, int], torch.cuda.CUDAGraph] = {}
        self._warm = False

    # ---- helpers -----------------------------------------------------------------
    def s(self, bi: int, name: str, shape=None) -> torch.Tensor:
        off, n = self.soff[(bi, name)]
        t = self.scratch[off:off + n]
        return t.view(shape) if shape is not None else t

    def W(self, key: str) -> torch.Tensor:
        """Weights the GEMMs of this plan read: the executor's choice, or the fp32 master in eval mode."""
        return self.ex.view(self.ex.P, key) if self.eval else self.ex.W(key)

    def acquire_slot(self) -> int:
        if not self.free:
            raise RuntimeError("more microbatches in flight than control-count slots")
        return self.free.pop(0)

    def release_slot(self, slot: int) -> None:
        self.free.append(slot)

    def final_out(self) -> torch.Tensor:
        return self.act[-1]["out"]

    def input_grad(self) -> torch.Tensor:
        first = self.ex.blocks[0]
        a = self.act[0]
        if isinstance(first, ConvBlock):
            return a["dx"] if first.conv is not None else a["dx_orphan"]
        if isinstance(first, DropoutOp):
            return a["dx"]
        return a["dx_bf16"]

    # ---- the kernel sequences ------------------------------------------------------
    def _forward(self, slot: int, out_ptr_override: Optional[torch.Tensor] = None, publish=None, wait=None) -> None:
        """``wait``: (flag_ptr, expect_ctr, max_spins, status) of the mailbox slot this pass consumes — acquired inside the
        pass's first kernel (the scratch zeroing) instead of a stand-alone wait launch.  An eval-mode plan runs the same
        sequence with BatchNorm on the running statistics (no conv statistics, no fused cut tail) and no dropout."""
        ex = self.ex
        ev = self.eval
        N.zero_(self.scratch, wait=wait)
        x: torch.Tensor = self.x_in[slot]
        nb = len(ex.blocks)
        for bi, b in enumerate(ex.blocks):
            a = self.act[bi]
            is_final = bi == nb - 1
            if isinstance(b, ConvBlock):
                a["in"] = x
                plain = b.conv is not None and b.bn is None          # cut right after the conv (e.g. cut 4)
                if plain:
                    tgt = a["y"] if not (is_final and out_ptr_override is not None) else out_ptr_override
                    facc = self.part
                    N.conv3x3_fwd(x, self.W(f"layer{b.conv}.weight"), tgt, ex.view(ex.P, f"layer{b.conv}.bias"),
                                  acc=facc, counters=self.tile_counters)
                    if is_final and publish is not None:
                        N.set_flag(publish["flag"].data_ptr() if hasattr(publish["flag"], "data_ptr") else publish["flag"],
                                   0, publish["seq"], publish.get("hint_ptr", 0))
                    a["out"] = a["y"]
                    a["y_eff"] = a["y"]
                    x = tgt
                    continue
                fuse = (ex.fused_cut and not ev and is_final and out_ptr_override is not None and b.conv is not None and b.bn is not None
                        and b.cin > 4 and N.fused_cut_supported(self.B, b.H, b.W, b.cin, b.cout, b.pool, ke=ex.ke))
                if fuse:
                    # cut-tail kernel: GEMM + BN statistics + BN/ReLU/pool + store into the (peer) mailbox + flag
                    st = ex.bn_state[b.bn]
                    bar = a.get("grid_bar")
                    if bar is None:
                        bar = a["grid_bar"] = torch.zeros(4, device=ex.device, dtype=torch.int32)
                    keep_y = a["y"] if not ex.recompute or ex.is_last else None
                    kw = {}
                    if publish is not None:
                        kw = dict(flag=publish["flag"], seq=publish["seq"], hint=publish.get("hint"))
                    N.conv_bn_act_p2p(x, ex.W(f"layer{b.conv}.weight"), ex.view(ex.P, f"layer{b.conv}.bias"),
                                      ex.view(ex.P, f"layer{b.bn}.weight"), ex.view(ex.P, f"layer{b.bn}.bias"),
                                      st["running_mean"], st["running_var"], st["num_batches_tracked"], a["save_mean"],
                                      a["save_invstd"], self.s(bi, "sum"), self.s(bi, "sumsq"), keep_y, out_ptr_override,
                                      b.relu, b.pool, bar, **kw)
                    a["y_eff"] = a["y"]
                    x = out_ptr_override
                    continue
                if b.conv is not None:
                    s1, s2 = (None, None) if ev else (self.s(bi, "sum"), self.s(bi, "sumsq"))
                    bias = ex.view(ex.P, f"layer{b.conv}.bias")
                    if b.cin <= 4:
                        N.conv3x3_small_fwd(x, ex.view(ex.P, f"layer{b.conv}.weight"), bias, a["y"], s1, s2)
                    else:
                        facc = self.part
                        N.conv3x3_fwd(x, self.W(f"layer{b.conv}.weight"), a["y"], bias, s1, s2, acc=facc,
                                      counters=self.tile_counters)
                    y = a["y"]
                else:
                    y = x
                    if b.bn is not None and not ev:
                        s1, s2 = self.s(bi, "sum"), self.s(bi, "sumsq")
                        N.col_stats(y.reshape(-1, b.cout), s1, s2)
                out = a["out"] if not (is_final and out_ptr_override is not None) else out_ptr_override
                kw = {}
                if is_final and publish is not None:
                    kw = dict(ticket=self.ticket, flag=publish["flag"], seq=publish["seq"], hint=publish.get("hint"))
                if b.bn is not None and ev:
                    st = ex.bn_state[b.bn]
                    N.bn_relu_pool_infer(y, ex.view(ex.P, f"layer{b.bn}.weight"), ex.view(ex.P, f"layer{b.bn}.bias"),
                                         st["running_mean"], st["running_var"], out, b.H, b.W, b.relu, b.pool)
                elif b.bn is not None:
                    st = ex.bn_state[b.bn]
                    N.bn_relu_pool_fwd(y, self.s(bi, "sum"), self.s(bi, "sumsq"), ex.view(ex.P, f"layer{b.bn}.weight"),
                                       ex.view(ex.P, f"layer{b.bn}.bias"), st["running_mean"], st["running_var"],
                                       st["num_batches_tracked"], a["save_mean"], a["save_invstd"], out, b.H, b.W,
                                       b.relu, b.pool, **kw)
                else:
                    N.bn_relu_pool_fwd(y, None, None, None, None, None, None, None, a.get("save_mean"), a.get("save_invstd"),
                                       out, b.H, b.W, b.relu, b.pool, update_running=False, identity=True, **kw)
                a["y_eff"] = y
                x = a["out"] if out is a["out"] else out
            elif isinstance(b, DropoutOp):
                xin = x.reshape(self.B, -1)
                a["in"] = xin
                if ev:                                     # inference: dropout is the identity
                    a["out"] = xin
                else:
                    N.dropout_fwd(xin, a["out"], a["mask"], b.p, ex.seed + b.idx, ex.step_ctr)
                x = a["out"]
            else:
                xin = x.reshape(self.B, -1)
                a["in"] = xin
                w = self.W(f"layer{b.lin}.weight")
                if self.fp32:
                    acc = N.linear_fwd_f32(xin, w, self.part)      # slice partials, summed by linear_finalize
                else:
                    acc = self.s(bi, "acc", (self.B, b.fout))
                    N.linear_fwd(xin, w, acc, k_split=max(1, min(8, (b.fin // 64) // 8)))
                if ev:
                    N.linear_finalize(acc, ex.view(ex.P, f"layer{b.lin}.bias"),
                                      None if a["out"] is a["logits"] else a["out"], a["logits"], None, b.relu)
                else:
                    N.linear_finalize(acc, ex.view(ex.P, f"layer{b.lin}.bias"), a["out"], a["logits"], a["mask"], b.relu,
                                      b.drop, ex.seed + b.lin, ex.step_ctr)
                x = a["out"]

    def _backward(self, dout: torch.Tensor, grad_out_override: Optional[torch.Tensor] = None, publish_grad=None) -> None:
        """dout: gradient w.r.t. the stage output — or fp32 dlogits on the last stage.  ``publish_grad = (flag_ptr, seq)``:
        when the stage input gradient is produced by the cut-head conv dgrad (stored straight into the upstream stage's
        mailbox), that kernel's last CTA also publishes the slot flag; ``self.grad_published`` tells the caller."""
        ex = self.ex
        self.grad_published = False
        g: Any = dout
        main = torch.cuda.current_stream()
        side = self.side
        forked = False

        clip = ex.clip > 0.0                       # clip-grad-norm: the update needs the global norm -> one SGD at the end

        def sgd_block(bi):
            if clip:
                return
            lo, hi = ex.block_range[bi]
            N.sgd_momentum(ex.P[lo:hi], ex.G[lo:hi], ex.M[lo:hi], None if ex.PB is None else ex.PB[lo:hi], ex.lr, ex.mu)

        def on_side(fn):
            """Run ``fn`` (weight-gradient launches) on the side stream after everything issued so far on ``main``."""
            nonlocal forked
            ev = torch.cuda.Event()
            ev.record(main)
            with torch.cuda.stream(side):
                side.wait_event(ev)
                fn()
            forked = True

        bn_reduced = set()          # blocks whose dgamma / dbeta were produced by the downstream dgrad epilogue
        for bi in range(len(ex.blocks) - 1, -1, -1):
            b, a = ex.blocks[bi], self.act[bi]
            need_dx = not (bi == 0 and ex.is_first)
            if isinstance(b, LinearBlock):
                # g: fp32 [B, fout] accumulated gradient (dacc) or bf16 gradient from the wire
                if g.dtype != torch.float32:
                    g = g.float()                                   # compat path only (outside graphs)
                N.linear_bwd_prep(g, a["out"], a["mask"], a["dz"], ex.view(ex.G, f"layer{b.lin}.bias"), b.relu, b.drop)
                wkey, bkey = f"layer{b.lin}.weight", f"layer{b.lin}.bias"
                fuse_sgd = ex.fp32 and not clip and self.B <= 32
                if not ex.fp32:
                    on_side(lambda a=a, b=b: N.linear_wgrad(a["dz"], a["in"], ex.view(ex.G, f"layer{b.lin}.weight")))
                elif not fuse_sgd:
                    on_side(lambda a=a, wkey=wkey: N.linear_wgrad_f32(a["dz"], a["in"], g=ex.view(ex.G, wkey)))
                if need_dx:
                    if ex.fp32:                                     # slice partials, summed by the consumer of g
                        dacc = N.linear_dgrad_f32(a["dz"], ex.W(wkey), self.part)
                    else:
                        dacc = self.s(bi, "dacc_in", (self.B, b.fin))
                        N.linear_dgrad(a["dz"], ex.W(wkey), dacc, k_split=max(1, min(8, (b.fout // 64) // 8)))
                    g = dacc
                    if bi == 0:                                     # stage input gradient leaves in the activation dtype
                        N.dropout_bwd(dacc, None, a["dx_bf16"], 0.0)
                # this block's optimizer step runs on the side stream as soon as its dgrad (the last reader of the
                # weights) has been issued: the 134 MB classifier update hides behind the conv backward chain.  In
                # tf32 mode the update rides on the weight-gradient pass itself (no gradient buffer traffic at all).
                if fuse_sgd:
                    on_side(lambda a=a, wkey=wkey, bkey=bkey: N.linear_wgrad_f32(
                        a["dz"], a["in"], sgd=(ex.view(ex.P, wkey), ex.view(ex.M, wkey), ex.view(ex.P, bkey), ex.view(ex.M, bkey),
                                               ex.view(ex.G, bkey), ex.lr, ex.mu)))
                else:
                    on_side(lambda bi=bi: sgd_block(bi))
            elif isinstance(b, DropoutOp):
                N.dropout_bwd(g, a["mask"], a["dx"], b.p)
                g = a["dx"]
            else:
                if g.dim() == 3 or g.dtype != ex.act_dtype:         # a Linear block's fp32 slice partials / bf16-mode accumulator
                    tmp = a["dout_bf16"]
                    N.dropout_bwd(g, None, tmp, 0.0)
                    g = tmp
                g = g.reshape(a["out"].shape)
                y = a["y_eff"]
                if b.conv is not None:
                    dy = a["dy"]
                else:
                    dy = a["dx_orphan"]
                    if bi == 0 and grad_out_override is not None:
                        dy = grad_out_override
                if b.conv is not None and b.bn is None:
                    dy = g.reshape(y.shape)
                elif b.bn is not None:
                    N.bn_relu_pool_bwd(g, y, ex.view(ex.P, f"layer{b.bn}.weight"), ex.view(ex.P, f"layer{b.bn}.bias"),
                                       a["save_mean"], a["save_invstd"], ex.view(ex.G, f"layer{b.bn}.weight"),
                                       ex.view(ex.G, f"layer{b.bn}.bias"), dy, b.H, b.W, b.relu, b.pool,
                                       grid_bar=a["bwd_bar"] if ex.fused_bn_bwd else None, reduced=bi in bn_reduced)
                else:
                    N.bn_relu_pool_bwd(g, y, None, None, a["save_mean"], a["save_invstd"], None, None, dy, b.H, b.W,
                                       b.relu, b.pool, identity=True)
                if b.conv is not None:
                    if b.bn is None:
                        N.col_stats(dy.reshape(-1, b.cout), ex.view(ex.G, f"layer{b.conv}.bias"), None)
                    # else: a conv bias feeding train-mode BatchNorm has an identically zero gradient
                    # (sum_p dy = gamma*invstd*(sum dz - P*mean(dz) - mean(dz*xhat)*sum xhat) = 0): G stays 0.
                    if b.cin <= 4:
                        on_side(lambda a=a, b=b, dy=dy: N.conv3x3_small_wgrad(a["in"], dy, ex.view(ex.G, f"layer{b.conv}.weight")))
                    else:
                        on_side(lambda a=a, b=b, dy=dy: N.conv3x3_wgrad(a["in"], dy, ex.view(ex.G, f"layer{b.conv}.weight")))
                        if need_dx:
                            dx = a["dx"] if not (bi == 0 and grad_out_override is not None) else grad_out_override
                            dacc = self.part
                            stats = None
                            up = ex.blocks[bi - 1] if bi > 0 else None
                            if (ex.fused_bn_stats and not ex.fp32 and isinstance(up, ConvBlock) and up.conv is not None and up.bn is not None
                                    and (ex.fused_bn_stats >= 2 or not up.pool) and dx is a["dx"]):
                                ua = self.act[bi - 1]
                                stats = (ua["y_eff"], ua["save_mean"], ua["save_invstd"], ex.view(ex.P, f"layer{up.bn}.weight"),
                                         ex.view(ex.P, f"layer{up.bn}.bias"), up.relu, up.pool, ex.view(ex.G, f"layer{up.bn}.weight"),
                                         ex.view(ex.G, f"layer{up.bn}.bias"))
                                bn_reduced.add(bi - 1)
                            pub = None
                            if bi == 0 and grad_out_override is not None and publish_grad is not None and stats is None:
                                pub = (self.ticket[1:2], publish_grad[0], publish_grad[1])
                                self.grad_published = True
                            N.conv3x3_dgrad(dy, ex.W(f"layer{b.conv}.weight"), dx, acc=dacc, counters=self.tile_counters,
                                            bn_stats=stats, publish=pub)
                            g = dx
                else:
                    g = dy
                if bi in ex.block_range:
                    on_side(lambda bi=bi: sgd_block(bi))
        if forked:
            main.wait_stream(side)                      # join: every weight gradient and parameter update is complete
        if clip:
            # torch.nn.utils.clip_grad_norm_ + optimizer.step() (other/Vanilla_SL/src/Scheduler.py:204-205) on the flat buffers
            N.zero_(self.gnorm)
            N.sumsq(ex.G, self.gnorm)
            N.clip_scale(ex.G, self.gnorm, ex.clip)
            N.sgd_momentum(ex.P, ex.G, ex.M, ex.PB, ex.lr, ex.mu)
        N.counter_inc(ex.step_ctr)

    def _last(self, slot: int = 0, labels: Optional[torch.Tensor] = None, grad_out_override=None, wait=None,
              publish_grad=None) -> None:
        ex = self.ex
        self._forward(slot, wait=wait)
        logits = self.act[-1]["logits"]
        N.zero_(ex.loss_buf)
        N.ce_fwd_bwd(logits, self.labels if labels is None else labels, self.dlogits, ex.loss_buf, ex.nan_flag)
        self._backward(self.dlogits, grad_out_override, publish_grad=publish_grad)

    def bind_inputs(self, tensors) -> None:
        """Use externally owned buffers (mailbox slots) as the stage-input slots."""
        assert len(tensors) >= 1 and tuple(tensors[0].shape) == tuple(self.x_in[0].shape), \
            (tuple(tensors[0].shape), tuple(self.x_in[0].shape))
        self.x_in = list(tensors)
        self.n_slots = len(tensors)
        self.free = list(range(self.n_slots))
        self.graphs.clear()

    # ---- graph management ---------------------------------------------------------
    def run_forward(self, slot: int) -> None:
        self._exec(("fwd", slot), lambda: self._forward(slot))

    def run_backward(self, slot: int) -> None:
        def body():
            if self.ex.recompute:
                self._forward(slot)
            self._backward(self.dout_in)
        self._exec(("bwd", slot), body)

    def run_last(self) -> None:
        self._exec(("last", 0), lambda: self._last())

    def run_eval(self, metrics=None) -> None:
        """Eval-mode forward of ``x_in[0]``; ``metrics = (loss_total, correct, count)`` device accumulators: the same graph
        also adds this batch's loss / accuracy against ``labels`` (last stage only)."""
        def body():
            self._forward(0)
            if metrics is not None:
                N.eval_metrics(self.act[-1]["logits"], self.labels, *metrics)
        self._exec(("eval", int(metrics is not None)), body)

    def _exec(self, key, fn) -> None:
        ex = self.ex
        if not ex.use_graphs:
            fn()
            return
        g = self.graphs.get(key)
        if g is not None:
            g.replay()
            return
        if not self._warm:
            fn()                                       # first call ever: run eagerly (this is the real step)
            self._warm = True
            return
        # second call onwards for this key: capture, then replay (capture itself does not execute)
        from ..utils.timing import capture_graph
        g = capture_graph(torch.cuda.current_stream(), fn)
        self.graphs[key] = g
        g.replay()
