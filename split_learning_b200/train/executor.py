"""Stage executors.

``StageExecutor`` is the contract between the trainer loops and whatever runs a stage:
  * ``TorchExecutor``  — reference math through ``torch.nn``/autograd on any device.  Used on
    CPU (tests, plumbing config #1), for model families that do not yet have a native
    plan, and as the numerics oracle.
  * ``B200Executor``   — (``b200_executor.py``) VGG-family stages compiled to hand-written
    sm_90a kernels + CUDA graphs; selected automatically on CUDA.

Reference semantics preserved (SURVEY §3.3/§3.4):
  * non-last stages *recompute* the forward with current weights when the gradient comes
    back (src/train/VGG16.py:89-92) unless ``recompute=False`` (activation stashing);
  * one optimizer step per microbatch; SGD(lr, momentum) for VGG-like CNNs
    (src/train/VGG16.py:62,139), AdamW(lr, weight-decay) for BERT/KWT/ViT
    (src/train/BERT.py:69, src/train/KWT.py:62);
  * optional ``clip-grad-norm`` on the last stage (other/Vanilla_SL/src/Scheduler.py:204-205).
The NaN check is kept on-device and read once per epoch (reference reads ``loss.item()``
every step, quirk C7).
"""
from __future__ import annotations

from typing import Any, Dict, Optional

import torch
import torch.nn as nn

from ..models import SplitModel

_ADAMW_MODELS = ("BERT", "KWT", "VIT")


def make_optimizer(model: nn.Module, model_name: str, learning: dict, shadow: bool = False) -> torch.optim.Optimizer:
    params = [p for p in model.parameters() if p.requires_grad]
    lr = float(learning.get("learning-rate", 0.01))
    adamw = model_name.upper() in _ADAMW_MODELS
    if params and params[0].is_cuda:
        # CUDA: one flat buffer + the fused sm_90a optimizer kernels (no silent fallback: a missing library raises)
        from ..ops.optim import FlatFusedOptimizer
        return FlatFusedOptimizer(params, "adamw" if adamw else "sgd", lr=lr, momentum=float(learning.get("momentum", 0.0)),
                                  weight_decay=float(learning.get("weight-decay", 0.01)), shadow=shadow)
    if model_name.upper() in _ADAMW_MODELS:
        return torch.optim.AdamW(params, lr=lr, weight_decay=float(learning.get("weight-decay", 0.01)))
    return torch.optim.SGD(params, lr=lr, momentum=float(learning.get("momentum", 0.0)))


class StageExecutor:
    """Interface; see module docstring."""

    device: Any
    is_first: bool
    is_last: bool

    def forward_only(self, data_id, x) -> torch.Tensor: ...
    def backward(self, data_id, grad) -> Optional[torch.Tensor]: ...
    def forward_backward_last(self, x, labels) -> torch.Tensor: ...
    def state_dict(self) -> Dict[str, torch.Tensor]: ...
    def load_state_dict(self, sd) -> None: ...
    def nan_detected(self) -> bool: ...
    def in_flight(self) -> int: ...
    def last_loss(self) -> Optional[float]: ...


class TorchExecutor(StageExecutor):
    def __init__(self, model: SplitModel, model_name: str, learning: dict, device="cpu", is_first=False,
                 is_last=False, recompute: bool = True, clip_grad_norm: float = 0.0, native: bool = False,
                 graphs: bool = False):
        self.model = model.to(device)       # parameters must sit on the device before the optimizer re-homes them
        self.native = bool(native)
        if self.native:                     # blocks -> fused sm_90a ops (train/token_native.py, train/cnn_native.py)
            from . import cnn_native, token_native
            (cnn_native if cnn_native.supports(self.model) else token_native).nativize(self.model)
        self.model_name = model_name
        self.device = device
        self.is_first, self.is_last = is_first, is_last
        self.recompute = recompute
        self.clip = float(clip_grad_norm or 0.0)
        self.opt = make_optimizer(self.model, model_name, learning, shadow=self.native)
        self.criterion = nn.CrossEntropyLoss()
        self._store: Dict[Any, Any] = {}
        self._nan = torch.zeros((), dtype=torch.bool, device=device)
        self._loss = None
        self.graphs = bool(graphs) and self.native
        if self.graphs:
            self._graphs: Dict[Any, Any] = {}
            self._warm: Dict[Any, int] = {}
            self._replay_ctr = torch.zeros(1, dtype=torch.int32, device=device)
            self._loss_buf = torch.zeros((), device=device)
            self._cap_stream = torch.cuda.Stream(device)
        self.model.train()

    # -- helpers -------------------------------------------------------------
    def _call(self, x):
        out = self._call_model(x)
        return out.float() if self.native and out.dtype != torch.float32 else out    # stage boundary is fp32

    def _call_model(self, x):
        if isinstance(x, dict):
            return self.model(input_ids=x["input_ids"]) if self.is_first else self.model(x)
        if self.model_name.upper() == "BERT" and self.is_first:
            return self.model(input_ids=x)
        return self.model(x)

    def _prep_input(self, x):
        if isinstance(x, dict):
            return {k: v.to(self.device) for k, v in x.items() if k != "labels"}
        x = x.to(self.device)
        if not self.is_first and x.is_floating_point():
            x = x.float().detach().requires_grad_(True)
        return x

    # -- CUDA-graph capture of whole steps (native token models) -------------------------------------
    # A step of these models is a few hundred small kernels issued from Python (~30 us each on the host) while the GPU
    # needs a fraction of that: after two eager warm-up calls per input signature the whole call — forward, autograd
    # backward, gradient clipping, fused AdamW — is captured once and replayed.  What would be baked into the graph
    # lives on the device instead: the AdamW step count (bias correction) and a replay counter mixed into every
    # dropout seed (``ops.nn.set_seed_offset``).
    _MAX_GRAPHS = 6

    def _graphed(self, kind: str, tensors, body):
        from ..ops import nn as F
        F.set_seed_offset(self._replay_ctr)
        key = (kind,) + tuple((tuple(t.shape), t.dtype) for t in tensors)
        ent = self._graphs.get(key)
        if ent is None:
            seen = self._warm.get(key, 0)
            if seen < 2 or len(self._graphs) >= self._MAX_GRAPHS:
                self._warm[key] = seen + 1
                return body(*tensors)
            from ..utils.timing import capture_graph
            statics = [torch.empty_like(t) for t in tensors]
            for st, t in zip(statics, tensors):
                st.copy_(t)
            outs = []
            cur = torch.cuda.current_stream()
            self._cap_stream.wait_stream(cur)
            g = capture_graph(self._cap_stream, lambda: outs.extend(body(*statics)))
            ent = self._graphs[key] = (statics, g, outs)
        statics, g, outs = ent
        for st, t in zip(statics, tensors):
            st.copy_(t, non_blocking=True)
        g.replay()
        return tuple(o.clone() if o is not None else None for o in outs)

    def _tick(self):
        if self.graphs:
            from ..ops import native as N
            N.counter_inc(self._replay_ctr)

    # -- bodies (run eagerly, or once under capture) -----------------------------------------------------
    def _body_forward(self, x):
        self._tick()
        with torch.no_grad():
            return (self._call(x),)

    def _body_backward(self, x, grad):
        self._tick()
        self.opt.zero_grad(set_to_none=True)
        want_dx = x.is_floating_point() and not self.is_first
        if want_dx:
            x = x.detach().requires_grad_(True)
        out = self._call(x)
        out.backward(gradient=grad.to(out.dtype))
        self.opt.step()
        return (x.grad if want_dx else None,)

    def _body_last(self, x, labels):
        self._tick()
        self.opt.zero_grad(set_to_none=True)
        want_dx = x.is_floating_point() and not self.is_first
        if want_dx:
            x = x.detach().requires_grad_(True)
        out = self._call(x)
        loss = self.criterion(out, labels)
        self._nan |= torch.isnan(loss.detach())
        self._loss_buf.copy_(loss.detach())
        loss.backward()
        if self.clip > 0:
            nn.utils.clip_grad_norm_(self.model.parameters(), self.clip)
        self.opt.step()
        return (x.grad if want_dx else None,)

    # -- StageExecutor -----------------------------------------------------------
    def forward_only(self, data_id, x) -> torch.Tensor:
        self.model.train()
        x = self._prep_input(x)
        if self.graphs and self.recompute and isinstance(x, torch.Tensor):
            out, = self._graphed("fwd", (x.detach(),), self._body_forward)
            self._store[data_id] = (x, None)
            return out
        if self.recompute:
            with torch.no_grad():
                out = self._call(x)
            self._store[data_id] = (x, None)
        else:
            out = self._call(x)
            self._store[data_id] = (x, out)
        return out.detach()

    def backward(self, data_id, grad) -> Optional[torch.Tensor]:
        self.model.train()
        x, out = self._store.pop(data_id)
        if self.graphs and out is None and isinstance(x, torch.Tensor):
            gx, = self._graphed("bwd", (x.detach(), grad.to(self.device).float()), self._body_backward)
            return gx
        self.opt.zero_grad(set_to_none=True)
        if out is None:                       # faithful mode: recompute with *current* weights
            out = self._call(x)
        out.backward(gradient=grad.to(self.device).to(out.dtype))
        self.opt.step()
        if isinstance(x, torch.Tensor) and x.requires_grad:
            return x.grad
        return None

    def forward_backward_last(self, x, labels) -> Optional[torch.Tensor]:
        self.model.train()
        x = self._prep_input(x)
        labels = labels.to(self.device)
        if self.graphs and isinstance(x, torch.Tensor):
            gx, = self._graphed("last", (x.detach(), labels), self._body_last)
            self._loss = self._loss_buf
            return gx
        self.opt.zero_grad(set_to_none=True)
        out = self._call(x)
        loss = self.criterion(out, labels)
        self._nan |= torch.isnan(loss.detach())
        self._loss = loss.detach()
        loss.backward()
        if self.clip > 0:
            nn.utils.clip_grad_norm_(self.model.parameters(), self.clip)
        self.opt.step()
        if isinstance(x, torch.Tensor) and x.requires_grad:
            return x.grad
        return None

    def state_dict(self):
        return {k: v.detach().clone() for k, v in self.model.state_dict().items()}

    def load_state_dict(self, sd):
        self.model.load_state_dict(sd)
        if hasattr(self.opt, "refresh_shadow"):
            self.opt.refresh_shadow()

    def nan_detected(self) -> bool:
        return bool(self._nan.item())

    def reset_epoch(self):
        self._nan.zero_()
        self._store.clear()

    def in_flight(self) -> int:
        return len(self._store)

    def last_loss(self):
        return None if self._loss is None else float(self._loss.item())


def make_executor(model: SplitModel, model_name: str, learning: dict, device, is_first: bool, is_last: bool,
                  b200_opts: Optional[dict] = None) -> StageExecutor:
    """Pick the executor: native sm_90a plan on CUDA for supported tables, torch otherwise."""
    opts = b200_opts or {}
    kind = opts.get("executor", "auto")
    dev = torch.device(device)
    clip = float(learning.get("clip-grad-norm", 0.0) or 0.0) if is_last else 0.0
    if kind in ("auto", "b200") and dev.type == "cuda":
        from .b200_executor import B200Executor, supports
        if supports(model):
            # ``b200.precision`` (tf32 = the reference's precision, default; bf16 = fast mode); ``clip-grad-norm`` applies
            # on the last stage only, as in other/Vanilla_SL/src/Scheduler.py:204-205
            lrn = dict(learning)
            if opts.get("precision") and not lrn.get("precision"):
                lrn["precision"] = opts["precision"]
            if not is_last:
                lrn["clip-grad-norm"] = 0.0
            return B200Executor(model, model_name, lrn, device=dev, is_first=is_first, is_last=is_last,
                                recompute=bool(opts.get("recompute", True)))
        from .cnn_native import supports as cnn_supports
        from .token_native import supports as token_supports
        if (token_supports(model) or cnn_supports(model)) and opts.get("native-tokens", True):
            return TorchExecutor(model, model_name, learning, device=dev, is_first=is_first, is_last=is_last,
                                 recompute=bool(opts.get("recompute", True)), clip_grad_norm=clip, native=True,
                                 graphs=bool(opts.get("token-graphs", True)))
        if kind == "b200":
            raise RuntimeError(f"no native sm_90a plan for {type(model).__name__}")
    return TorchExecutor(model, model_name, learning, device=dev, is_first=is_first, is_last=is_last,
                         recompute=bool(opts.get("recompute", True)), clip_grad_norm=clip)
