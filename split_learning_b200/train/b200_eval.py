"""Native full-model evaluation of a VGG-family model (server-side validation on the sm_90a kernels).

``NativeEvaluator`` runs the eval-mode forward of ``B200Executor`` (BatchNorm on the running statistics, no dropout, fp32
numerics) for layers 0..end, plus one kernel that adds each batch's mean cross-entropy, correct predictions and sample
count to device accumulators.  Per batch size the forward and the metrics are one CUDA graph on the evaluator's own stream;
the host reads the totals once, after the last batch.  Nothing for training is allocated: no gradient, momentum, bf16
shadow, backward activation or exportable memory.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch

from ..ops import native as N
from .b200_executor import B200Executor, supports


def native_eval_supported(model_cls) -> bool:
    """Whether ``model_cls(0, end)`` has a native eval plan — decided from the layer table on the meta device."""
    try:
        with torch.device("meta"):
            model = model_cls()
        return supports(model)
    except Exception:                 # a model family without a layer table (token models) has no native plan
        return False


class NativeEvaluator:
    def __init__(self, model_cls, state_dict: Dict[str, torch.Tensor], device, use_graphs: bool = True):
        with torch.device("meta"):
            model = model_cls()
        self.ex = B200Executor(model, "VGG16", {}, device, is_first=True, is_last=True, use_graphs=use_graphs,
                               eval_only=True, state_dict=state_dict)
        self.device = self.ex.device
        # [0] loss total (fp64), [1] correct, [2] samples (int64 views of the same words)
        self.acc = torch.zeros(4, dtype=torch.float64, device=self.device)
        ints = self.acc.view(torch.int64)
        self.metrics = (self.acc[0:1], ints[1:2], ints[2:3])
        self.host = torch.zeros(4, dtype=torch.float64).pin_memory()

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        self.ex.stream.synchronize()
        self.ex.load_state_dict(sd)

    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """Eval-mode fp32 logits of one batch (the kernel sequence ``evaluate`` runs)."""
        return self.ex.eval_forward(x)

    @torch.no_grad()
    def evaluate(self, source, pump: Optional[Callable[[], None]] = None) -> Dict[str, float]:
        """Same result dict as ``validation.evaluate``: loss = mean of the per-batch mean losses, accuracy in percent.
        ``source`` yields (x [B, C, H, W], labels [B]) on any device."""
        ex = self.ex
        batches = 0
        ex._enter()
        with torch.cuda.stream(ex.stream):
            N.zero_(self.acc)
            for i, (x, y) in enumerate(source):
                pl = ex.eval_plan(int(x.shape[0]))
                pl.x_in[0].copy_(x, non_blocking=True)
                pl.labels.copy_(torch.as_tensor(y), non_blocking=True)
                pl.run_eval(self.metrics)
                batches += 1
                if pump is not None and i % 5 == 4:
                    pump()
            self.host.copy_(self.acc, non_blocking=True)
        ex.stream.synchronize()
        ints = self.host.view(torch.int64)
        loss, correct, total = float(self.host[0]), int(ints[1]), int(ints[2])
        return {"val_loss": loss / max(batches, 1), "val_acc": 100.0 * correct / max(total, 1),
                "val_correct": correct, "val_total": total}
