"""Table-driven cut-able models.

Every model family is declared as an ordered table of ``LayerSpec`` entries
(1-based index == the cut-point vocabulary of the reference).  A stage is
``Klass(start_layer=a, end_layer=b)`` and owns exactly the entries with
``a < i <= b``; each owned entry becomes the attribute ``layer{i}`` so that
state-dict keys are globally unique and a full-model checkpoint is just the
union of the stage dicts (reference behaviour: src/model/VGG16_CIFAR10.py:4-117,
src/Server.py:410-434).

The same table is what the native stage executor compiles into a fused kernel
plan (``split_learning_b200/train/b200_executor.py``), so models are *data*
here, not code.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn


@dataclass(frozen=True)
class LayerSpec:
    """One indexed layer of a cut-able model.

    kind   : symbolic op name understood by both executors
             ("conv3x3", "bn2d", "relu", "maxpool2", "flatten", "dropout",
              "linear", or "module" for opaque torch sub-modules)
    args   : constructor arguments for the op
    """

    kind: str
    args: Tuple[Any, ...] = ()
    kwargs: Dict[str, Any] = field(default_factory=dict)

    def build(self) -> nn.Module:
        return _BUILDERS[self.kind](*self.args, **self.kwargs)


def _conv3x3(cin, cout):
    return nn.Conv2d(cin, cout, kernel_size=3, stride=1, padding=1)


_BUILDERS: Dict[str, Callable[..., nn.Module]] = {
    "conv3x3": _conv3x3,
    "conv": lambda *a, **k: nn.Conv2d(*a, **k),
    "bn2d": lambda c: nn.BatchNorm2d(c),
    "relu": lambda: nn.ReLU(),
    "maxpool2": lambda: nn.MaxPool2d(kernel_size=2, stride=2),
    "avgpool": lambda k: nn.AvgPool2d(k),
    "flatten": lambda start=1, end=-1: nn.Flatten(start, end),
    "dropout": lambda p: nn.Dropout(p),
    "linear": lambda i, o: nn.Linear(i, o),
    "module": lambda factory, *a, **k: factory(*a, **k),
}


def register_layer_kind(kind: str, builder: Callable[..., nn.Module]) -> None:
    _BUILDERS[kind] = builder


class SplitModel(nn.Module):
    """A contiguous slice ``(start_layer, end_layer]`` of a layer table."""

    #: subclasses set this: list of LayerSpec, index 0 == layer1
    LAYERS: Sequence[LayerSpec] = ()
    #: name used by registry / checkpoints ("VGG16"), and dataset ("CIFAR10")
    MODEL_NAME = ""
    DATA_NAME = ""

    def __init__(self, start_layer: int = 0, end_layer: Optional[int] = None):
        super().__init__()
        n = self.num_layers()
        if end_layer is None or end_layer == -1:
            end_layer = n
        if not (0 <= start_layer <= end_layer <= n):
            raise ValueError(
                f"{type(self).__name__}: invalid slice ({start_layer}, {end_layer}] of {n} layers")
        self.start_layer = int(start_layer)
        self.end_layer = int(end_layer)
        for i in self.owned_indices():
            setattr(self, f"layer{i}", self.LAYERS[i - 1].build())

    # -- table helpers -----------------------------------------------------
    @classmethod
    def num_layers(cls) -> int:
        return len(cls.LAYERS)

    def owned_indices(self) -> range:
        return range(self.start_layer + 1, self.end_layer + 1)

    def owned_specs(self) -> List[Tuple[int, LayerSpec]]:
        return [(i, self.LAYERS[i - 1]) for i in self.owned_indices()]

    # -- forward -----------------------------------------------------------
    def forward(self, x, **kwargs):
        if isinstance(x, dict):  # tolerate HF-style batches
            x = x["input_ids"]
        for i in self.owned_indices():
            x = getattr(self, f"layer{i}")(x)
        return x

    # -- convenience -------------------------------------------------------
    @classmethod
    def full_state_dict_keys(cls) -> List[str]:
        return list(cls().state_dict().keys())

    @classmethod
    def example_input(cls, batch: int, device="cpu") -> torch.Tensor:
        raise NotImplementedError

    @classmethod
    def num_classes(cls) -> int:
        raise NotImplementedError
