"""Server-side validation of the merged full model (reference src/val/*.py, get_val.py).

Full model on the test split, batch 100 (images) / 20 (text, audio), CE as mean of batch
means + accuracy, logged through the server logger.  ``get_val`` returns ``(ok, metrics)``;
``strict=True`` adds the Vanilla_SL gate that fails the round on NaN / exploding loss
(other/Vanilla_SL/src/Validation.py:46,55-56).  ``pump`` is called every 5 batches — the
hook DCSL uses to keep its AMQP heartbeat alive (other/DCSL/src/Validation.py:48-52); here it
lets the broker thread breathe / watchdogs tick.

``native`` (``b200.native-validation``) selects the backend: ``false`` (default) the torch modules above; ``true`` the
native eval plan on the test split resident in HBM — ``train/b200_eval.py`` for VGG16_CIFAR10, ``train/token_eval.py``
for ViT_CIFAR10, BERT_AGNEWS and BERT_EMOTION — an error where there is none; ``auto`` native where supported, torch
otherwise with one log line giving the reason.  Metrics carry ``val_backend``.
"""
from __future__ import annotations

import logging
import math
from typing import Any, Callable, Dict, Optional, Tuple

import torch
import torch.nn as nn

from .data import data_loader
from .models import get_model_class

_NATIVE: Dict[Tuple, Any] = {}          # (model, data, device, synthetic) -> (evaluator, resident test split)


@torch.no_grad()
def evaluate(model: nn.Module, loader, device, pump: Optional[Callable[[], None]] = None) -> Dict[str, float]:
    criterion = nn.CrossEntropyLoss()
    model.eval()
    correct = total = 0
    total_loss, batches = 0.0, 0
    for i, batch in enumerate(loader):
        if isinstance(batch, dict):
            x, y = batch["input_ids"].to(device), batch["labels"].to(device)
            out = model(input_ids=x) if "input_ids" in model.forward.__code__.co_varnames else model(x)
        else:
            x, y = batch[0].to(device), torch.as_tensor(batch[1]).to(device)
            out = model(x)
        total_loss += float(criterion(out, y))
        correct += int((out.argmax(1) == y).sum())
        total += int(y.numel())
        batches += 1
        if pump is not None and i % 5 == 4:
            pump()
    return {"val_loss": total_loss / max(batches, 1), "val_acc": 100.0 * correct / max(total, 1),
            "val_correct": correct, "val_total": total}


def native_mode(native) -> str:
    """Normalise a ``b200.native-validation`` value to "false" | "true" | "auto"."""
    if native is None or isinstance(native, bool):
        return "true" if native else "false"
    s = str(native).strip().lower()
    if s in ("false", "0", "no", "off", ""):
        return "false"
    if s in ("true", "1", "yes", "on"):
        return "true"
    if s == "auto":
        return "auto"
    raise ValueError(f"b200.native-validation must be true, false or auto, got {native!r}")


def native_unsupported_reason(klass, data_name: str, device) -> Optional[str]:
    """Why the native evaluator cannot run this (model, data, device) — None when it can."""
    dev = torch.device(device)
    if dev.type != "cuda" or not torch.cuda.is_available():
        return "no CUDA device"
    from .train.token_eval import token_eval_supported
    if token_eval_supported(klass):
        if str(data_name).upper() != klass.DATA_NAME:
            return f"no resident test split for {data_name}"
        return None
    if str(data_name).upper() != "CIFAR10":
        return f"no resident test split for {data_name}"
    from .train.b200_eval import native_eval_supported
    if not native_eval_supported(klass):
        return f"{klass.__name__} has no native eval plan"
    return None


def _native_evaluate(klass, model_name, data_name, state_dict_full, device, pump, synthetic) -> Dict[str, float]:
    from .data import resident_test_loader
    from .train.b200_eval import NativeEvaluator
    from .train.token_eval import NativeTokenEvaluator, token_eval_supported
    dev = torch.device(device)
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    key = (model_name, str(data_name).upper(), str(dev), synthetic)
    hit = _NATIVE.get(key)
    if hit is None:
        cls = NativeTokenEvaluator if token_eval_supported(klass) else NativeEvaluator
        hit = _NATIVE[key] = (cls(klass, state_dict_full, dev), resident_test_loader(data_name, dev, synthetic))
    else:
        hit[0].load_state_dict(state_dict_full)
    evaluator, source = hit
    return evaluator.evaluate(source, pump)


def get_val(model_name: str, data_name: str, state_dict_full, logger=None, strict: bool = False,
            device: Optional[str] = None, pump=None, synthetic: Optional[bool] = None,
            native=False, speech_features: str = "engine") -> Tuple[bool, Dict[str, float]]:
    """``speech_features``: the Speech Commands MFCC recipe of the test loader (``b200.speech-features``); it must be the
    recipe the model was trained on."""
    try:
        klass = get_model_class(model_name, data_name)
    except ValueError:
        return False, {}
    device = device or ("cuda" if torch.cuda.is_available() else "cpu")
    mode = native_mode(native)
    backend = "torch"
    if mode != "false":
        reason = native_unsupported_reason(klass, data_name, device)
        if reason is None:
            backend = "native"
        elif mode == "true":
            raise RuntimeError(f"b200.native-validation is true but {model_name}/{data_name} on {device} cannot run "
                               f"natively: {reason}")
        else:
            line = f"native validation unavailable ({reason}): validating with torch"
            if logger is not None:
                logger.log_info(line)
            else:
                logging.getLogger(__name__).info(line)
    if backend == "native":
        m = _native_evaluate(klass, model_name, data_name, state_dict_full, device, pump, synthetic)
    else:
        model = klass()
        model.load_state_dict(state_dict_full)
        model.to(device)
        loader = data_loader(data_name=data_name, train=False, synthetic=synthetic, speech_features=speech_features)
        m = evaluate(model, loader, device, pump)
    m["val_backend"] = backend
    line = "Test set:Loss: {:.4f}; Accuracy: {}/{} ({:.2f}%)\n".format(
        m["val_loss"], m["val_correct"], m["val_total"], m["val_acc"])
    if logger is not None:
        logger.log_info(line)
    if strict and (math.isnan(m["val_loss"]) or abs(m["val_loss"]) > 1e6):
        return False, m
    return True, m
