"""FedAvg over state-dicts.

Semantics of reference src/Utils.py:35-66: weighted mean over the *union* of keys (a key
missing from some dicts is averaged over the present ones but still divided by the total
weight), fp32 accumulation, NaN → 0 before weighting, integer/bool tensors rounded back to
their dtype (this is how ``num_batches_tracked`` survives).  ``fedasync_merge`` is the
2LS running merge (other/2LS/src/Server.py:224-233).

On CUDA the per-key loop is replaced by one flat pass through the fused sm_90a kernel
(``ops.fedavg_flat``); across GPUs ``parallel.fedavg_allreduce`` performs the same math
in place over NVLink peer memory.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

_INT_DTYPES = (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8, torch.bool)


def fedavg_state_dicts(state_dicts: Sequence[Dict[str, torch.Tensor]],
                       weights: Optional[Sequence[float]] = None) -> Dict[str, torch.Tensor]:
    dicts = [sd for sd in state_dicts if sd is not None]
    if not dicts:
        return {}
    if weights is None:
        weights = [1.0] * len(dicts)
    weights = [float(w) for w in weights]
    total = float(sum(weights))
    keys: List[str] = []
    seen = set()
    for sd in dicts:                       # deterministic union (first-seen order)
        for k in sd:
            if k not in seen:
                seen.add(k)
                keys.append(k)
    out: Dict[str, torch.Tensor] = {}
    for k in keys:
        acc = None
        proto = None
        for sd, w in zip(dicts, weights):
            t = sd.get(k)
            if t is None:
                continue
            if proto is None:
                proto = t
            t32 = torch.nan_to_num(t.detach().float(), nan=0.0, posinf=float("inf"), neginf=float("-inf"))
            acc = t32 * w if acc is None else acc.add_(t32, alpha=w)
        avg = acc / total
        if proto.dtype in _INT_DTYPES:
            avg = avg.round().to(proto.dtype)
        else:
            avg = avg.to(proto.dtype)
        out[k] = avg
    return out


def fedasync_merge(global_sd: Optional[Dict[str, torch.Tensor]], new_sd: Dict[str, torch.Tensor],
                   alpha: float) -> Dict[str, torch.Tensor]:
    """g <- (1-alpha) g + alpha n  (keys only in one side are copied)."""
    if not global_sd:
        return {k: v.clone() for k, v in new_sd.items()}
    out = {}
    for k in set(global_sd) | set(new_sd):
        if k not in new_sd:
            out[k] = global_sd[k]
        elif k not in global_sd:
            out[k] = new_sd[k]
        else:
            g, n = global_sd[k], new_sd[k]
            m = (1.0 - alpha) * g.float() + alpha * n.float()
            out[k] = m.round().to(g.dtype) if g.dtype in _INT_DTYPES else m.to(g.dtype)
    return out


def has_nan(sd: Dict[str, torch.Tensor]) -> bool:
    return any(torch.isnan(v).any().item() for v in sd.values() if v.is_floating_point())
