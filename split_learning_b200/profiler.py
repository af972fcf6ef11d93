"""Offline device profiler → ``profiling.json`` (reference profiling.py:22-120).

Per indexed layer: forward time (ns, x3 fudge for fwd+bwd like the reference, :73), output
bytes (:74); ``speed`` = samples/s (:76); ``network`` = bytes/ns link bandwidth.  Timing uses
CUDA events around each ``layer{i}`` (not host clocks + synchronize), averaged over repeats.
The bandwidth probe measures what the data plane really uses here: a peer-to-peer copy into
another GPU's memory when one is visible, else a device-local copy (the reference publishes
1-9 MB blobs to RabbitMQ, :80-109).
"""
from __future__ import annotations

import json
import time
from typing import Dict, Optional

import torch

from .models import get_model_class


def profile_model(model_name: str, batch: int = 4, data_name: Optional[str] = None, repeats: int = 20,
                  device: Optional[str] = None) -> Dict:
    device = device or ("cuda" if torch.cuda.is_available() else "cpu")
    klass = get_model_class(model_name, data_name)
    model = klass().to(device).eval()
    x = klass.example_input(batch, device=device)
    cuda = torch.device(device).type == "cuda"
    n = klass.num_layers()
    times = [0.0] * n
    sizes = [0] * n
    with torch.no_grad():
        for _ in range(5):                                # warm up
            model(x)
        for _ in range(repeats):
            h = x
            for i in range(1, n + 1):
                if cuda:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                else:
                    t0 = time.perf_counter()
                # run exactly layer i through the model's own forward logic
                stage = _stage_cache(klass, i, model, device)
                h = stage(h) if not isinstance(h, dict) else stage(**h)
                if cuda:
                    e1.record()
                    torch.cuda.synchronize()
                    times[i - 1] += e0.elapsed_time(e1) * 1e6
                else:
                    times[i - 1] += (time.perf_counter() - t0) * 1e9
                sizes[i - 1] = h.nelement() * h.element_size()
    exe = [round(t / repeats * 3, 2) for t in times]
    total = sum(exe)
    return {"exe_time": exe, "size_data": sizes, "speed": round(batch / (total * 1e-9), 2) if total > 0 else 0.0}


def profile_speed(model_name: str, batch: int = 4, data_name: Optional[str] = None, rounds: int = 100,
                  device: Optional[str] = None, train: Optional[bool] = None) -> Dict:
    """Whole-model throughput only — the FLEX profiler (other/FLEX/profiling.py:23-92): BERT-like models time a full
    training step (forward of the mean, backward, AdamW), CNNs a forward pass; returns ``{"speed": samples/s}``.
    The step runs through the stage executor, i.e. the native sm_90a path on CUDA."""
    from .train.executor import make_executor
    device = device or ("cuda" if torch.cuda.is_available() else "cpu")
    klass = get_model_class(model_name, data_name)
    train = (model_name.upper() in ("BERT", "KWT", "VIT")) if train is None else train
    x = klass.example_input(batch, device=device)
    cuda = torch.device(device).type == "cuda"
    if train:
        ex = make_executor(klass(), model_name, {"learning-rate": 1e-5, "weight-decay": 0.01}, device, True, True)
        y = torch.zeros(batch, dtype=torch.long, device=device)
        fn = lambda: ex.forward_backward_last(x, y)
    else:
        model = klass().to(device).eval()

        def fn():
            with torch.no_grad():
                model(x)
    for _ in range(3):
        fn()
    if cuda:
        torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(rounds):
        fn()
    if cuda:
        torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / rounds
    return {"speed": round(batch / dt, 2)}


_CACHE: Dict = {}


def _stage_cache(klass, i, full, device):
    key = (klass, i, id(full))
    st = _CACHE.get(key)
    if st is None:
        st = klass(start_layer=i - 1, end_layer=i).to(device).eval()
        st.load_state_dict({k: v for k, v in full.state_dict().items() if k in st.state_dict()})
        _CACHE[key] = st
    return st


def probe_bandwidth(sizes_mb=(1, 2, 4, 8), repeats: int = 20) -> float:
    """bytes per nanosecond of the cut-edge path (peer copy if 2+ GPUs, else local copy)."""
    if not torch.cuda.is_available():
        src = torch.empty(8 << 20, dtype=torch.uint8)
        t0 = time.perf_counter()
        for _ in range(repeats):
            src.clone()
        return (8 << 20) * repeats / ((time.perf_counter() - t0) * 1e9)
    dst_dev = "cuda:1" if torch.cuda.device_count() > 1 else "cuda:0"
    speeds = []
    for mb in sizes_mb:
        a = torch.empty(mb << 20, dtype=torch.uint8, device="cuda:0")
        b = torch.empty(mb << 20, dtype=torch.uint8, device=dst_dev)
        b.copy_(a)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(repeats):
            b.copy_(a, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        speeds.append((mb << 20) * repeats / (e0.elapsed_time(e1) * 1e6))
    return round(sum(speeds) / len(speeds), 4)


def write_speed_profile(model_name: str, batch: int = 4, path: str = "profiling.json", data_name: Optional[str] = None,
                        rounds: int = 100) -> Dict:
    info = profile_speed(model_name, batch, data_name, rounds)
    with open(path, "w") as f:
        json.dump(info, f)
    return info


def write_profile(model_name: str, batch: int = 4, path: str = "profiling.json", data_name: Optional[str] = None) -> Dict:
    info = profile_model(model_name, batch, data_name)
    info["network"] = probe_bandwidth()
    with open(path, "w", encoding="utf-8") as f:
        json.dump(info, f, ensure_ascii=False, indent=4)
    return info
