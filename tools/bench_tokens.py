"""Step time of the token-model families and MobileNetv1, native sm_90a ops vs stock torch modules (same executor, same optimizer).

    python tools/bench_tokens.py [--steps 30] [--warmup 10]

Two stages on one GPU (first: forward, recompute + backward; last: forward + loss + backward + AdamW), the
reference's training step (src/train/BERT.py, src/train/KWT.py).  Device-timed with CUDA events.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from split_learning_b200.models import get_model_class  # noqa: E402
from split_learning_b200.ops import native as N  # noqa: E402
from split_learning_b200.train.executor import TorchExecutor  # noqa: E402

CASES = [("KWT", "SPEECHCOMMANDS", 8, 32), ("ViT", "CIFAR10", 6, 32), ("BERT", "AGNEWS", 6, 8), ("BERT", "EMOTION", 12, 8),
         ("MobileNetv1", "CIFAR10", 15, 32)]


def run(name, data, cut, batch, native, steps, warmup, graphs=False):
    cls = get_model_class(name, data)
    learning = {"learning-rate": 1e-4, "weight-decay": 0.01}
    torch.manual_seed(0)
    e1 = TorchExecutor(cls(0, cut), name, learning, "cuda", True, False, native=native, graphs=graphs)
    e2 = TorchExecutor(cls(cut, len(cls.LAYERS)), name, learning, "cuda", False, True, native=native, graphs=graphs)
    x = cls.example_input(batch, device="cuda")
    y = torch.randint(0, cls.num_classes(), (batch,), device="cuda")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches0 = 0
    for it in range(warmup + steps):
        if it == warmup:
            torch.cuda.synchronize()
            launches0 = N.LAUNCHES
            ev0.record()
        a = e1.forward_only(it, x)
        gx = e2.forward_backward_last(a, y)
        e1.backward(it, gx)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / steps
    return {"ms_per_step": round(ms, 3), "samples_per_s": round(batch / ms * 1e3, 1), "loss": round(e2.last_loss(), 4),
            "native_launches_per_step": (N.LAUNCHES - launches0) // steps}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    N.require()
    N.preload()
    rows = []
    for name, data, cut, batch in CASES:
        r = {"model": f"{name}_{data}", "cut": cut, "batch": batch}
        for native in (False, True):
            r["native" if native else "torch"] = run(name, data, cut, batch, native, a.steps, a.warmup)
        r["native_graphs"] = run(name, data, cut, batch, True, a.steps, a.warmup, graphs=True)
        r["speedup"] = round(r["torch"]["ms_per_step"] / r["native"]["ms_per_step"], 2)
        r["speedup_graphs"] = round(r["torch"]["ms_per_step"] / r["native_graphs"]["ms_per_step"], 2)
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
