"""Time server-side validation of the token models: stock torch modules fed by the host loader (``validation.evaluate``)
against the native eval program on the test split resident in HBM (``NativeTokenEvaluator``).

    python tools/bench_token_validation.py [--models vit,bert] [--rounds 3] [--out results/token_validation.json]

ViT_CIFAR10 on 10,000 images in batches of 100, BERT_AGNEWS on 2,000 samples in batches of 20 (synthetic samples with
the test splits' shapes, seeded weights).  Per model and path: wall time of whole passes (host clock around a pass that
ends in a device synchronise), alternating the two paths for ``--rounds`` rounds after one warm-up pass each, and the
device time of one extra pass (sum of kernel and copy times from ``torch.profiler``).  The card name and power limit are
read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.utils.data import DataLoader  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return q or torch.cuda.get_device_name(0)


def device_ms(fn) -> float:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        total += getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return total / 1e3


def setup(name, dev):
    from split_learning_b200.data import SyntheticDataset
    from split_learning_b200.data.gpu_loader import ResidentBatches
    from split_learning_b200.data.loaders import BatchedTensorLoader
    from split_learning_b200.models import BERT_AGNEWS, ViT_CIFAR10
    torch.manual_seed(0)
    if name == "vit":
        cls, ds = ViT_CIFAR10, SyntheticDataset("CIFAR10", [1000] * 10, seed=7)
        host = BatchedTensorLoader(ds, 100, shuffle=False)
        resident = ResidentBatches(ds.data, ds.labels, 100, dev)
    else:
        cls, ds = BERT_AGNEWS, SyntheticDataset("AGNEWS", [500] * 4, seed=7)
        host = DataLoader(ds, batch_size=20, shuffle=False)
        resident = ResidentBatches(ds.data, ds.labels, 20, dev)
    return cls, cls().state_dict(), host, resident


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="vit,bert")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_token_validation needs a CUDA device")
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    from split_learning_b200.validation import evaluate
    dev = torch.device("cuda:0")
    result = {"card": card(), "models": {}}
    for name in a.models.split(","):
        cls, sd, host, resident = setup(name, dev)
        model = cls()
        model.load_state_dict(sd)
        model.to(dev)
        native = NativeTokenEvaluator(cls, sd, dev)
        paths = {"torch_host_loader": lambda: evaluate(model, host, dev),
                 "native_resident": lambda: native.evaluate(resident)}
        metrics = {k: fn() for k, fn in paths.items()}                         # warm-up (native: eager pass + ...)
        metrics["native_resident"] = paths["native_resident"]()               # ... the pass that captures the graphs
        wall = {k: [] for k in paths}
        for _ in range(a.rounds):
            for k, fn in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                wall[k].append((time.perf_counter() - t0) * 1e3)
        row = {"samples": metrics["native_resident"]["val_total"]}
        for k, fn in paths.items():
            row[k] = {"wall_ms": [round(v, 2) for v in wall[k]], "wall_ms_median": round(statistics.median(wall[k]), 2),
                      "device_ms": round(device_ms(fn), 2), "val_loss": metrics[k]["val_loss"],
                      "val_correct": metrics[k]["val_correct"]}
        row["wall_speedup"] = round(row["torch_host_loader"]["wall_ms_median"] / row["native_resident"]["wall_ms_median"], 2)
        result["models"][name] = row
        print(json.dumps({name: row}), flush=True)
        del native, model
        torch.cuda.empty_cache()
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
