"""Training throughput of VGG16_MNIST split at layer 7, batch 32: the native program (``make_executor`` -> cnn_native,
whole-step CUDA graphs) against the stock torch modules (``b200.executor: torch``).

    python tools/bench_vgg_mnist.py [--steps 200] [--warmup 30] [--rounds 3] [--out DIR]

Each round times both arms over ``--steps`` steps with CUDA events after ``--warmup`` untimed steps, arms alternating;
prints one JSON line per arm and round, then a summary with the card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def _executors(native: bool, learning):
    from split_learning_b200.models import VGG16_MNIST
    from split_learning_b200.train.executor import make_executor
    opts = None if native else {"executor": "torch"}
    torch.manual_seed(0)
    e1 = make_executor(VGG16_MNIST(0, 7), "VGG16", learning, "cuda", True, False, opts)
    e2 = make_executor(VGG16_MNIST(7, 51), "VGG16", learning, "cuda", False, True, opts)
    assert bool(getattr(e1, "native", False)) == native and bool(getattr(e2, "native", False)) == native
    return e1, e2


def _time(arm, data, steps, warmup):
    e1, e2 = arm
    n = len(data)

    def step(it):
        x, y = data[it % n]
        a = e1.forward_only(it, x)
        gx = e2.forward_backward_last(a, y)
        e1.backward(it, gx)

    for it in range(warmup):
        step(it)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for it in range(warmup, warmup + steps):
        step(it)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory for a JSON copy of the results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vgg_mnist: no CUDA device")
    from split_learning_b200.ops import native as N
    N.require()
    N.preload()
    learning = {"learning-rate": 0.01, "momentum": 0.5}
    g = torch.Generator().manual_seed(1)
    data = [(torch.randn(args.batch, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (args.batch,), generator=g))
            for _ in range(8)]
    arms = {"native": _executors(True, learning), "torch": _executors(False, learning)}
    rates = {k: [] for k in arms}
    for r in range(args.rounds):
        for name, arm in arms.items():
            sec = _time(arm, data, args.steps, args.warmup if r == 0 else 5)
            ips = args.steps * args.batch / sec
            rates[name].append(ips)
            print(json.dumps({"round": r, "arm": name, "seconds": round(sec, 4), "images_per_s": round(ips, 1)}), flush=True)
    card, limits = _card()
    summary = {"model": "VGG16_MNIST", "cut": 7, "batch": args.batch, "steps": args.steps, "card": card,
               "power_limit_and_max_sm_clock": limits,
               "median_images_per_s": {k: round(statistics.median(v), 1) for k, v in rates.items()},
               "all_images_per_s": {k: [round(x, 1) for x in v] for k, v in rates.items()}}
    summary["native_over_torch"] = round(summary["median_images_per_s"]["native"] / summary["median_images_per_s"]["torch"], 3)
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_vgg_mnist.json"), "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
