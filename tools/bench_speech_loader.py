"""KWT / Speech Commands input pipeline: the host loader (scipy read + NumPy MFCC per ``__getitem__``) against the
GPU-resident split of ``b200.gpu-loader`` (host reads once, ``mfcc_kernel`` once, one ``feature_batch`` gather per
microbatch).

    python tools/bench_speech_loader.py [--clips 3000] [--rounds 3] [--steps 90] [--recipe engine|reference] [--out FILE]

Writes a seeded tree of ``--clips`` one-second wav files to a temporary directory, then alternates, ``--rounds`` times:
  host_epoch_s      one epoch of ``data_loader(..., gpu_loader=False)`` at batch 32 (wall)
  resident_*        construction of the resident split: host file reads (wall), ``mfcc`` kernel time (CUDA events), total
  train_*_steps_s   KWT training steps per second at batch 32 (two stages cut at 8, native token blocks, CUDA graphs, built
                    by ``make_executor``), fed by each loader, wall clock over ``--steps`` full microbatches
  mfcc_*_kernel_ms  ``mfcc`` kernel time for the whole split in each MFCC recipe (engine: 400-sample window, 512-point
                    DFT; reference: 480 / 480), the same clips, alternating (CUDA events, one launch per 2048 clips)
The loaders and the resident split use ``--recipe`` (``b200.speech-features``).  Prints one JSON line with every round,
the medians, the card name and its power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from split_learning_b200.data import data_loader  # noqa: E402
from split_learning_b200.data.gpu_loader import GpuFeatureLoader  # noqa: E402
from split_learning_b200.data.loaders import SPEECH_CHUNK, speech_features  # noqa: E402
from split_learning_b200.data.gpu_loader import mfcc_features, mfcc_tables  # noqa: E402
from split_learning_b200.data.speechcommands import CLASSES, RECIPES, SAMPLE_RATE, SpeechCommandsDataset, clip_length, \
    read_wave  # noqa: E402
from split_learning_b200.models import get_model_class  # noqa: E402
from split_learning_b200.ops import native as N  # noqa: E402
from split_learning_b200.train.executor import make_executor  # noqa: E402

BATCH, CUT = 32, 8


def write_tree(root: str, clips: int, seed: int = 0) -> None:
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    base = os.path.join(root, "SpeechCommands", "speech_commands_v0.02")
    t = np.arange(SAMPLE_RATE) / SAMPLE_RATE
    for i in range(clips):
        c = CLASSES[i % len(CLASSES)]
        os.makedirs(os.path.join(base, c), exist_ok=True)
        f0 = 150.0 * (1 + i % len(CLASSES)) * rng.uniform(0.9, 1.1)
        wave = 8000 * np.sin(2 * np.pi * f0 * t) * np.hanning(SAMPLE_RATE) + rng.standard_normal(SAMPLE_RATE) * 500
        wavfile.write(os.path.join(base, c, f"{i:05d}.wav"), SAMPLE_RATE, wave.clip(-32768, 32767).astype(np.int16))


def card() -> dict:
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def executors(dev):
    cls = get_model_class("KWT", "SPEECHCOMMANDS")
    learning = {"learning-rate": 1e-3, "weight-decay": 0.01}
    opts = {"native-tokens": True, "token-graphs": True}
    torch.manual_seed(0)
    e1 = make_executor(cls(0, CUT), "KWT", learning, dev, True, False, opts)
    e2 = make_executor(cls(CUT, len(cls.LAYERS)), "KWT", learning, dev, False, True, opts)
    return e1, e2


def train_steps(e1, e2, loader, steps: int, dev) -> float:
    """Steps per second over ``steps`` full microbatches of ``loader`` (wall clock, ends in a device synchronise)."""
    done = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while done < steps:
        for x, y in loader:
            if x.shape[0] != BATCH:
                continue
            a = e1.forward_only(done, x)
            gx = e2.forward_backward_last(a, torch.as_tensor(y).to(dev, non_blocking=True))
            e1.backward(done, gx)
            done += 1
            if done == steps:
                break
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def staged_clips(paths, dev, recipe: str):
    """The clips of ``paths`` read, padded or truncated as the recipe does, and uploaded; with the recipe's tables."""
    L = clip_length(recipe)
    waves = torch.from_numpy(np.stack([np.pad(w, (0, max(0, L - w.size)))[:L] for w in
                                       (read_wave(p, recipe) for p in paths)])).to(dev)
    return recipe, waves, mfcc_tables(dev, recipe)


def mfcc_kernel_ms(staged, reps: int = 5) -> float:
    """Median over ``reps`` of the ``mfcc`` kernel time (CUDA events) for all staged clips, SPEECH_CHUNK per launch."""
    recipe, waves, tables = staged
    valid = torch.ones(waves.shape[0], dtype=torch.uint8, device=waves.device)
    out = torch.empty(waves.shape[0], 40, 98, device=waves.device)
    times = []
    for _ in range(reps + 1):                              # the first pass loads the module and is not counted
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for lo in range(0, waves.shape[0], SPEECH_CHUNK):
            hi = lo + SPEECH_CHUNK
            mfcc_features(waves[lo:hi], valid[lo:hi], tables, out=out[lo:hi], recipe=recipe)
        ev[1].record()
        ev[1].synchronize()
        times.append(ev[0].elapsed_time(ev[1]))
    return statistics.median(times[1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=90)
    ap.add_argument("--recipe", choices=RECIPES, default="engine")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speech_loader needs a CUDA device")
    N.require()
    N.preload()
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.clips)
        dist = [a.clips] * len(CLASSES)                      # the whole tree
        paths = [p for p, _ in SpeechCommandsDataset(root=root).samples]
        res = {"clips": len(paths), "batch": BATCH, "recipe": a.recipe, **card(), "rounds": []}
        e1, e2 = executors(dev)
        gpu = data_loader("SPEECHCOMMANDS", BATCH, dist, train=True, synthetic=False, root=root, device=dev, gpu_loader=True,
                          speech_features=a.recipe)
        assert isinstance(gpu, GpuFeatureLoader)
        train_steps(e1, e2, gpu, 3, dev)                     # graph capture, module loads
        staged = [staged_clips(paths, dev, recipe) for recipe in RECIPES]
        for _ in range(a.rounds):
            r = {}
            host = data_loader("SPEECHCOMMANDS", BATCH, dist, train=True, synthetic=False, root=root, speech_features=a.recipe)
            t0 = time.perf_counter()
            n = sum(int(x.shape[0]) for x, _ in host)
            r["host_epoch_s"] = time.perf_counter() - t0
            assert n == len(paths)
            timing = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            speech_features(paths, dev, timing=timing, recipe=a.recipe)
            torch.cuda.synchronize()
            r["resident_total_s"] = time.perf_counter() - t0
            r["resident_host_reads_s"] = timing["host_s"]
            r["resident_mfcc_kernel_ms"] = timing["mfcc_ms"]
            r["train_host_loader_steps_s"] = train_steps(e1, e2, host, a.steps, dev)
            r["train_gpu_loader_steps_s"] = train_steps(e1, e2, gpu, a.steps, dev)
            for st in staged:
                r[f"mfcc_{st[0]}_kernel_ms"] = mfcc_kernel_ms(st)
            res["rounds"].append({k: round(v, 4) for k, v in r.items()})
        res["median"] = {k: round(statistics.median(r[k] for r in res["rounds"]), 4) for k in res["rounds"][0]}
        res["loss"] = round(float(e2.last_loss()), 4)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
