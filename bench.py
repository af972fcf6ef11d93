#!/usr/bin/env python
"""Headline benchmark: VGG16/CIFAR10 split-learning throughput (images/s) on N H100s.

    python bench.py --gpus N --steps K --warmup W            # this framework
    python bench.py --impl reference --gpus N ...            # unmodified reference (baseline/_ref)

Config (BASELINE.json): VGG16_CIFAR10 cut at layer 7, microbatch 32, control-count 3,
SGD(lr 5e-4, momentum 0.5); N = 1 → both stages on one GPU, N = 2 → one GPU per stage,
N = 4/8 → N/2 replicas per stage (independent 1:1 chains, FedAvg at round end, outside the
timed steps as in the reference).  Weak scaling: every first-stage replica processes its own
32-image microbatches.  Synthetic CIFAR-10-shaped data (seeded: identical inputs from run to run),
random-init weights, tf32 tensor-core convolutions with fp32 accumulation (``--precision bf16``:
bf16 activations with fp32 master weights).

Timing: W warm-up steps, then exactly K steps between barrier + cuda synchronize, CUDA events
on the launching stream, max over ranks.  ``value`` = device-resident inputs (kernel pipeline
only); ``e2e`` = same K steps through ``LocalPipeline.run`` / the stage runner with a pinned
host→device copy of every microbatch and a device→host read of every step's loss.
The per-step working set (fp32 master + momentum + gradient + bf16 shadow ≈ 470 MB/stage-2
replica) exceeds the 50 MB L2, so no explicit L2 flush is needed between iterations.

``--dump-outputs DIR`` (N = 1): after the timed steps, write what the last timed step computed as
DIR/<name>.npy (float32): the loss, the activation that crossed each cut and the gradient that came
back (NCHW), and a fixed seeded sample of every stage's updated fp32 parameters.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference-nccl"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--depth", type=int, default=3, help="control-count (microbatches in flight)")
    ap.add_argument("--cut", type=int, default=7)
    ap.add_argument("--cuts", default=None, help="N=1 only: comma list for an N-stage pipeline on one GPU, e.g. 5,10")
    ap.add_argument("--precision", default="tf32", choices=["tf32", "bf16"],
                    help="tf32 (default) = the reference's precision: fp32 tensors, wgmma tf32 convolutions with fp32 "
                         "accumulation, fp32 Linear/BN/SGD; bf16 = opt-in fast mode")
    ap.add_argument("--placement", default="ring", choices=["ring", "split"],
                    help="N > 1: ring = N chains, GPU r hosts stage 1 of chain r and stage 2 of chain r-1 (default; per-GPU work "
                         "constant in N); split = clients [N/2, N/2], one stage replica per GPU (BASELINE configs #2/#3)")
    ap.add_argument("--scenario", default=None, choices=["split", "clusters", "three-stage"],
                    help="run ONLY the public-API path on a named BASELINE.json configuration, one client per GPU: split = [N/2, N/2] "
                         "cut 7 (#2/#3), clusters = two clusters cut 7 / 14 (#4), three-stage = cuts [5, 10], non-IID 0.5 (#5)")
    ap.add_argument("--no-api", action="store_true", help="skip the run through the public API (server + client FSMs over the broker)")
    ap.add_argument("--rounds", type=int, default=4, help="public-API run: global rounds (the first one pays graph capture and wiring)")
    ap.add_argument("--no-selfcheck", action="store_true", help="skip the cross-GPU vs single-GPU loss-trajectory check")
    ap.add_argument("--no-graphs", action="store_true")
    ap.add_argument("--timeout", type=float, default=1500.0)
    ap.add_argument("--breakdown", action="store_true", help="also report device time per stage program (F / L / B)")
    ap.add_argument("--no-overlap", action="store_true", help="N=1: run both stages on one stream")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="N=1: write the outputs of the last timed step to DIR/<name>.npy (compare two builds output for output)")
    args = ap.parse_args()
    if args.dump_outputs and (args.gpus > 1 or args.scenario or args.impl != "ours"):
        ap.error("--dump-outputs is supported for --gpus 1 --impl ours without --scenario")
    return args


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int = 0):
        self.rows = []
        self.proc = None
        self.gpu = gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.gpu)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append((time.perf_counter(), line.strip()))

    def stop(self, t0: float, t1: float) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        rows = [r for (t, r) in self.rows if t0 <= t <= t1] or [r for (_, r) in self.rows[-3:]]
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            f = [x.strip() for x in r.split(",")]
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
                for n, v in zip(names, f[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except (ValueError, IndexError):
                pass
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


DTYPE_LABEL = {
    "tf32": "fp32 tensors; conv = wgmma tf32 with fp32 accumulate (the reference's cuDNN-TF32 default), "
            "Linear/BN/CE/SGD = fp32",
    "bf16": "bf16 activations + bf16 weight shadow, fp32 master/accumulate (opt-in fast mode)",
}


def synthetic_batches(n: int, batch: int, seed: int):
    import torch
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = torch.randn(batch, 3, 32, 32, generator=g).pin_memory()
        y = torch.randint(0, 10, (batch,), generator=g).pin_memory()
        out.append((x, y))
    return out


PARAM_SAMPLE = 1 << 21          # parameters per stage in a --dump-outputs sample (8 MB of float32)


def dump_outputs(out_dir: str, pipe, exs, last_it: int) -> None:
    """What the last timed step (microbatch ``last_it``) handed back to the caller of the pipeline, as float32 .npy files."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    path = lambda name: os.path.join(out_dir, name + ".npy")
    slot = last_it % pipe.depth
    np.save(path("loss"), pipe.loss()[:1].float().cpu().numpy())
    for i, st in enumerate(pipe.stages[:-1]):
        np.save(path(f"cut{i}_activation"), st.fwd_out.payload[slot].float().permute(0, 3, 1, 2).cpu().numpy())
        np.save(path(f"cut{i}_gradient"), st.grad_in.payload[slot].float().permute(0, 3, 1, 2).cpu().numpy())
    rng = np.random.default_rng(0)
    for i, ex in enumerate(exs):
        n = ex.P.numel()
        idx = np.sort(rng.choice(n, min(n, PARAM_SAMPLE), replace=False))
        np.save(path(f"stage{i}_params_sample"), ex.P[torch.from_numpy(idx).to(ex.P.device)].float().cpu().numpy())


def run_ours(args) -> dict:
    import torch
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 or world > 1:
        from split_learning_b200.parallel.runner import bench_multi_gpu
        return bench_multi_gpu(args)
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.ops import native as N
    from split_learning_b200.parallel.pipeline import LocalPipeline
    from split_learning_b200.train.b200_executor import B200Executor

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    learning = {"learning-rate": 0.0005, "momentum": 0.5, "batch-size": args.batch, "control-count": args.depth,
                "precision": args.precision}
    W, K, B = args.warmup, args.steps, args.batch
    cuts = [int(c) for c in args.cuts.split(",")] if args.cuts else [args.cut]
    bounds = [0] + cuts + [52]
    exs = [B200Executor(VGG16_CIFAR10(bounds[i], bounds[i + 1]), "VGG16", learning, dev, is_first=(i == 0),
                        is_last=(i == len(bounds) - 2), use_graphs=not args.no_graphs) for i in range(len(bounds) - 1)]
    pipe = LocalPipeline(exs, B, args.depth, overlap=not (args.no_overlap or args.breakdown))
    pool = synthetic_batches(16, B, seed=1)
    loss_host = torch.zeros(4).pin_memory()

    def batches(n):
        for i in range(n):
            yield pool[i % len(pool)]

    # setup (graph capture for every slot) + W warm-up steps through the public API
    pipe.run(batches(2 * args.depth + 2))
    pipe.synchronize()
    pipe.run(batches(W))
    pipe.synchronize()

    sampler = ClockSampler(0)
    sampler.start()
    time.sleep(0.3)
    # ---- (1) kernel pipeline only: inputs already resident in the device slots --------------
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = N.LAUNCHES
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.cuda.stream(pipe.stream):
        e0.record()
    for _ in range(K):
        if pipe.it_f - pipe.it_b >= pipe.depth:
            pipe.step_backward()
        pipe.step_forward()
    while pipe.it_b < pipe.it_f:
        pipe.step_backward()
    pipe.join()
    with torch.cuda.stream(pipe.stream):
        e1.record()
    torch.cuda.synchronize()
    ms_dev = e0.elapsed_time(e1)
    per_step = sum(st.launches_per.get(k, 0) for st in pipe.stages for k in ("F", "B", "L"))
    # ---- (2) end to end: pinned H2D of every microbatch + D2H of every loss -----------------
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    with torch.cuda.stream(pipe.stream):
        f0.record()
    n = 0
    for x, y in batches(K):
        if pipe.it_f - pipe.it_b >= pipe.depth:
            pipe.step_backward()
        pipe.feed(x, y)
        pipe.step_forward()
        with torch.cuda.stream(pipe.loss_stream):
            loss_host.copy_(pipe.loss(), non_blocking=True)
        n += 1
    while pipe.it_b < pipe.it_f:
        pipe.step_backward()
    pipe.join()
    with torch.cuda.stream(pipe.stream):
        f1.record()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    ms_e2e = f0.elapsed_time(f1)
    clocks = sampler.stop(t0, t1)
    pipe.synchronize()
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, pipe, exs, pipe.it_f - 1)
    breakdown = None
    if args.breakdown:
        evs = []
        for _ in range(50):
            if pipe.it_f - pipe.it_b >= pipe.depth:
                a = torch.cuda.Event(enable_timing=True); a.record(pipe.stream)
                pipe.step_backward()
                b = torch.cuda.Event(enable_timing=True); b.record(pipe.stream)
                evs.append(("B", a, b))
            it = pipe.it_f
            a = torch.cuda.Event(enable_timing=True); a.record(pipe.stream)
            pipe.stages[0].forward(it)
            b = torch.cuda.Event(enable_timing=True); b.record(pipe.stream)
            pipe.stages[-1].last(it)
            c = torch.cuda.Event(enable_timing=True); c.record(pipe.stream)
            pipe.it_f += 1
            evs += [("F", a, b), ("L", b, c)]
        while pipe.it_b < pipe.it_f:
            pipe.step_backward()
        torch.cuda.synchronize()
        acc = {}
        for k, a, b in evs:
            acc.setdefault(k, []).append(a.elapsed_time(b) * 1e3)
        breakdown = {k: {"us": sum(v) / len(v), "launches": (pipe.stages[0] if k != "L" else pipe.stages[-1]).launches_per.get(k)}
                     for k, v in acc.items()}
    loss = float(loss_host[0])
    value = K * B / (ms_dev / 1e3)
    return {
        "metric": "VGG16/CIFAR10 split images/sec", "value": value, "unit": "images/s", "n_gpus": 1, "steps": K, "warmup": W,
        "ms_per_step": ms_dev / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": DTYPE_LABEL[args.precision],
        "data": "synthetic",
        "config": {"model": "VGG16_CIFAR10", "global_batch": B, "microbatch": B, "seq_len": None, "cut_layers": cuts,
                   "clients": [1] * (len(cuts) + 1), "control_count": args.depth,
                   "parallelism": f"pp{len(cuts) + 1} (all stages on one GPU, one stream per stage)",
                   "optimizer": "SGD lr=5e-4 momentum=0.5, step per microbatch", "recompute": True,
                   "cuda_graphs": not args.no_graphs,
                   "l2": "per-step working set ~470 MB (fp32 master+momentum+grad+bf16 shadow) > 50 MB L2; no flush needed"},
        "e2e": {"value": K * B / (ms_e2e / 1e3), "unit": "images/s", "ms_per_step": ms_e2e / K,
                "h2d_bytes_per_step": B * 3 * 32 * 32 * 4 + B * 8, "d2h_bytes_per_step": 16},
        "gpu_launches": per_step * K, "launches_per_step": per_step, "clocks": clocks, "final_loss": loss, "impl": "ours",
        **({"breakdown": breakdown} if breakdown else {}),
    }


def main():
    args = parse()
    if args.impl in ("reference", "reference-nccl"):
        sys.path.insert(0, os.path.join(ROOT, "baseline"))
        from run_reference import main as ref_main
        out = ref_main(args, transport="nccl" if args.impl == "reference-nccl" else "broker")
    elif args.scenario:
        from split_learning_b200.parallel.api_bench import run_api
        sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0")))
        sampler.start()
        t0 = time.perf_counter()
        api = run_api(args)
        clocks = sampler.stop(t0, time.perf_counter())
        out = None
        if api:
            r = api.get("steady_round") or {}
            out = {"metric": "VGG16/CIFAR10 split images/sec", "value": r.get("images_per_s_device"), "unit": "images/s",
                   "n_gpus": args.gpus, "steps": api.get("microbatches_per_client_per_round"), "warmup": 0,
                   "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": DTYPE_LABEL[args.precision],
                   "data": "synthetic", "impl": "ours", "measured_through": "public API (server + clients over the broker)",
                   "config": {"model": "VGG16_CIFAR10", "scenario": args.scenario, "clients": api.get("clients"),
                              "cut_layers": api.get("cut_layers"), "non_iid_rate": api.get("non_iid_rate"), "microbatch": args.batch,
                              "control_count": args.depth},
                   "e2e": {"value": r.get("images_per_s_device"), "round_wall_ms": r.get("wall_ms"),
                           "round_overhead_ms": r.get("overhead_ms"), "images_per_s_whole_round": r.get("images_per_s_round")},
                   "clocks": clocks, "api": api}
    else:
        out = run_ours(args)
        if not args.no_api and not args.cuts and (args.gpus == 1 or args.placement == "ring"):
            # the same metric end to end through the public API (what a user runs): server + client FSMs over the broker,
            # pinned-host inputs copied in every step, every step's loss copied out, FedAvg + UPDATE at round end
            from split_learning_b200.parallel.api_bench import run_api
            try:
                api = run_api(args)
            except Exception as e:              # the kernel-pipeline numbers above stand on their own
                api = {"error": f"{type(e).__name__}: {e}"[:300]}
            if out and api and "steady_round" in api:
                r = api["steady_round"]
                out["e2e_pipeline_loop"] = out.get("e2e")
                out["e2e"] = {"value": r["images_per_s_device"], "unit": "images/s", "path": api["path"],
                              "ms_per_step": r["device_ms"] / api["microbatches_per_client_per_round"],
                              "h2d_bytes_per_step": api["h2d_bytes_per_step"], "d2h_bytes_per_step": api["d2h_bytes_per_step"],
                              "steps_per_round": api["microbatches_per_client_per_round"], "rounds": len(api.get("rounds", [])),
                              "round_wall_ms": r["wall_ms"], "round_overhead_ms": r["overhead_ms"],
                              "images_per_s_whole_round": r["images_per_s_round"], "train_loss": r["train_loss"]}
                out["api"] = api
            elif out is not None and api:
                out["api"] = api
    if out and int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps(out), flush=True)
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()
    except Exception:
        pass


if __name__ == "__main__":
    main()
