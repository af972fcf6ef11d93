"""Reference arm of ``bench.py --impl reference``.

Runs the UNMODIFIED reference (verbatim copy in baseline/_ref, sha256-checked) through its
own public classes — ``src.Server.Server`` and ``src.RpcClient.RpcClient`` with the stock
``Train_VGG16`` loops, stock model, stock ``data_loader`` and SGD — on the same metric/config
as our arm: VGG16/CIFAR10 split at cut 7, batch 32, control-count 3, N GPUs =
``clients: [N/2, N/2]`` (N=1: both stages share the GPU).  What is substituted, and why:
  * ``pika``  → baseline/shims/pika (no RabbitMQ server in the image; same API, in-box broker);
  * ``peft``  → import-only stub (not installable offline; never called on the VGG16 path);
  * ``torchvision.datasets.CIFAR10`` → synthetic CIFAR-shaped images (no network/dataset).
No split_learning_b200 model, kernel or engine code is on this path.
Timing: a delivery hook in the shim timestamps the W-th and (W+K)-th gradient message reaching
each first-stage client (cuda-synchronised, CUDA events + host clock); value = total images of
the K steady-state steps / max time over first-stage ranks.
"""
from __future__ import annotations

import copy
import json
import os
import sys
import threading
import time
import uuid

HERE = os.path.dirname(os.path.abspath(__file__))


def _prepare_imports():
    from install_reference import install   # noqa: local module
    ref = install()
    man = json.load(open(os.path.join(ref, "MANIFEST.json")))
    if not all(v["matches_reference"] for v in man["files"].values()):
        raise RuntimeError("baseline/_ref differs from the reference tree")
    for p in (ref, os.path.join(HERE, "shims")):
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    import torchvision
    from fake_cifar import SyntheticCIFAR10
    torchvision.datasets.CIFAR10 = SyntheticCIFAR10
    return ref, man["outcome"]


def _config(n_first: int, n_last: int, batches: int):
    per_label = (batches * 32 + 9) // 10
    return {
        "name": "Split Learning",
        "server": {
            "global-round": 1, "clients": [n_first, n_last], "auto-mode": False, "model": "VGG16",
            "data-name": "CIFAR10", "parameters": {"load": False, "save": True}, "validation": False,
            "data-distribution": {"non-iid": False, "num-sample": per_label * 10, "num-label": 10,
                                  "dirichlet": {"alpha": 1}, "refresh": True},
            "random-seed": 1,
            "manual": {"cluster-mode": False, "no-cluster": {"cut-layers": [7]},
                       "cluster": {"num-cluster": 1, "cut-layers": [[7]], "infor-cluster": [[n_first, n_last]]}},
            "cluster-selection": {"num-cluster": 1, "algorithm-cluster": "KMeans", "selection-mode": False},
        },
        "rabbit": {"address": "127.0.0.1", "username": "admin", "password": "admin", "virtual-host": "/"},
        "log_path": "/tmp", "debug_mode": False,
        "learning": {"learning-rate": 0.0005, "weight-decay": 0.01, "momentum": 0.5, "batch-size": 32, "control-count": 3},
    }


PROFILE = {"exe_time": [1.0] * 52, "size_data": [1.0] * 52, "speed": 1.0, "network": 1.0}


def child_main(layer_id: int, port: int, W: int, K: int, out_path: str, device: str) -> None:
    """One reference client in its own OS process (how the reference is deployed: ``python client.py --layer_id N``)."""
    sys.path.insert(0, HERE)
    _prepare_imports()
    import torch
    import pika
    from src.RpcClient import RpcClient
    torch.cuda.set_device(torch.device(device))
    pika.use_remote("127.0.0.1", port)
    marks, counts = [], {"n": 0}

    def hook(queue, body):
        if not queue.startswith("gradient_queue_1_"):
            return
        counts["n"] += 1
        if counts["n"] in (W, W + K):
            torch.cuda.synchronize()
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((time.perf_counter(), ev))
    pika.on_get.append(hook)
    cid = uuid.uuid4()
    conn = pika.BlockingConnection(pika.ConnectionParameters("127.0.0.1"))
    c = RpcClient(cid, layer_id, conn.channel(), device)
    c.send_to_server({"action": "REGISTER", "client_id": cid, "layer_id": layer_id, "profile": PROFILE,
                      "cluster": -1, "message": "Hello from Client!"})
    c.wait_response()
    ms = 0.0
    if len(marks) == 2:
        torch.cuda.synchronize()
        ms = marks[0][1].elapsed_time(marks[1][1])
    with open(out_path, "w") as f:
        json.dump({"layer": layer_id, "ms": ms, "wall_ms": (marks[1][0] - marks[0][0]) * 1e3 if len(marks) == 2 else 0.0}, f)


def _single_box_processes(args, cfg, port: int, W: int, K: int, device: str = "cuda:0", host_server: bool = True) -> float:
    """One GPU's share of the ring / N = 1 deployment: (rank 0: server + broker here,) one subprocess per client — a
    first-stage and a last-stage client — both on ``device``."""
    import subprocess
    import tempfile
    import pika
    th = None
    if host_server:
        from src.Server import Server
        pika.serve("127.0.0.1", port)
        os.chdir("/tmp")

        def serve():
            try:
                Server(copy.deepcopy(cfg)).start()
            except SystemExit:
                pass
        th = threading.Thread(target=serve, daemon=True, name="ref-server")
        th.start()
    outs, procs = [], []
    for layer in (1, 2):
        out = tempfile.mktemp(prefix=f"ref_l{layer}_", suffix=".json")
        outs.append(out)
        log = open(out + ".log", "w")
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--child", str(layer), str(port), str(W), str(K),
                                       out, device], stdout=subprocess.DEVNULL, stderr=log))
    for p in procs:
        try:
            p.wait(args.timeout)
        except subprocess.TimeoutExpired:
            p.kill()
    if th is not None:
        th.join(60)
    ms = 0.0
    for o in outs:
        if os.path.exists(o):
            ms = max(ms, json.load(open(o))["ms"])
        elif os.path.exists(o + ".log"):
            tail = open(o + ".log").read().strip().splitlines()[-3:]
            sys.stderr.write("reference child failed: " + " | ".join(tail) + "\n")
    return ms


def main(args, transport: str = "broker") -> dict:
    """``transport``: "broker" = pickled NumPy through the in-box broker (what the reference does over RabbitMQ);
    "nccl" = the hot activation / gradient payloads over torch.distributed NCCL isend/recv (see shims/pika)."""
    impl = "reference" if transport == "broker" else "reference-nccl"
    sys.path.insert(0, HERE)
    try:
        ref, outcome = _prepare_imports()
    except Exception as e:  # noqa
        return {"impl": "reference", "unavailable": f"{type(e).__name__}: {e}"[:200]}
    import torch
    import pika                                  # the shim
    from src.RpcClient import RpcClient          # reference code
    from src.Server import Server                # reference code

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    n = args.gpus
    if world != max(n, 1) and not (n == 1 and world == 1):
        return {"impl": "reference", "unavailable": f"WORLD_SIZE {world} != --gpus {n}"}
    if not torch.cuda.is_available():
        return {"impl": "reference", "unavailable": "no CUDA device"}
    torch.cuda.set_device(local_rank)
    device = f"cuda:{local_rank}"
    W, K = args.warmup, args.steps
    ring = transport == "broker" and getattr(args, "placement", "ring") == "ring" and n > 1
    if ring:                                     # same deployment as our arm: N chains, 2 clients (stage 1 + stage 2) per GPU
        n_first = n_last = n
    else:
        n_first = max(1, n // 2)
        n_last = max(1, n - n_first) if n > 1 else 1
    batches = W + K + 4
    cfg = _config(n_first, n_last, batches)
    port = 29655 + (int(os.environ.get("MASTER_PORT", "0")) % 97)

    if transport == "nccl" and world < 2:
        return {"impl": impl, "unavailable": "NCCL p2p needs one rank per client (>= 2 GPUs); N=1 puts both clients on one GPU"}
    if world == 1:
        t_wall = time.perf_counter()
        ms_total = _single_box_processes(args, cfg, port, W, K)
        if ms_total <= 0:
            return {"impl": "reference", "unavailable": "timing marks missing (single-box process mode)"}
        return _result(n, n_first, n_last, K, W, ms_total, outcome, time.perf_counter() - t_wall,
                       "one OS process per client (both on cuda:0) + server/broker process")
    if ring:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device(device))
        t_wall = time.perf_counter()
        ms_local = _single_box_processes(args, cfg, port, W, K, device=device, host_server=(rank == 0))
        t = torch.tensor([ms_local], device=device)
        bad = torch.tensor([float(ms_local <= 0)], device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX)
        dist.barrier()
        dist.destroy_process_group()
        if rank != 0:
            return {}
        if float(bad.item()) > 0:
            return {"impl": "reference", "unavailable": "timing marks missing on some rank (ring deployment)"}
        res = _result(n, n_first, n_last, K, W, float(t.item()), outcome, time.perf_counter() - t_wall,
                      "ring: one first-stage and one last-stage client process per GPU (+ server/broker on rank 0)")
        res["config"]["placement"] = "ring"
        return res
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device(device))
        if rank == 0:
            pika.serve("127.0.0.1", port)
        dist.barrier()
        pika.use_remote("127.0.0.1", port)
        if transport == "nccl":
            pika.use_nccl(rank, n_first, n_last, device)
            warm = torch.zeros(8, device=device)             # communicator setup outside the timed region
            dist.all_reduce(warm)
            torch.cuda.synchronize()

    # ---- delivery hook: time K steps between the W-th and (W+K)-th gradient delivery --------
    marks = {}
    counts = {}
    lock = threading.Lock()

    def hook(queue, body):
        if not queue.startswith("gradient_queue_1_"):
            return
        with lock:
            c = counts[queue] = counts.get(queue, 0) + 1
        if c == W or c == W + K:
            torch.cuda.synchronize()
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.setdefault(queue, []).append((time.perf_counter(), ev))
    pika.on_get.append(hook)

    threads = []
    if rank == 0:
        os.chdir("/tmp")                         # the reference writes app.log / *.pth into the CWD

        def serve():
            try:
                Server(copy.deepcopy(cfg)).start()
            except SystemExit:
                pass
        threads.append(threading.Thread(target=serve, daemon=True, name="ref-server"))

    def client(layer_id):
        cid = uuid.uuid4()
        conn = pika.BlockingConnection(pika.ConnectionParameters("127.0.0.1"))
        c = RpcClient(cid, layer_id, conn.channel(), device)
        c.send_to_server({"action": "REGISTER", "client_id": cid, "layer_id": layer_id, "profile": PROFILE,
                          "cluster": -1, "message": "Hello from Client!"})
        c.wait_response()

    if world == 1:
        roles = [1, 2]
    else:
        roles = [1 if rank < n_first else 2]
    for layer in roles:
        threads.append(threading.Thread(target=client, args=(layer,), daemon=True, name=f"ref-client-l{layer}"))
    t_wall = time.perf_counter()
    for t in threads:
        t.start()
    for t in threads:
        t.join(args.timeout)
    if any(t.is_alive() for t in threads):
        return {"impl": "reference", "unavailable": "reference run timed out"}

    # ---- reduce ------------------------------------------------------------------------------
    ms = 0.0
    for q, m in marks.items():
        if len(m) == 2:
            torch.cuda.synchronize()
            ms = max(ms, m[0][1].elapsed_time(m[1][1]), 0.0)
    t = torch.tensor([ms], device=device)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.barrier()
    ms_total = float(t.item())
    if dist is not None:
        dist.destroy_process_group()
    if rank != 0:
        return {}
    if ms_total <= 0:
        return {"impl": "reference", "unavailable": "timing marks missing"}
    res = _result(n, n_first, n_last, K, W, ms_total, outcome, time.perf_counter() - t_wall, "one OS process (rank) per client")
    if transport == "nccl":
        res["impl"] = impl
        res["config"]["transport"] = ("torch.distributed NCCL isend/recv for intermediate_queue_* / gradient_queue_* payloads "
                                      "(header + control verbs on the in-box broker); reference trainers unmodified")
        res["nccl"] = pika.nccl_stats()
    return res


def _result(n, n_first, n_last, K, W, ms_total, outcome, wall, deployment) -> dict:
    images = n_first * K * 32
    value = images / (ms_total / 1e3)
    return {
        "impl": "reference", "metric": "VGG16/CIFAR10 split images/sec", "value": value, "unit": "images/s",
        "n_gpus": n, "steps": K, "warmup": W, "ms_per_step": ms_total / K, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "fp32 (cuDNN TF32 convs, torch defaults)", "data": "synthetic",
        "config": {"model": "VGG16_CIFAR10", "global_batch": 32 * n_first, "microbatch": 32, "cut_layers": [7],
                   "clients": [n_first, n_last], "control_count": 3, "parallelism": f"pp2 x dp{n_first}",
                   "transport": "in-box broker (pika shim) + pickle, as the reference does over RabbitMQ",
                   "l2": "inputs stream through host pickling each step", "install": outcome, "deployment": deployment},
        "e2e": {"value": value, "unit": "images/s", "h2d_bytes_per_step": 32 * 3 * 32 * 32 * 4 + 32 * 64 * 16 * 16 * 4 * 2,
                "d2h_bytes_per_step": 32 * 64 * 16 * 16 * 4 * 2},
        "gpu_launches": None, "wall_seconds": wall,
    }


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "--child":
    child_main(int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sys.argv[6], sys.argv[7])
