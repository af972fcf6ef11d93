"""Cost of server-side validation of VGG16/CIFAR10: 10,000 seeded CIFAR-shaped uint8 test images evaluated three ways.

  torch_host      ``validation.evaluate`` fed by the host recipe (PIL -> ToTensor -> Normalize in a one-worker
                  ``DataLoader``, batch 100): wall time
  torch_resident  the same torch modules on inputs already normalised on the GPU (cuDNN TF32 convolutions, fp32 Linear):
                  device time (CUDA events, no host sync inside the loop)
  native          ``NativeEvaluator`` on the resident uint8 split (one normalise kernel + one graph replay per batch):
                  device time of ``evaluate``, and wall time of ``load_state_dict`` + ``evaluate``

Prints one JSON object (images/s and ms per way, the card, its clocks and power limit); ``--out`` also writes it.

    python tools/bench_validation.py [--images 10000] [--repeats 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def _card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["clock_max_sm"], info["clock_sm_at_start"] = [s.strip() for s in q.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError):
        info["nvidia_smi"] = "unavailable"
    return info


class _HostSplit(torch.utils.data.Dataset):
    """uint8 HWC images through the reference's test transform (PIL -> ToTensor -> Normalize)."""

    def __init__(self, images, labels):
        import torchvision.transforms as T
        from split_learning_b200.data.gpu_loader import CIFAR_MEAN, CIFAR_STD
        self.images, self.labels = images.numpy(), labels
        self.tf = T.Compose([T.ToTensor(), T.Normalize(CIFAR_MEAN, CIFAR_STD)])

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, i):
        from PIL import Image
        return self.tf(Image.fromarray(self.images[i])), int(self.labels[i])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validation needs a CUDA device")
    from split_learning_b200.data.gpu_loader import CIFAR_MEAN, CIFAR_STD, GpuImageLoader
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.train.b200_eval import NativeEvaluator
    from split_learning_b200.validation import evaluate
    dev = torch.device("cuda:0")
    n = a.images
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (n, 32, 32, 3), generator=g, dtype=torch.uint8)
    labels = torch.randint(0, 10, (n,), generator=g)
    torch.manual_seed(0)
    model = VGG16_CIFAR10()
    sd = model.state_dict()
    model = model.to(dev).eval()
    res = {"card": _card(), "images": n, "batch": 100, "repeats": a.repeats}

    # 1. torch, host DataLoader recipe (wall; evaluate() syncs per batch through float(loss))
    loader = torch.utils.data.DataLoader(_HostSplit(images, labels), batch_size=100, shuffle=False, num_workers=1)
    t0 = time.perf_counter()
    m_host = evaluate(model, loader, dev)
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) * 1e3
    res["torch_host"] = {"wall_ms": host_ms, "images_per_s": n / host_ms * 1e3, "val_loss": m_host["val_loss"],
                         "val_correct": m_host["val_correct"]}

    # 2. torch on GPU-normalised inputs (device time)
    src = GpuImageLoader(images, labels, 100, dev, CIFAR_MEAN, CIFAR_STD, augment=False, shuffle=False)
    xs = [(x.clone(), y.clone()) for x, y in src]

    def torch_pass():
        loss = torch.zeros((), device=dev, dtype=torch.float64)
        correct = torch.zeros((), device=dev, dtype=torch.int64)
        with torch.no_grad():
            for x, y in xs:
                out = model(x)
                loss += F.cross_entropy(out, y).double()
                correct += (out.argmax(1) == y).sum()
        return loss, correct

    torch_pass()
    times = []
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loss_t, correct_t = torch_pass()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = statistics.median(times)
    res["torch_resident"] = {"device_ms": ms, "images_per_s": n / ms * 1e3, "device_ms_all": times,
                             "val_loss": float(loss_t) / len(xs), "val_correct": int(correct_t)}

    # 3. native evaluator on the resident uint8 split
    ev = NativeEvaluator(VGG16_CIFAR10, sd, dev)
    ev.evaluate(src)
    ev.evaluate(src)                       # first pass eager, second captures the graphs
    dev_times, wall_times = [], []
    for _ in range(a.repeats):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        ev.load_state_dict(sd)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ev.ex.stream)
        m_nat = ev.evaluate(src)
        e1.record(ev.ex.stream)
        e1.synchronize()
        wall_times.append((time.perf_counter() - t0) * 1e3)
        dev_times.append(e0.elapsed_time(e1))
    ms, wall = statistics.median(dev_times), statistics.median(wall_times)
    res["native"] = {"device_ms": ms, "images_per_s": n / ms * 1e3, "device_ms_all": dev_times,
                     "wall_ms_with_load_state_dict": wall, "wall_ms_all": wall_times,
                     "val_loss": m_nat["val_loss"], "val_correct": m_nat["val_correct"]}
    res["native_vs_torch_resident_speedup"] = res["torch_resident"]["device_ms"] / ms
    res["native_wall_vs_torch_host_speedup"] = host_ms / wall
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
