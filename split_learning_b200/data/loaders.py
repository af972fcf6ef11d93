"""Data loaders.

Real datasets follow the reference's recipes (src/dataset/dataloader.py):
  * CIFAR10  — RandomCrop(32, pad 4) + HFlip + Normalize; per-label ``random.sample`` of
    ``distribution[label]`` indices; shuffle; test batch 100  (:61-92)
  * MNIST    — ToTensor + Normalize (variants)
  * AGNEWS   — CSV + BertTokenizer('bert-base-cased'), max_len 128  (:16-59)
  * SPEECHCOMMANDS — 10-class subset, NumPy MFCC 40x98  (:95-122)
They need files under ``./data`` (no network here).  When the files are missing, or
``synthetic=True`` / ``SLB200_SYNTHETIC=1``, a ``SyntheticDataset`` with the same tensor
shapes, dtypes and per-label counts is used instead (what ``bench.py`` uses).
"""
from __future__ import annotations

import os
import random
from collections import defaultdict
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch.utils.data import DataLoader, Dataset, Subset

# name -> (sample shape, dtype, num classes, test batch size)
DATASET_SHAPES: Dict[str, Tuple[Tuple[int, ...], torch.dtype, int, int]] = {
    "CIFAR10": ((3, 32, 32), torch.float32, 10, 100),
    "MNIST": ((1, 28, 28), torch.float32, 10, 100),
    "AGNEWS": ((128,), torch.long, 4, 20),
    "EMOTION": ((128,), torch.long, 6, 20),
    "SPEECHCOMMANDS": ((40, 98), torch.float32, 10, 20),
}


class SyntheticDataset(Dataset):
    """Deterministic random samples with exact per-label counts.  Samples are generated once
    into a pinned-able tensor (class-dependent mean so that a model can actually learn)."""

    def __init__(self, data_name: str, distribution: Sequence[int], seed: int = 0, vocab: int = 28996):
        shape, dtype, ncls, _ = DATASET_SHAPES[data_name.upper()]
        labels: List[int] = []
        for lbl, cnt in enumerate(distribution):
            labels += [lbl % ncls] * int(cnt)
        g = torch.Generator().manual_seed(seed)
        n = len(labels)
        self.labels = torch.tensor(labels, dtype=torch.long)
        if dtype == torch.long:
            self.data = torch.randint(1, vocab, (n,) + shape, generator=g)
            self.data[:, 0] = 101
            self.data[:, 1] = 1000 + self.labels          # a learnable signal
        else:
            self.data = torch.randn((n,) + shape, generator=g)
            self.data += (self.labels.float().view(-1, *([1] * len(shape))) - (ncls - 1) / 2) * 0.25
        self.as_dict = dtype == torch.long

    def __len__(self):
        return self.labels.numel()

    def __getitem__(self, i):
        if self.as_dict:
            return {"input_ids": self.data[i], "attention_mask": torch.ones_like(self.data[i]),
                    "labels": self.labels[i]}
        return self.data[i], self.labels[i]


class BatchedTensorLoader:
    """Loader for a dataset that is already a pair of in-memory tensors: one ``index_select`` per microbatch straight into a
    page-locked staging slot instead of ``batch_size`` ``__getitem__`` calls + ``default_collate`` (≈0.3 ms per CIFAR
    microbatch with ``torch.utils.data.DataLoader``, comparable to the whole device time of a first-stage step).
    Same iteration contract as ``DataLoader(ds, batch_size, shuffle, drop_last=False)``: a fresh permutation per epoch, the
    short batch last.  ``pin=True`` yields pinned slots, one per microbatch of an epoch (epochs of up to
    ``MAX_PINNED_BATCHES`` microbatches; longer ones yield pageable tensors) — a slot is rewritten one epoch later, after the
    consumer's H2D copies of the previous epoch have completed."""

    MAX_PINNED_BATCHES = 512          # beyond this the consumer stages through its own bounded pinned ring instead

    def __init__(self, dataset, batch_size: int, shuffle: bool = True, pin: bool = False, seed: int = 0):
        self.dataset, self.batch_size, self.shuffle = dataset, int(batch_size), shuffle
        self.pin = bool(pin) and (len(dataset) + int(batch_size) - 1) // int(batch_size) <= self.MAX_PINNED_BATCHES
        self.drop_last = False
        self._gen = torch.Generator().manual_seed(seed + 1)
        self._slots: dict = {}

    def __len__(self):
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def _slot(self, i: int, b: int):
        if not self.pin:
            return None, None
        key = (i, b)
        if key not in self._slots:
            d, l = self.dataset.data, self.dataset.labels
            try:
                self._slots[key] = (torch.empty((b,) + tuple(d.shape[1:]), dtype=d.dtype).pin_memory(),
                                    torch.empty((b,), dtype=l.dtype).pin_memory())
            except RuntimeError:              # no CUDA runtime to page-lock with
                self.pin = False
                return None, None
        return self._slots[key]

    def __iter__(self):
        n, B = len(self.dataset), self.batch_size
        order = torch.randperm(n, generator=self._gen) if self.shuffle else torch.arange(n)
        for i, lo in enumerate(range(0, n, B)):
            idx = order[lo: lo + B]
            ox, oy = self._slot(i, idx.numel())
            if ox is None:
                yield self.dataset.data.index_select(0, idx), self.dataset.labels.index_select(0, idx)
            else:
                torch.index_select(self.dataset.data, 0, idx, out=ox)
                torch.index_select(self.dataset.labels, 0, idx, out=oy)
                yield ox, oy


def synthetic_loader(data_name: str, batch_size: int, distribution: Sequence[int], train: bool = True,
                     seed: int = 0, pin: bool = False):
    ds = SyntheticDataset(data_name, distribution, seed=seed)
    if not ds.as_dict:
        return BatchedTensorLoader(ds, batch_size, shuffle=train, pin=pin, seed=seed)
    return DataLoader(ds, batch_size=batch_size, shuffle=train, drop_last=False)


def _select_by_label(labels: Sequence[int], distribution: Sequence[int]) -> List[int]:
    by_label = defaultdict(list)
    for idx, l in enumerate(labels):
        by_label[int(l)].append(idx)
    picked: List[int] = []
    for label, count in enumerate(distribution):
        pool = by_label.get(label, [])
        picked.extend(random.sample(pool, min(int(count), len(pool))))
    return picked


def _cifar10(batch_size, distribution, train, root="./data"):
    import torchvision
    import torchvision.transforms as T
    norm = T.Normalize((0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010))
    if train:
        tf = T.Compose([T.RandomCrop(32, padding=4), T.RandomHorizontalFlip(), T.ToTensor(), norm])
        ds = torchvision.datasets.CIFAR10(root=root, train=True, download=False, transform=tf)
        return DataLoader(Subset(ds, _select_by_label(ds.targets, distribution)), batch_size=batch_size, shuffle=True)
    ds = torchvision.datasets.CIFAR10(root=root, train=False, download=False, transform=T.Compose([T.ToTensor(), norm]))
    return DataLoader(ds, batch_size=100, shuffle=False, num_workers=1)


def _mnist(batch_size, distribution, train, root="./data"):
    import torchvision
    import torchvision.transforms as T
    tf = T.Compose([T.ToTensor(), T.Normalize((0.1307,), (0.3081,))])
    ds = torchvision.datasets.MNIST(root=root, train=train, download=False, transform=tf)
    if train:
        return DataLoader(Subset(ds, _select_by_label(ds.targets.tolist(), distribution)), batch_size=batch_size, shuffle=True)
    return DataLoader(ds, batch_size=100, shuffle=False)


def _agnews(batch_size, distribution, train, root="./data"):
    import pandas as pd
    from transformers import BertTokenizer
    from .text import TokenizedTextDataset
    tok = BertTokenizer.from_pretrained("bert-base-cased")
    df = pd.read_csv(os.path.join(root, "AGNEWS_TRAIN.csv" if train else "AGNEWS_TEST.csv"))
    dist = distribution if train else [500, 500, 500, 500]
    idx = _select_by_label(df["label"].tolist(), dist)
    texts = [df["text"].iloc[i] for i in idx]
    labels = [int(df["label"].iloc[i]) for i in idx]
    ds = TokenizedTextDataset(texts, labels, tok, max_length=128)
    return DataLoader(ds, batch_size=batch_size if train else 20, shuffle=train)


def _speechcommands(batch_size, distribution, train, root="./data"):
    from .speechcommands import CLASSES, SpeechCommandsDataset
    ds = SpeechCommandsDataset(root=root, subset="training" if train else "testing")
    if not train:
        return DataLoader(ds, batch_size=20, shuffle=False)
    if distribution is None:
        return DataLoader(ds, batch_size=batch_size, shuffle=True)
    labels = [CLASSES.index(name) for _, name in ds.samples]
    return DataLoader(Subset(ds, _select_by_label(labels, distribution)), batch_size=batch_size, shuffle=True)


_REAL = {"CIFAR10": _cifar10, "MNIST": _mnist, "AGNEWS": _agnews, "SPEECHCOMMANDS": _speechcommands}
_PRESENT = {"CIFAR10": "cifar-10-batches-py", "MNIST": "MNIST", "AGNEWS": "AGNEWS_TRAIN.csv",
            "SPEECHCOMMANDS": "SpeechCommands"}


def real_data_available(data_name: str, root: str = "./data") -> bool:
    marker = _PRESENT.get(data_name.upper())
    return bool(marker) and os.path.exists(os.path.join(root, marker))


def gpu_image_loader(name: str, batch_size: int, distribution: Sequence[int], device, synthetic: bool, root: str = "./data",
                     seed: int = 0):
    """Training loader whose dataset lives on the GPU and whose microbatches are built by one kernel
    (``data/gpu_loader.py``): CIFAR10 (crop + flip + normalise, the reference recipe) and MNIST (normalise)."""
    from .gpu_loader import CIFAR_MEAN, CIFAR_STD, MNIST_MEAN, MNIST_STD, GpuImageLoader
    shape, _, ncls, _ = DATASET_SHAPES[name]
    c, h, w = shape
    if synthetic:
        labels: List[int] = []
        for lbl, cnt in enumerate(distribution):
            labels += [lbl % ncls] * int(cnt)
        y = torch.tensor(labels, dtype=torch.long)
        g = torch.Generator().manual_seed(seed)
        img = torch.randn(len(labels), h, w, c, generator=g) * 40.0 + 128.0 + (y.float().view(-1, 1, 1, 1) - (ncls - 1) / 2) * 10.0
        images = img.clamp_(0, 255).to(torch.uint8)
    else:
        import numpy as np
        import torchvision
        if name == "CIFAR10":
            ds = torchvision.datasets.CIFAR10(root=root, train=True, download=False)
            data, targets = ds.data, list(ds.targets)                       # uint8 [N, 32, 32, 3]
        else:
            ds = torchvision.datasets.MNIST(root=root, train=True, download=False)
            data, targets = ds.data.numpy()[..., None], ds.targets.tolist()  # uint8 [N, 28, 28, 1]
        pick = _select_by_label(targets, distribution)
        images = torch.from_numpy(np.ascontiguousarray(data[pick]))
        y = torch.tensor([targets[i] for i in pick], dtype=torch.long)
    mean, std = (CIFAR_MEAN, CIFAR_STD) if name == "CIFAR10" else (MNIST_MEAN, MNIST_STD)
    return GpuImageLoader(images, y, batch_size, device, mean, std, augment=(name == "CIFAR10"), seed=seed)


_WARNED: set = set()


def data_loader(data_name: Optional[str] = None, batch_size: Optional[int] = None,
                distribution: Optional[Sequence[int]] = None, train: bool = True,
                synthetic: Optional[bool] = None, root: str = "./data", seed: int = 0, device=None,
                gpu_loader: bool = False) -> DataLoader:
    name = str(data_name).upper()
    if name not in DATASET_SHAPES:
        raise ValueError(f"Dataset {data_name} not supported.")
    explicit = synthetic is not None or os.environ.get("SLB200_SYNTHETIC", "0") == "1"
    if synthetic is None:
        synthetic = os.environ.get("SLB200_SYNTHETIC", "0") == "1" or not real_data_available(name, root)
    if synthetic and not explicit and name not in _WARNED:
        # never train on noise silently: the reference would download the dataset or fail (src/dataset/dataloader.py:61-84)
        _WARNED.add(name)
        import warnings
        msg = (f"dataset {name} not found under {root!r}: using SYNTHETIC {name}-shaped samples (random, class-dependent mean). "
               "Accuracy / loss numbers of this run are meaningless; set b200.synthetic-data: true (or SLB200_SYNTHETIC=1) to "
               "acknowledge, or place the real dataset files.")
        warnings.warn(msg, RuntimeWarning, stacklevel=2)
        print("\033[93m[WARNING] " + msg + "\033[0m", flush=True)
    if not train:
        seed = seed + 7919                     # held-out stream: validation never re-draws the training samples
    if (gpu_loader and train and name in ("CIFAR10", "MNIST") and device is not None and torch.device(device).type == "cuda"
            and distribution is not None and len(distribution) > 0):
        return gpu_image_loader(name, int(batch_size), distribution, device, bool(synthetic), root, seed)
    if synthetic or name not in _REAL:
        shape, dtype, ncls, test_bs = DATASET_SHAPES[name]
        if distribution is None or len(distribution) == 0:
            distribution = [max(1, (100 if not train else 500) // ncls)] * ncls
        pin = train and device is not None and torch.device(device).type == "cuda"
        return synthetic_loader(name, batch_size if train else test_bs, distribution, train=train, seed=seed, pin=pin)
    return _REAL[name](batch_size, distribution, train, root)
