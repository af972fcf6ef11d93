"""GPU-resident training loaders (``b200.gpu-loader: true``): images and Speech Commands features.

The reference builds every microbatch on the host: PIL crop / flip / ToTensor / Normalize per sample in a
``DataLoader`` (src/dataset/dataloader.py:61-84), then ``.to(device)``.  CIFAR-10 is 150 MB of uint8 — it fits in a
corner of an H100's 80 GB of HBM — so here the selected training subset lives on the GPU once and each microbatch is ONE kernel
(``image_batch_kernel``): gather by shuffled index, RandomCrop(32, padding 4), RandomHorizontalFlip, /255, Normalize,
written as the fp32 NCHW stage input.  No host work and no H2D copy per step; the iterator yields device tensors, which
every executor and the device data plane accept as they are.

Speech Commands (KWT) is held as its MFCC features: the host reads each ``.wav`` once, ``mfcc_kernel`` turns the clips into
[40, 98] features in fp64 with the tables of ``speechcommands.mfcc()`` or, with ``b200.speech-features: reference``,
``mfcc_reference()`` (the same values the host loader computes per ``__getitem__``), and each microbatch is one gather
(``GpuFeatureLoader``, ``feature_batch_kernel``).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from ..ops import native as N

CIFAR_MEAN, CIFAR_STD = (0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010)
MNIST_MEAN, MNIST_STD = (0.1307,), (0.3081,)


class GpuImageLoader:
    """Iterable of (x [B, C, H, W] fp32, y [B] int64) device tensors; ``len()`` = microbatches per epoch."""

    def __init__(self, images_u8: torch.Tensor, labels: torch.Tensor, batch_size: int, device, mean: Sequence[float],
                 std: Sequence[float], augment: bool = True, pad: int = 4, shuffle: bool = True, drop_last: bool = False,
                 seed: Optional[int] = None):
        if images_u8.dtype != torch.uint8 or images_u8.dim() != 4:
            raise ValueError("images must be uint8 [N, H, W, C]")
        self.device = torch.device(device)
        self.images = images_u8.contiguous().to(self.device)
        self.labels = labels.long().to(self.device)
        self.n, self.h, self.w, self.c = self.images.shape
        self.batch_size, self.augment, self.pad, self.shuffle, self.drop_last = batch_size, augment, pad, shuffle, drop_last
        self.mean, self.std = tuple(mean), tuple(std)
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(int(seed) if seed is not None else torch.initial_seed() & 0x7FFFFFFF)
        N.require()

    def __len__(self):
        return self.n // self.batch_size if self.drop_last else (self.n + self.batch_size - 1) // self.batch_size

    def draw(self, b: int):
        """Per-sample augmentation parameters (device int32): crop offsets in [-pad, pad], flip in {0, 1}."""
        if not self.augment:
            z = torch.zeros(b, dtype=torch.int32, device=self.device)
            return z, z, z
        r = torch.randint(0, 2 * self.pad + 1, (2, b), device=self.device, generator=self.gen, dtype=torch.int32) - self.pad
        f = torch.randint(0, 2, (b,), device=self.device, generator=self.gen, dtype=torch.int32)
        return r[0].contiguous(), r[1].contiguous(), f

    def batch(self, idx: torch.Tensor, dx=None, dy=None, flip=None):
        b = idx.numel()
        if dx is None:
            dx, dy, flip = self.draw(b)
        out = torch.empty(b, self.c, self.h, self.w, dtype=torch.float32, device=self.device)
        N.image_batch(self.images, idx.contiguous(), dx, dy, flip, out, self.mean, self.std)
        return out, self.labels[idx]

    def __iter__(self):
        order = (torch.randperm(self.n, device=self.device, generator=self.gen) if self.shuffle
                 else torch.arange(self.n, device=self.device))
        for k in range(len(self)):
            yield self.batch(order[k * self.batch_size:(k + 1) * self.batch_size])


class GpuFeatureLoader:
    """Iterable of (x [B, *sample] fp32, y [B] int64) device tensors gathered from a resident fp32 split, one
    ``feature_batch`` launch per microbatch; ``len()`` = microbatches per epoch, a fresh permutation per epoch drawn on the
    device generator, the short batch last.  Speech Commands: the [N, 40, 98] MFCC features (``speech_gpu_loader``)."""

    def __init__(self, features: torch.Tensor, labels: torch.Tensor, batch_size: int, device, shuffle: bool = True,
                 seed: Optional[int] = None):
        if features.dtype != torch.float32 or features.dim() < 2:
            raise ValueError("features must be fp32 [N, ...]")
        self.device = torch.device(device)
        self.features = features.to(self.device).contiguous()
        self.labels = labels.long().to(self.device).contiguous()
        self.n = self.features.shape[0]
        self.batch_size, self.shuffle = int(batch_size), shuffle
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(int(seed) if seed is not None else torch.initial_seed() & 0x7FFFFFFF)
        N.require()

    def __len__(self):
        return (self.n + self.batch_size - 1) // self.batch_size

    def batch(self, idx: torch.Tensor):
        b = idx.numel()
        x = torch.empty((b,) + tuple(self.features.shape[1:]), dtype=torch.float32, device=self.device)
        y = torch.empty(b, dtype=torch.long, device=self.device)
        N.feature_batch(self.features, self.labels, idx.contiguous(), x, y)
        return x, y

    def __iter__(self):
        order = (torch.randperm(self.n, device=self.device, generator=self.gen) if self.shuffle
                 else torch.arange(self.n, device=self.device))
        for k in range(len(self)):
            yield self.batch(order[k * self.batch_size:(k + 1) * self.batch_size])


def mfcc_tables(device, recipe: str = "engine"):
    """``speechcommands.mfcc_tables(recipe)`` as fp64 device tensors (the kernel's window, filterbank, DCT and twiddles)."""
    from .speechcommands import mfcc_tables as host_tables
    return {k: torch.from_numpy(v).to(device=device, dtype=torch.float64).contiguous() for k, v in host_tables(recipe).items()}


def mfcc_features(waves: torch.Tensor, valid: torch.Tensor, tables: dict, out: Optional[torch.Tensor] = None,
                  recipe: str = "engine") -> torch.Tensor:
    """fp32 [n, 40, 98] MFCC features of fp32 waveforms [n, L] (already padded or truncated to the recipe's
    ``clip_length``) on the GPU, one ``mfcc`` launch with the recipe's ``tables``; clips with ``valid == 0`` get zeros, as
    ``SpeechCommandsDataset`` gives unreadable files."""
    from .speechcommands import FRAMES, HOP, LOG_FLOOR, N_MFCC, PREEMPH, REF_LOG_EPS, speech_recipe
    recipe = speech_recipe(recipe)
    if out is None:
        out = torch.empty(waves.shape[0], N_MFCC, FRAMES, dtype=torch.float32, device=waves.device)
    N.mfcc(waves, valid, out, tables["window"], tables["fb"], tables["dct"], tables["twiddle"], HOP, PREEMPH,
           LOG_FLOOR if recipe == "engine" else REF_LOG_EPS, recipe)
    return out


class ResidentBatches:
    """Iterable of (x, y) slices of device-resident tensors, in order, ``batch_size`` at a time (short batch last)."""

    def __init__(self, x: torch.Tensor, y: torch.Tensor, batch_size: int, device):
        self.x = x.to(device).contiguous()
        self.y = y.long().to(device)
        self.batch_size = int(batch_size)

    def __len__(self):
        return (self.x.shape[0] + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        for lo in range(0, self.x.shape[0], self.batch_size):
            yield self.x[lo:lo + self.batch_size], self.y[lo:lo + self.batch_size]


def reference_batch(images_u8, idx, dx, dy, flip, mean, std, pad: int = 4):
    """The same transform with plain torch ops (numerics oracle of the kernel)."""
    x = images_u8[idx].permute(0, 3, 1, 2).float() / 255.0
    b, c, h, w = x.shape
    xp = torch.nn.functional.pad(x, (pad, pad, pad, pad))
    out = torch.empty_like(x)
    for i in range(b):
        xi = xp[i, :, pad + int(dy[i]):pad + int(dy[i]) + h, :]
        if int(flip[i]):
            # flip happens after the crop in the reference pipeline: output x reads cropped column W-1-x
            xi = xi[:, :, pad + int(dx[i]):pad + int(dx[i]) + w].flip(-1)
        else:
            xi = xi[:, :, pad + int(dx[i]):pad + int(dx[i]) + w]
        out[i] = xi
    m = torch.tensor(mean, device=x.device).view(1, -1, 1, 1)
    s = torch.tensor(std, device=x.device).view(1, -1, 1, 1)
    return (out - m) / s
