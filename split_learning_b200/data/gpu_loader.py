"""GPU-resident image loader (``b200.gpu-loader: true``).

The reference builds every microbatch on the host: PIL crop / flip / ToTensor / Normalize per sample in a
``DataLoader`` (src/dataset/dataloader.py:61-84), then ``.to(device)``.  CIFAR-10 is 150 MB of uint8 — it fits in a
corner of an H100's 80 GB of HBM — so here the selected training subset lives on the GPU once and each microbatch is ONE kernel
(``image_batch_kernel``): gather by shuffled index, RandomCrop(32, padding 4), RandomHorizontalFlip, /255, Normalize,
written as the fp32 NCHW stage input.  No host work and no H2D copy per step; the iterator yields device tensors, which
every executor and the device data plane accept as they are.
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
