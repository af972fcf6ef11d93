"""Speech Commands (10-class subset) with a NumPy MFCC front-end.

The shape of the reference's recipe (src/dataset/SPEECHCOMMANDS.py:11-47: pre-emphasis 0.97,
25 ms Hamming frames / 10 ms hop at 16 kHz, power spectrum, 40 mel filters, log, DCT → 40
coefficients, 98 frames), written here as vectorised framing + one matmul per stage.  It is not
the reference's exact recipe (a known open issue, see PARITY.md): the reference frames with
n_fft = 480 directly where this zero-pads a 400-sample window to 512, takes 20·log10 with exact
zeros replaced by eps where this takes ln(max(·, 1e-10)), and uses scipy's orthonormal DCT.
Unreadable files become zeros (:116-118).  ``b200.gpu-loader`` computes the same features on
the GPU from ``mfcc_tables()`` (data/gpu_loader.py).
"""
from __future__ import annotations

import os
from typing import List, Tuple

import numpy as np
import torch
from torch.utils.data import Dataset

CLASSES = ["yes", "no", "up", "down", "left", "right", "on", "off", "stop", "go"]
SAMPLE_RATE, N_MFCC, N_MELS, N_FFT, WIN, HOP, FRAMES = 16000, 40, 40, 512, 400, 160, 98
PREEMPH, LOG_FLOOR = 0.97, 1e-10


def _mel_filterbank(n_mels=N_MELS, n_fft=N_FFT, sr=SAMPLE_RATE) -> np.ndarray:
    hz2mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    mel2hz = lambda m: 700.0 * (10 ** (m / 2595.0) - 1.0)
    pts = mel2hz(np.linspace(hz2mel(0.0), hz2mel(sr / 2), n_mels + 2))
    bins = np.floor((n_fft + 1) * pts / sr).astype(int)
    fb = np.zeros((n_mels, n_fft // 2 + 1))
    for m in range(1, n_mels + 1):
        l, c, r = bins[m - 1], bins[m], bins[m + 1]
        if c > l:
            fb[m - 1, l:c] = (np.arange(l, c) - l) / (c - l)
        if r > c:
            fb[m - 1, c:r] = (r - np.arange(c, r)) / (r - c)
    return fb


def _dct_matrix(n_out=N_MFCC, n_in=N_MELS) -> np.ndarray:
    k = np.arange(n_out)[:, None]
    n = np.arange(n_in)[None, :]
    m = np.cos(np.pi * k * (2 * n + 1) / (2 * n_in)) * np.sqrt(2.0 / n_in)
    m[0] *= 1.0 / np.sqrt(2.0)
    return m


_FB, _DCT, _WINDOW = _mel_filterbank(), _dct_matrix(), np.hamming(WIN)


def mfcc(wave: np.ndarray) -> np.ndarray:
    """float waveform (any length) → (40, 98) float32 MFCC."""
    w = np.asarray(wave, dtype=np.float64).ravel()
    need = WIN + HOP * (FRAMES - 1)
    w = np.pad(w, (0, max(0, need - w.size)))[:need]
    w = np.append(w[0], w[1:] - PREEMPH * w[:-1])
    idx = np.arange(WIN)[None, :] + HOP * np.arange(FRAMES)[:, None]
    frames = w[idx] * _WINDOW
    power = (np.abs(np.fft.rfft(frames, N_FFT)) ** 2) / N_FFT
    mel = np.log(np.maximum(power @ _FB.T, LOG_FLOOR))
    return (mel @ _DCT.T).T.astype(np.float32)


def mfcc_tables():
    """The fp64 tables of ``mfcc()`` as the GPU kernel takes them (``ops.native.mfcc``): the window, the mel filterbank, the
    DCT matrix, and the (cos, sin) of 2 pi j / N_FFT for j < N_FFT, whose entry (k * t) mod N_FFT is the twiddle of bin k
    at sample t."""
    j = np.arange(N_FFT) * (2.0 * np.pi / N_FFT)
    return {"window": _WINDOW, "fb": _FB, "dct": _DCT, "twiddle": np.stack([np.cos(j), np.sin(j)], axis=1)}


def read_wave(path: str) -> np.ndarray:
    """A ``.wav`` file as the flat float32 waveform ``mfcc()`` is given: int16 scaled by 1/32768, other sample types
    converted as they are, channels interleaved.  Raises when the file cannot be read."""
    from scipy.io import wavfile
    _, wav = wavfile.read(path)
    return (wav.astype(np.float32) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float32)).ravel()


class SpeechCommandsDataset(Dataset):
    def __init__(self, root="./data", subset="training"):
        base = os.path.join(root, "SpeechCommands", "speech_commands_v0.02")
        self.samples: List[Tuple[str, str]] = []
        held = set()
        for lst in ("validation_list.txt", "testing_list.txt"):
            p = os.path.join(base, lst)
            if os.path.exists(p):
                with open(p) as f:
                    names = {l.strip() for l in f}
                if (lst.startswith("testing") and subset == "testing") or \
                   (lst.startswith("validation") and subset == "validation"):
                    self.samples = [(os.path.join(base, n), n.split("/")[0]) for n in sorted(names)
                                    if n.split("/")[0] in CLASSES]
                held |= names
        if subset == "training" and os.path.isdir(base):
            for c in CLASSES:
                d = os.path.join(base, c)
                if os.path.isdir(d):
                    for fn in sorted(os.listdir(d)):
                        if fn.endswith(".wav") and f"{c}/{fn}" not in held:
                            self.samples.append((os.path.join(d, fn), c))

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        path, name = self.samples[i]
        try:
            feat = mfcc(read_wave(path))
        except Exception:
            feat = np.zeros((N_MFCC, FRAMES), dtype=np.float32)
        return torch.from_numpy(feat), CLASSES.index(name)
