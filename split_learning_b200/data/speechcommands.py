"""Speech Commands (10-class subset) with a NumPy MFCC front-end, in two recipes (``b200.speech-features``).

Both have the shape of the reference's recipe (src/dataset/SPEECHCOMMANDS.py:11-47: pre-emphasis 0.97, Hamming frames
with a 10 ms hop at 16 kHz, power spectrum, 40 mel filters, log, DCT → 40 coefficients, 98 frames), written here as
vectorised framing + one matmul per stage.

``engine`` (the default, ``mfcc()``): clips of L = 15 920 samples, fp64 pre-emphasis, a 400-sample window zero-padded
to a 512-point rFFT, ln(max(·, 1e-10)); int32 files are converted without scaling.

``reference`` (``mfcc_reference()``): the reference's recipe — clips of 16 000 samples, pre-emphasis in fp32 as NumPy
computes it on the float32 waveform, a 480-sample window and 480-point rFFT, 20·log10 with exact zeros replaced by
``np.finfo(float).eps``, int32 files scaled by 2^-31.  The orthonormal DCT matrix agrees with scipy's DCT-II to ~1e-14.

Unreadable files become zeros (:116-118); in the reference recipe so do multi-channel files, which the reference turns
into a wrongly shaped tensor.  ``b200.gpu-loader`` computes the same features on the GPU from ``mfcc_tables(recipe)``
(data/gpu_loader.py).
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
# the reference recipe: n_fft = window = 480, the same hop, 98 = 1 + (16000 - 480) // 160 frames of a 16 000-sample clip
REF_N_FFT = REF_WIN = 480
REF_L = REF_WIN + HOP * (FRAMES - 1)
REF_LOG_EPS = float(np.finfo(float).eps)          # replaces mel energies that are exactly 0 before 20·log10
RECIPES = ("engine", "reference")


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
_REF_FB, _REF_WINDOW = _mel_filterbank(n_fft=REF_N_FFT), np.hamming(REF_WIN)


def speech_recipe(value) -> str:
    """Normalise a ``b200.speech-features`` value to "engine" | "reference" (None: "engine")."""
    s = "engine" if value is None else str(value).strip().lower()
    if s not in RECIPES:
        raise ValueError(f"b200.speech-features must be engine or reference, got {value!r}")
    return s


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


def mfcc_reference(wave: np.ndarray) -> np.ndarray:
    """The reference recipe: float32 waveform (any length; padded or truncated to REF_L) → (40, 98) float32 MFCC.
    Pre-emphasis p[t] = fp32(w[t] - fp32(0.97f * w[t-1])) on the float32 samples; everything after it in fp64; one
    rounding to fp32 at the end."""
    w = np.asarray(wave, dtype=np.float32).ravel()
    w = np.pad(w, (0, max(0, REF_L - w.size)))[:REF_L]
    p = np.append(w[0], w[1:] - np.float32(PREEMPH) * w[:-1])
    idx = np.arange(REF_WIN)[None, :] + HOP * np.arange(FRAMES)[:, None]
    frames = p[idx].astype(np.float64) * _REF_WINDOW
    power = (np.abs(np.fft.rfft(frames, REF_N_FFT)) ** 2) / REF_N_FFT
    e = power @ _REF_FB.T
    mel = 20.0 * np.log10(np.where(e == 0.0, REF_LOG_EPS, e))
    return (mel @ _DCT.T).T.astype(np.float32)


def mfcc_tables(recipe: str = "engine"):
    """The fp64 tables of ``mfcc()`` (or of ``mfcc_reference()``) as the GPU kernel takes them (``ops.native.mfcc``): the
    window, the mel filterbank, the DCT matrix, and the (cos, sin) of 2 pi j / n_fft for j < n_fft, whose entry
    (k * t) mod n_fft is the twiddle of bin k at sample t."""
    n_fft, window, fb = (N_FFT, _WINDOW, _FB) if speech_recipe(recipe) == "engine" else (REF_N_FFT, _REF_WINDOW, _REF_FB)
    j = np.arange(n_fft) * (2.0 * np.pi / n_fft)
    return {"window": window, "fb": fb, "dct": _DCT, "twiddle": np.stack([np.cos(j), np.sin(j)], axis=1)}


def clip_length(recipe: str = "engine") -> int:
    """Samples per clip the recipe pads or truncates to: 15 920 (engine) or 16 000 (reference)."""
    return WIN + HOP * (FRAMES - 1) if speech_recipe(recipe) == "engine" else REF_L


def read_wave(path: str, recipe: str = "engine") -> np.ndarray:
    """A ``.wav`` file as the flat float32 waveform the recipe's MFCC is given: int16 scaled by 1/32768, other sample
    types converted as they are (reference recipe: int32 scaled by 2^-31), channels interleaved.  Raises when the file
    cannot be read, and in the reference recipe when it has more than one channel."""
    from scipy.io import wavfile
    _, wav = wavfile.read(path)
    if speech_recipe(recipe) == "engine":
        return (wav.astype(np.float32) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float32)).ravel()
    if wav.ndim != 1:
        raise ValueError(f"{path}: {wav.shape[1]} channels")
    if wav.dtype == np.int16:
        return wav.astype(np.float32) / 32768.0
    if wav.dtype == np.int32:
        return wav.astype(np.float32) / 2147483648.0
    return wav.astype(np.float32)


class SpeechCommandsDataset(Dataset):
    def __init__(self, root="./data", subset="training", recipe: str = "engine"):
        self.recipe = speech_recipe(recipe)
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
            feat = (mfcc if self.recipe == "engine" else mfcc_reference)(read_wave(path, self.recipe))
        except Exception:
            feat = np.zeros((N_MFCC, FRAMES), dtype=np.float32)
        return torch.from_numpy(feat), CLASSES.index(name)
