"""Speech Commands loaders without a GPU: ``gpu_loader`` changes nothing off CUDA, and the fp64 tables the MFCC kernel is
given are the host recipe's own arrays, with twiddles that reproduce the host spectrum."""
import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from split_learning_b200.data import data_loader
from split_learning_b200.data import speechcommands as sc
from split_learning_b200.data.loaders import BatchedTensorLoader

from speech_tree import make_tree

DIST = [7, 3, 5, 2, 4, 6, 1, 3, 2, 4]


def _batches(loader):
    return [(x.clone(), torch.as_tensor(y).clone()) for x, y in loader]


@pytest.mark.parametrize("device,gpu_loader", [(None, True), ("cpu", True), ("cpu", False)])
def test_synthetic_loader_unchanged_off_cuda(device, gpu_loader):
    ref = data_loader("SPEECHCOMMANDS", 8, DIST, train=True, synthetic=True, seed=3)
    got = data_loader("SPEECHCOMMANDS", 8, DIST, train=True, synthetic=True, seed=3, device=device, gpu_loader=gpu_loader)
    assert type(got) is type(ref) is BatchedTensorLoader
    assert torch.equal(got.dataset.data, ref.dataset.data) and torch.equal(got.dataset.labels, ref.dataset.labels)
    for (xa, ya), (xb, yb) in zip(_batches(got), _batches(ref), strict=True):
        assert torch.equal(xa, xb) and torch.equal(ya, yb)


@pytest.mark.parametrize("device", [None, "cpu"])
def test_real_loader_unchanged_off_cuda(tmp_path, device):
    tree = make_tree(tmp_path, per_class=2)
    dist = [100] * 10                                   # every training clip of every class
    ref = data_loader("SPEECHCOMMANDS", 4, dist, train=True, synthetic=False, root=str(tmp_path))
    got = data_loader("SPEECHCOMMANDS", 4, dist, train=True, synthetic=False, root=str(tmp_path), device=device,
                      gpu_loader=True)
    assert type(got) is type(ref) is DataLoader
    key = lambda b: sorted((int(y), x.numpy().tobytes()) for xs, ys in b for x, y in zip(xs, ys))
    assert key(_batches(got)) == key(_batches(ref))
    assert sum(x.shape[0] for x, _ in _batches(got)) == len(tree["train"])


def test_tables_are_the_host_arrays():
    t = sc.mfcc_tables()
    assert np.array_equal(t["window"], sc._WINDOW) and np.array_equal(t["fb"], sc._FB) and np.array_equal(t["dct"], sc._DCT)
    assert all(t[k].dtype == np.float64 for k in t)
    assert t["twiddle"].shape == (sc.N_FFT, 2) and t["fb"].shape == (sc.N_MELS, sc.N_FFT // 2 + 1)
    j = np.arange(sc.N_FFT)
    assert np.allclose(t["twiddle"][:, 0], np.cos(2 * np.pi * j / sc.N_FFT), rtol=0, atol=1e-15)
    assert np.allclose(t["twiddle"][:, 1], np.sin(2 * np.pi * j / sc.N_FFT), rtol=0, atol=1e-15)


def _table_mfcc(wave):
    """The kernel's algorithm in NumPy: direct DFT with twiddle (k * t) mod N_FFT from the table, then the host's mel,
    log and DCT."""
    t = sc.mfcc_tables()
    L = sc.WIN + sc.HOP * (sc.FRAMES - 1)
    w = np.pad(np.asarray(wave, np.float64).ravel(), (0, max(0, L - np.size(wave))))[:L]
    w = np.append(w[0], w[1:] - sc.PREEMPH * w[:-1])
    frames = w[np.arange(sc.WIN)[None, :] + sc.HOP * np.arange(sc.FRAMES)[:, None]] * t["window"]
    j = (np.arange(sc.N_FFT // 2 + 1)[:, None] * np.arange(sc.WIN)[None, :]) % sc.N_FFT
    re, im = frames @ t["twiddle"][j, 0].T, frames @ t["twiddle"][j, 1].T
    power = (re * re + im * im) / sc.N_FFT
    mel = np.log(np.maximum(power @ t["fb"].T, sc.LOG_FLOOR))
    return (mel @ t["dct"].T).T.astype(np.float32)


def test_table_dft_matches_host_mfcc():
    rng = np.random.default_rng(1)
    L = sc.WIN + sc.HOP * (sc.FRAMES - 1)
    tt = np.arange(L) / sc.SAMPLE_RATE
    for wave in (np.sin(2 * np.pi * (100 + 3000 * tt) * tt).astype(np.float32), (rng.standard_normal(L) * 0.1).astype(np.float32),
                 np.zeros(L, np.float32), rng.standard_normal(9000).astype(np.float32)):
        ref, got = sc.mfcc(wave), _table_mfcc(wave)
        tol = np.spacing(np.abs(ref)) + 1e-9 * np.abs(ref).max()
        assert np.all(np.abs(got.astype(np.float64) - ref) <= tol)


def test_read_wave_is_the_dataset_conversion(tmp_path):
    tree = make_tree(tmp_path, per_class=1)
    ds = sc.SpeechCommandsDataset(root=str(tmp_path))
    paths = {p: i for i, (p, _) in enumerate(ds.samples)}
    stereo = [p for p in paths if p.endswith(tree["stereo"])][0]
    w = sc.read_wave(stereo)
    assert w.dtype == np.float32 and w.ndim == 1 and w.size == 2 * 9000
    assert np.array_equal(ds[paths[stereo]][0].numpy(), sc.mfcc(w))
    bad = [p for p in paths if p.endswith(tree["unreadable"])][0]
    with pytest.raises(Exception):
        sc.read_wave(bad)
    assert not ds[paths[bad]][0].numpy().any()
