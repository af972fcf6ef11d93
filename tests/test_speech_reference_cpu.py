"""The reference MFCC recipe (``b200.speech-features: reference``) on the host: ``mfcc_reference`` and the dataset against
features the reference itself computed (``tests/golden/speech_mfcc_reference.npz``, written by ``tools/make_golden.py``),
the fp64 tables the GPU kernel is given, the option's parsing, and its routing to the training and test loaders.

Bound against the reference's fp64 ``compute_mfcc``: |ours - ref| <= ulp32(|ref|) + 1e-13 * max|ref| of the clip.
  * Pre-emphasis, framing, window, rFFT and 20·log10 are the same operations on the same values: the fp32 pre-emphasis is
    bitwise the reference's, the frames are the same fp64 products, and both call NumPy's fp64 rFFT.  The power divides
    by 480 where the reference multiplies by 1/480: at most 1 ulp64 relative, 20·log10 turns it into < 1e-14 absolute.
  * The DCT is a matrix here and scipy's fftpack there.  Each computes 40-term sums of fp64 products, an error of at most
    about 40 · 2^-53 · sum_m |d_km · mel_m| each.  |d_km| <= sqrt(2/40) and, the DCT being orthonormal,
    sum_m |mel_m| <= sqrt(40) · ||mel||_2 = sqrt(40) · ||mfcc||_2 <= 40 · max|ref|: together about 8e-14 · max|ref|.
  * Ours is rounded to fp32 once: at most half an ulp32 of a value within the above of ref, i.e. within ulp32(|ref|).
Against the reference's fp32 ``__getitem__`` features the same bound holds: both are single roundings of fp64 values
within 1e-13 · max|ref| of each other.
"""
import os

import numpy as np
import pytest
import torch

from split_learning_b200.data import data_loader
from split_learning_b200.data import speechcommands as sc

from speech_tree import make_tree

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "speech_mfcc_reference.npz"))
CLIPS = sorted(k[len("clip/"):] for k in GOLDEN.files if k.startswith("clip/"))


def _assert_close(got, ref, rel=1e-13):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape == (sc.N_MFCC, sc.FRAMES)
    tol = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + rel * np.abs(ref).max()
    err = np.abs(got - ref)
    assert np.all(err <= tol), f"max error {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)}"


def _as_float(clip):
    """The reference's conversion of a clip's samples (int16 / 2^15, int32 / 2^31, float32 as is)."""
    scale = {np.dtype(np.int16): 32768.0, np.dtype(np.int32): 2147483648.0}.get(clip.dtype, 1.0)
    return clip.astype(np.float32) / np.float32(scale)


def test_golden_clips_cover_the_cases():
    dtypes = {GOLDEN[f"clip/{n}"].dtype for n in CLIPS}
    sizes = {GOLDEN[f"clip/{n}"].size for n in CLIPS}
    assert dtypes == {np.dtype(np.int16), np.dtype(np.int32), np.dtype(np.float32)}
    assert min(sizes) < sc.REF_L < max(sizes)
    assert not GOLDEN["clip/silence"].any()


@pytest.mark.parametrize("name", CLIPS)
def test_mfcc_reference_matches_compute_mfcc(name):
    _assert_close(sc.mfcc_reference(_as_float(GOLDEN[f"clip/{name}"])), GOLDEN[f"mfcc/{name}"])


def test_silence_takes_the_eps_branch():
    ref = GOLDEN["mfcc/silence"]
    assert np.isclose(ref[0, 0], 20 * np.log10(sc.REF_LOG_EPS) * sc._DCT[0].sum(), rtol=1e-12)
    _assert_close(sc.mfcc_reference(np.zeros(123, np.float32)), ref)


def test_preemphasis_is_fp32():
    w = _as_float(GOLDEN["clip/noise"])
    f64 = sc.mfcc_reference(w)
    p = np.append(w[0], w[1:] - np.float32(0.97) * w[:-1])
    assert p.dtype == np.float32
    wide = np.append(w[0], w[1:].astype(np.float64) - 0.97 * w[:-1].astype(np.float64)).astype(np.float32)
    assert np.count_nonzero(p != wide) > 1000                # the fp64 pre-emphasis would be a different recipe
    assert np.array_equal(f64, sc.mfcc_reference(w.astype(np.float64)))   # the input is taken as float32 first


@pytest.mark.parametrize("name", CLIPS)
def test_reference_reader_scales_like_the_reference(tmp_path, name):
    from scipy.io import wavfile
    clip = GOLDEN[f"clip/{name}"]
    path = str(tmp_path / f"{name}.wav")
    wavfile.write(path, sc.SAMPLE_RATE, clip)
    w = sc.read_wave(path, "reference")
    assert w.dtype == np.float32 and np.array_equal(w, _as_float(clip))
    _assert_close(sc.mfcc_reference(w), GOLDEN[f"mfcc/{name}"])


def test_dataset_matches_reference_getitem(tmp_path):
    tree = make_tree(tmp_path, per_class=1)
    ds = sc.SpeechCommandsDataset(root=str(tmp_path), recipe="reference")
    assert ds.samples == sc.SpeechCommandsDataset(root=str(tmp_path)).samples
    rels = [os.path.relpath(p, tree["base"]).replace(os.sep, "/") for p, _ in ds.samples]
    assert sorted(f"item/{r}" for r in rels if r != tree["stereo"]) == sorted(k for k in GOLDEN.files if k.startswith("item/"))
    for i, rel in enumerate(rels):
        x, y = ds[i]
        assert x.dtype == torch.float32 and y == sc.CLASSES.index(rel.split("/")[0])
        if rel in (tree["unreadable"], tree["stereo"]):
            assert not x.numpy().any(), rel                   # unreadable and multi-channel files: zero rows
        else:
            _assert_close(x.numpy(), GOLDEN[f"item/{rel}"])
    assert not GOLDEN[f"item/{tree['unreadable']}"].any()


def test_reference_reader_refuses_multichannel(tmp_path):
    tree = make_tree(tmp_path, per_class=1)
    stereo = os.path.join(tree["base"], tree["stereo"])
    with pytest.raises(ValueError):
        sc.read_wave(stereo, "reference")
    assert sc.read_wave(stereo).size == 2 * 9000            # the engine recipe keeps interleaving the channels


def test_reference_tables():
    t = sc.mfcc_tables("reference")
    assert all(v.dtype == np.float64 for v in t.values())
    assert t["window"].shape == (sc.REF_WIN,) and np.array_equal(t["window"], np.hamming(480))
    assert t["fb"].shape == (sc.N_MELS, 241) and t["dct"].shape == (sc.N_MFCC, sc.N_MELS)
    assert np.array_equal(t["dct"], sc._DCT)
    assert (t["fb"].sum(axis=1) > 0).all()                 # no empty filter at n_fft = 480
    j = np.arange(480)
    assert t["twiddle"].shape == (480, 2)
    assert np.allclose(t["twiddle"], np.stack([np.cos(2 * np.pi * j / 480), np.sin(2 * np.pi * j / 480)], 1), rtol=0,
                       atol=1e-15)
    e = sc.mfcc_tables("engine")
    assert all(np.array_equal(e[k], v) for k, v in sc.mfcc_tables().items())
    assert sc.clip_length() == 15920 and sc.clip_length("reference") == 16000 == sc.REF_L
    with pytest.raises(ValueError, match="speech-features"):
        sc.mfcc_tables("fast")


def _table_mfcc_reference(wave):
    """The kernel's reference-recipe algorithm in NumPy: fp32 pre-emphasis, direct DFT with twiddle (k * t) mod 480 from
    the table, 20·log10 with exact zeros replaced by eps, DCT matrix."""
    t = sc.mfcc_tables("reference")
    w = np.pad(np.asarray(wave, np.float32), (0, max(0, sc.REF_L - np.size(wave))))[:sc.REF_L]
    p = np.append(w[0], w[1:] - np.float32(sc.PREEMPH) * w[:-1]).astype(np.float64)
    frames = p[np.arange(sc.REF_WIN)[None, :] + sc.HOP * np.arange(sc.FRAMES)[:, None]] * t["window"]
    j = (np.arange(241)[:, None] * np.arange(sc.REF_WIN)[None, :]) % sc.REF_N_FFT
    re, im = frames @ t["twiddle"][j, 0].T, frames @ t["twiddle"][j, 1].T
    e = ((re * re + im * im) / sc.REF_N_FFT) @ t["fb"].T
    mel = 20.0 * np.log10(np.where(e == 0.0, sc.REF_LOG_EPS, e))
    return (mel @ t["dct"].T).T.astype(np.float32)


@pytest.mark.parametrize("name", CLIPS)
def test_table_dft_matches_mfcc_reference(name):
    """The bound of the GPU test (one ulp32 + 1e-9 · max|ref|) holds for the kernel's algorithm on these clips."""
    w = _as_float(GOLDEN[f"clip/{name}"])
    _assert_close(_table_mfcc_reference(w), sc.mfcc_reference(w), rel=1e-9)


def test_option_default_and_parsing():
    import yaml
    from split_learning_b200.config import DEFAULT_B200, normalize
    raw = yaml.safe_load(open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "config.yaml")))
    assert DEFAULT_B200["speech-features"] == "engine"
    assert normalize(raw).b200["speech-features"] == "engine"
    for value, want in (("reference", "reference"), (" Reference ", "reference"), ("engine", "engine"), (None, "engine")):
        raw["b200"] = {"speech-features": value}
        assert normalize(raw).b200["speech-features"] == want
    for bad in ("ref", "torchaudio", 1, True):
        raw["b200"] = {"speech-features": bad}
        with pytest.raises(ValueError, match="b200.speech-features"):
            normalize(raw)
    with pytest.raises(ValueError, match="b200.speech-features"):
        data_loader("SPEECHCOMMANDS", 4, [1] * 10, train=True, synthetic=True, speech_features="mfcc")


def _samples(loader):
    return [(int(y), x.numpy().tobytes()) for xs, ys in loader for x, y in zip(xs, torch.as_tensor(ys))]


def test_loaders_without_the_option_are_unchanged(tmp_path):
    make_tree(tmp_path, per_class=1)
    dist = [100] * 10
    for train in (True, False):
        kw = dict(train=train, synthetic=False, root=str(tmp_path))
        base = data_loader("SPEECHCOMMANDS", 4, dist if train else None, **kw)
        ds = base.dataset.dataset if train else base.dataset
        assert ds.recipe == "engine"
        want = sorted((sc.CLASSES.index(n), (sc.mfcc(sc.read_wave(p)) if not p.endswith("broken.wav") else
                                             np.zeros((sc.N_MFCC, sc.FRAMES), np.float32)).tobytes())
                      for p, n in (ds.samples if not train else [ds.samples[i] for i in base.dataset.indices]))
        assert sorted(_samples(base)) == want
        explicit = data_loader("SPEECHCOMMANDS", 4, dist if train else None, speech_features="engine", **kw)
        assert sorted(_samples(explicit)) == want


def test_host_train_and_test_loaders_take_the_reference_recipe(tmp_path):
    tree = make_tree(tmp_path, per_class=1)
    root = str(tmp_path)

    def expect(path):
        try:
            return sc.mfcc_reference(sc.read_wave(path, "reference"))
        except Exception:
            return np.zeros((sc.N_MFCC, sc.FRAMES), np.float32)
    train = data_loader("SPEECHCOMMANDS", 4, [100] * 10, train=True, synthetic=False, root=root, speech_features="reference")
    ds = train.dataset.dataset
    assert ds.recipe == "reference"
    got = sorted(_samples(train))
    assert len(got) == len(tree["train"])
    assert got == sorted((sc.CLASSES.index(n), expect(p).tobytes()) for p, n in ds.samples)
    test = data_loader("SPEECHCOMMANDS", train=False, synthetic=False, root=root, speech_features="reference")
    assert test.dataset.recipe == "reference" and test.batch_size == 20
    assert _samples(test) == [(sc.CLASSES.index(n), expect(p).tobytes()) for p, n in test.dataset.samples]
    assert len(test.dataset) == 10


def test_synthetic_data_ignores_the_option():
    a = data_loader("SPEECHCOMMANDS", 8, [3] * 10, train=True, synthetic=True, seed=4, speech_features="reference")
    b = data_loader("SPEECHCOMMANDS", 8, [3] * 10, train=True, synthetic=True, seed=4)
    assert torch.equal(a.dataset.data, b.dataset.data) and torch.equal(a.dataset.labels, b.dataset.labels)


@pytest.mark.parametrize("recipe", [None, "engine", "reference"])
def test_get_val_routes_the_option_to_the_test_loader(monkeypatch, recipe):
    from split_learning_b200 import validation as V
    from split_learning_b200.models import get_model_class
    seen = []

    def spy(**kw):
        seen.append(kw)
        return data_loader(**kw)
    monkeypatch.setattr(V, "data_loader", spy)
    torch.manual_seed(0)
    sd = get_model_class("KWT", "SPEECHCOMMANDS")().state_dict()
    kw = {} if recipe is None else {"speech_features": recipe}
    ok, m = V.get_val("KWT", "SPEECHCOMMANDS", sd, device="cpu", synthetic=True, **kw)
    assert ok and m["val_backend"] == "torch" and m["val_total"] > 0
    assert len(seen) == 1 and seen[0]["train"] is False
    assert seen[0]["speech_features"] == (recipe or "engine")
