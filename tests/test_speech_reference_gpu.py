"""``mfcc_kernel`` in the reference recipe (``b200.speech-features: reference``) against the host recipe
``speechcommands.mfcc_reference()``, the engine recipe unchanged beside it, the launch refusals, the resident training
split against the host loader on a wav tree, and one KWT round through the public API with training and validation both
on the reference recipe."""
import os

import numpy as np
import pytest
import torch

from split_learning_b200.data import data_loader
from split_learning_b200.data import speechcommands as sc
from split_learning_b200.data.gpu_loader import GpuFeatureLoader, mfcc_features, mfcc_tables
from split_learning_b200.ops import native as N

from speech_tree import make_tree

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "speech_mfcc_reference.npz"))


def _assert_close(got, ref):
    """|gpu - ref| <= ulp32(ref) + 1e-9 * max|ref| of the clip: two fp64 pipelines (a direct DFT here, NumPy's rFFT on the
    host), each rounded to fp32 once."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    for g, r in zip(got, ref, strict=True):
        tol = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(r).max()
        err = np.abs(g - r)
        assert np.all(np.isfinite(g)) and np.all(err <= tol), \
            f"max error {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)}"


def _fit(w, n):
    w = np.asarray(w, np.float32).ravel()[:n]
    return np.pad(w, (0, n - w.size))


def _gpu(waves, recipe, valid=None):
    n = sc.clip_length(recipe)
    w = torch.from_numpy(np.stack([_fit(x, n) for x in waves])).to(DEV)
    v = (torch.ones(len(waves), dtype=torch.uint8, device=DEV) if valid is None
         else torch.tensor(valid, dtype=torch.uint8, device=DEV))
    return mfcc_features(w, v, mfcc_tables(DEV, recipe), recipe=recipe).cpu().numpy()


def _clips():
    """The golden clips as the reference reads them, random clips, silence and clips with trailing all-zero frames."""
    out = {}
    for k in sorted(GOLDEN.files):
        if k.startswith("clip/"):
            c = GOLDEN[k]
            scale = {np.dtype(np.int16): 32768.0, np.dtype(np.int32): 2147483648.0}.get(c.dtype, 1.0)
            out[k[5:]] = c.astype(np.float32) / np.float32(scale)
    rng = np.random.default_rng(7)
    for i in range(4):
        out[f"random{i}"] = (rng.standard_normal(int(rng.integers(4000, 20000))) * rng.uniform(0.01, 0.8)).astype(np.float32)
    out["tail_zeros"] = (rng.standard_normal(5000) * 0.3).astype(np.float32)          # frames 32..97 all zero
    gap = (rng.standard_normal(16000) * 0.2).astype(np.float32)
    gap[4000:9000] = 0.0                                                               # frames 26..53 all zero
    out["gap"] = gap
    return out


CLIPS = _clips()


def test_reference_kernel_matches_mfcc_reference():
    waves = list(CLIPS.values())
    got = _gpu(waves, "reference")
    ref = np.stack([sc.mfcc_reference(w) for w in waves])
    _assert_close(got, ref)


def test_reference_kernel_on_the_golden_clips_matches_compute_mfcc():
    names = [k[5:] for k in sorted(GOLDEN.files) if k.startswith("mfcc/")]
    got = _gpu([CLIPS[n] for n in names], "reference")
    _assert_close(got, np.stack([GOLDEN[f"mfcc/{n}"] for n in names]))


def test_zero_frames_take_the_eps_branch():
    """All-zero frames: mel energies exactly 0 on both sides, replaced by eps; coefficient 0 is the host's value and the
    others vanish to the DCT's rounding."""
    silence = np.zeros(sc.REF_L, np.float32)
    got = _gpu([silence, CLIPS["tail_zeros"], CLIPS["gap"]], "reference")
    c0 = np.float32(20 * np.log10(sc.REF_LOG_EPS) * sc._DCT[0].sum())
    # a frame is all zero after pre-emphasis when it starts after the last nonzero sample's successor
    zero_frames = {0: range(sc.FRAMES), 1: range(32, sc.FRAMES), 2: range(26, 54)}
    for i, frames in zero_frames.items():
        f = list(frames)
        host = sc.mfcc_reference([silence, CLIPS["tail_zeros"], CLIPS["gap"]][i])
        assert np.array_equal(got[i][0, f], host[0, f])
        assert np.all(np.abs(host[0, f].astype(np.float64) - float(c0)) <= np.spacing(abs(c0)))
        assert np.all(np.abs(got[i][1:, f]) <= 1e-9 * abs(c0))
    _assert_close(got, np.stack([sc.mfcc_reference(w) for w in (silence, CLIPS["tail_zeros"], CLIPS["gap"])]))


def test_engine_recipe_unchanged_on_the_same_clips():
    waves = list(CLIPS.values())
    default = _gpu(waves, "engine")
    n = sc.clip_length("engine")
    w = torch.from_numpy(np.stack([_fit(x, n) for x in waves])).to(DEV)
    t = mfcc_tables(DEV)
    out = torch.full((len(waves), sc.N_MFCC, sc.FRAMES), float("nan"), device=DEV)
    N.mfcc(w, torch.ones(len(waves), dtype=torch.uint8, device=DEV), out, t["window"], t["fb"], t["dct"], t["twiddle"],
           sc.HOP, sc.PREEMPH, sc.LOG_FLOOR)                                   # no recipe argument: today's launch
    assert np.array_equal(out.cpu().numpy(), default)
    _assert_close(default, np.stack([sc.mfcc(x) for x in waves]))
    assert not np.allclose(default, _gpu(waves, "reference"))


def test_invalid_rows_are_zero():
    waves = [CLIPS["noise"], CLIPS["chirp"], CLIPS["square"]]
    got = _gpu(waves, "reference", valid=[0, 1, 0])
    assert not got[0].any() and not got[2].any()
    _assert_close(got[1:2], sc.mfcc_reference(CLIPS["chirp"])[None])


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def test_refusals_write_nothing():
    t = mfcc_tables(DEV, "reference")
    tabs = (t["window"], t["fb"], t["dct"], t["twiddle"])
    w, v = torch.zeros(2, sc.REF_L, device=DEV), torch.ones(2, dtype=torch.uint8, device=DEV)
    out = _nan(2, sc.N_MFCC, sc.FRAMES)
    with pytest.raises(N.NativeError, match="recipe"):
        N.mfcc(w, v, out, *tabs, sc.HOP, sc.PREEMPH, sc.REF_LOG_EPS, recipe="fast")
    from ctypes import c_double, c_int
    p = N._p
    code = N.lib().slb_mfcc(p(w), p(v), p(t["window"]), p(t["fb"]), p(t["dct"]), p(t["twiddle"]), p(out), c_int(2),
                            c_int(sc.REF_L), c_int(sc.REF_WIN), c_int(sc.HOP), c_int(sc.FRAMES), c_int(sc.REF_N_FFT),
                            c_int(sc.N_MELS), c_int(sc.N_MFCC), c_double(sc.PREEMPH), c_double(sc.REF_LOG_EPS), c_int(2),
                            N._stream())
    assert code == -3                                                          # a recipe the library does not know
    with pytest.raises(N.NativeError):                                         # engine-length clips, reference tables
        N.mfcc(torch.zeros(2, sc.clip_length(), device=DEV), v, out, *tabs, sc.HOP, sc.PREEMPH, sc.REF_LOG_EPS,
               recipe="reference")
    # shared memory: 16 nfft + 64 win + 8 * 7 * (nbins + nmels) + 4 * span bytes; 4096-sample frames need ~454 KiB > 227 KiB
    nfft = 4096
    j = torch.arange(nfft, dtype=torch.float64, device=DEV) * (2 * np.pi / nfft)
    big = (torch.ones(nfft, dtype=torch.float64, device=DEV), torch.zeros(sc.N_MELS, nfft // 2 + 1, dtype=torch.float64,
           device=DEV), t["dct"], torch.stack([j.cos(), j.sin()], 1).contiguous())
    for recipe in ("engine", "reference"):
        with pytest.raises(N.NativeError):
            N.mfcc(torch.zeros(2, nfft, device=DEV), v, out[:, :, :1].contiguous(), *big, sc.HOP, sc.PREEMPH,
                   sc.REF_LOG_EPS, recipe=recipe)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


def test_resident_split_matches_host_loader(tmp_path):
    tree = make_tree(tmp_path, per_class=3)
    dist = [100] * 10
    kw = dict(train=True, synthetic=False, root=str(tmp_path), speech_features="reference")
    gpu = data_loader("SPEECHCOMMANDS", 4, dist, device=DEV, gpu_loader=True, **kw)
    host = data_loader("SPEECHCOMMANDS", 4, dist, **kw)
    assert isinstance(gpu, GpuFeatureLoader) and host.dataset.dataset.recipe == "reference"
    got = [(x.cpu().numpy(), int(y)) for xs, ys in gpu for x, y in zip(xs, ys)]
    ref = [(x.numpy(), int(y)) for xs, ys in host for x, y in zip(xs, ys)]
    assert len(got) == len(ref) == len(tree["train"])
    assert sum(not x.any() for x, _ in ref) == 2 and sum(not x.any() for x, _ in got) == 2   # unreadable + stereo
    pool = list(got)
    for x, y in ref:                                                        # match each host sample to one resident sample
        for j, (gx, gy) in enumerate(pool):
            tol = np.spacing(np.abs(x)) + 1e-9 * np.abs(x).max()
            if gy == y and np.all(np.abs(gx.astype(np.float64) - x) <= tol):
                pool.pop(j)
                break
        else:
            raise AssertionError(f"host sample of label {y} has no resident counterpart")
    engine = data_loader("SPEECHCOMMANDS", 4, dist, train=True, synthetic=False, root=str(tmp_path), device=DEV,
                         gpu_loader=True)
    assert not torch.allclose(engine.features.sort(0).values, gpu.features.sort(0).values)


def test_public_api_kwt_reference_features(tmp_path, monkeypatch):
    """One KWT round on a wav tree with ``speech-features: reference``, ``gpu-loader`` and ``validation``: the first stage's
    resident split holds reference features of the training files, and the server validates on the reference test loader."""
    import yaml
    from split_learning_b200 import validation as V
    from split_learning_b200.config import normalize
    from split_learning_b200.runner import run_inproc
    raw = yaml.safe_load(open("config.yaml"))
    tree = make_tree(tmp_path / "data", per_class=3)
    monkeypatch.chdir(tmp_path)                                  # the loaders read ./data
    monkeypatch.setenv("SLB200_WAIT_SPINS", str(1 << 23))
    monkeypatch.delenv("SLB200_SYNTHETIC", raising=False)
    test_loaders = []

    def spy(**kw):
        ld = data_loader(**kw)
        test_loaders.append((kw, ld))
        return ld
    monkeypatch.setattr(V, "data_loader", spy)
    raw["server"].update({"clients": [1, 1], "global-round": 1, "validation": True, "model": "KWT",
                          "data-name": "SPEECHCOMMANDS"})
    raw["server"]["manual"]["no-cluster"]["cut-layers"] = [8]
    raw["server"]["data-distribution"]["num-sample"] = 200
    raw["log_path"] = str(tmp_path)
    raw["learning"].update({"batch-size": 8, "control-count": 3, "learning-rate": 0.001})
    raw["b200"] = {"synthetic-data": False, "gpu-loader": True, "native-tokens": True, "token-graphs": True,
                   "speech-features": "reference", "watchdog-seconds": 120}
    srv = run_inproc(normalize(raw), devices=["cuda:0"], workdir=str(tmp_path), timeout=600)
    assert [h["ok"] for h in srv.history] == [True]
    first = [c for c in srv.clients_objs if c.layer_id == 1][0]
    feats = first.train_loader
    assert isinstance(feats, GpuFeatureLoader) and feats.n == len(tree["train"])
    base = tree["base"]
    host = {}
    for rel, label in tree["train"]:
        try:
            host[rel] = (sc.mfcc_reference(sc.read_wave(os.path.join(base, rel), "reference")), label)
        except Exception:
            host[rel] = (np.zeros((sc.N_MFCC, sc.FRAMES), np.float32), label)
    pool = [(x, int(y)) for x, y in zip(feats.features.cpu().numpy(), feats.labels.cpu())]
    for x, y in host.values():
        hits = [j for j, (gx, gy) in enumerate(pool)
                if gy == y and np.all(np.abs(gx.astype(np.float64) - x) <= np.spacing(np.abs(x)) + 1e-9 * np.abs(x).max())]
        assert hits, "training file without its reference features in the resident split"
        pool.pop(hits[0])
    assert len(test_loaders) == 1
    kw, ld = test_loaders[0]
    assert kw["speech_features"] == "reference" and kw["train"] is False and ld.dataset.recipe == "reference"
    m = srv.history[0]
    assert m.get("val_total") == 10 and np.isfinite(m["val_loss"])
