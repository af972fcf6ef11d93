"""GPU-resident Speech Commands loader (``b200.gpu-loader`` for KWT): the fp64 MFCC kernel against the host recipe
``speechcommands.mfcc()``, the per-microbatch gather, the loader's iteration contract, the real-data path on a small wav
tree, and one KWT round through the public API."""
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
L = sc.WIN + sc.HOP * (sc.FRAMES - 1)
DIST = [9, 4, 7, 3, 5, 8, 2, 6, 4, 5]


def _fit(w, n=L):
    w = np.asarray(w, np.float32).ravel()[:n]
    return np.pad(w, (0, n - w.size))


def _assert_close(got, ref):
    """|gpu - ref| <= ulp32(ref) + 1e-9 * max|ref| of the clip: two fp64 pipelines, each rounded to fp32 once."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    for g, r in zip(got, ref, strict=True):
        tol = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64) + 1e-9 * np.abs(r).max()
        err = np.abs(g - r)
        assert np.all(err <= tol), f"max error {err.max():.3e} at {np.unravel_index(err.argmax(), err.shape)}"


def _gpu_mfcc(waves, valid=None):
    w = torch.from_numpy(np.stack([_fit(x) for x in waves])).to(DEV)
    v = torch.ones(len(waves), dtype=torch.uint8, device=DEV) if valid is None else torch.tensor(valid, dtype=torch.uint8,
                                                                                                 device=DEV)
    return mfcc_features(w, v, mfcc_tables(DEV)).cpu().numpy()


def _inputs():
    rng = np.random.default_rng(0)
    t = np.arange(L) / sc.SAMPLE_RATE
    sweep = (0.6 * np.sin(2 * np.pi * (50.0 * t + 0.5 * 7900.0 / t[-1] * t * t))).astype(np.float32)
    noise = (rng.standard_normal(L) * 0.1).astype(np.float32)
    square = np.where((np.arange(L) // 40) % 2 == 0, 32767, -32768).astype(np.int16).astype(np.float32) / 32768.0
    silence = np.zeros(L, np.float32)
    short = (rng.standard_normal(7000) * 0.2).astype(np.float32)
    long = (rng.standard_normal(L + 4321) * 0.2).astype(np.float32)
    return {"sweep": sweep, "noise": noise, "square": square, "silence": silence, "short": short, "long": long}


@pytest.mark.parametrize("name", list(_inputs()))
def test_mfcc_matches_host_recipe(name):
    w = _inputs()[name]
    _assert_close(_gpu_mfcc([w]), sc.mfcc(w)[None])


def test_mfcc_silence_is_the_log_floor():
    got = _gpu_mfcc([np.zeros(L, np.float32)])[0]
    ref = sc.mfcc(np.zeros(L, np.float32))
    assert np.isclose(ref[0, 0], np.log(sc.LOG_FLOOR) * sc._DCT[0].sum(), rtol=1e-6)
    _assert_close(got[None], ref[None])


@pytest.mark.parametrize("n", [1, 5, 13])
def test_mfcc_batch(n):
    rng = np.random.default_rng(n)
    waves = [(rng.standard_normal(int(rng.integers(3000, L + 3000))) * rng.uniform(0.01, 0.5)).astype(np.float32)
             for _ in range(n)]
    _assert_close(_gpu_mfcc(waves), np.stack([sc.mfcc(w) for w in waves]))


def _ref_geometry(wave, frames):
    """``mfcc()`` with another number of frames (the kernel takes the frame geometry as arguments)."""
    need = sc.WIN + sc.HOP * (frames - 1)
    w = np.pad(np.asarray(wave, np.float64), (0, max(0, need - wave.size)))[:need]
    w = np.append(w[0], w[1:] - sc.PREEMPH * w[:-1])
    fr = w[np.arange(sc.WIN)[None, :] + sc.HOP * np.arange(frames)[:, None]] * sc._WINDOW
    power = (np.abs(np.fft.rfft(fr, sc.N_FFT)) ** 2) / sc.N_FFT
    return (np.log(np.maximum(power @ sc._FB.T, sc.LOG_FLOOR)) @ sc._DCT.T).T.astype(np.float32)


@pytest.mark.parametrize("frames", [1, 10, 15])
def test_mfcc_frames_not_a_multiple_of_the_group(frames):
    rng = np.random.default_rng(frames)
    n_s = sc.WIN + sc.HOP * (frames - 1)
    waves = np.stack([(rng.standard_normal(n_s) * 0.3).astype(np.float32) for _ in range(3)])
    t = mfcc_tables(DEV)
    out = torch.full((3, sc.N_MFCC, frames), float("nan"), device=DEV)
    N.mfcc(torch.from_numpy(waves).to(DEV), torch.ones(3, dtype=torch.uint8, device=DEV), out, t["window"], t["fb"], t["dct"],
           t["twiddle"], sc.HOP, sc.PREEMPH, sc.LOG_FLOOR)
    _assert_close(out.cpu().numpy(), np.stack([_ref_geometry(w, frames) for w in waves]))


def test_mfcc_invalid_rows_are_zero():
    w = _inputs()
    waves = [w["noise"], w["sweep"], w["square"], w["long"]]
    got = _gpu_mfcc(waves, valid=[1, 0, 1, 0])
    assert not got[1].any() and not got[3].any()
    _assert_close(got[[0, 2]], np.stack([sc.mfcc(waves[0]), sc.mfcc(waves[2])]))


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def test_mfcc_refusals_write_nothing():
    t = mfcc_tables(DEV)
    tabs = (t["window"], t["fb"], t["dct"], t["twiddle"])
    ok_w, ok_v = torch.zeros(2, L, device=DEV), torch.ones(2, dtype=torch.uint8, device=DEV)
    base = _nan(3, sc.N_MFCC, sc.FRAMES)
    cases = {
        "short rows": (torch.zeros(2, L - 4, device=DEV), ok_v, base[:2]),
        "misaligned waves": (torch.zeros(2 * L + 1, device=DEV)[1:].view(2, L), ok_v, base[:2]),
        "n = 0": (torch.zeros(0, L, device=DEV), ok_v[:0], base[:0]),
        "out rows": (ok_w, ok_v, base),
    }
    for what, (w, v, out) in cases.items():
        with pytest.raises(N.NativeError):
            N.mfcc(w, v, out, *tabs, sc.HOP, sc.PREEMPH, sc.LOG_FLOOR)
        torch.cuda.synchronize()
        assert torch.isnan(base).all(), what
    out = _nan(2, sc.N_MFCC, sc.FRAMES)
    with pytest.raises(N.NativeError):                       # hop inconsistent with L and frames
        N.mfcc(ok_w, ok_v, out, *tabs, sc.HOP + 4, sc.PREEMPH, sc.LOG_FLOOR)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


@pytest.mark.parametrize("b", [1, 20, 32, 7])
def test_feature_batch_is_index_select(b):
    g = torch.Generator(device=DEV).manual_seed(b)
    feats = torch.randn(50, sc.N_MFCC, sc.FRAMES, device=DEV, generator=g)
    labels = torch.randint(0, 10, (50,), device=DEV, generator=g)
    idx = torch.randperm(50, device=DEV, generator=g)[:b] if b != 7 else torch.arange(43, 50, device=DEV)
    x, y = _nan(b, sc.N_MFCC, sc.FRAMES), torch.full((b,), -1, dtype=torch.long, device=DEV)
    N.feature_batch(feats, labels, idx, x, y)
    assert torch.equal(x, feats.index_select(0, idx)) and torch.equal(y, labels.index_select(0, idx))


def test_feature_batch_refusals_write_nothing():
    feats, labels = torch.randn(10, 8, device=DEV), torch.arange(10, device=DEV)
    idx = torch.arange(4, device=DEV)
    y = torch.full((4,), -1, dtype=torch.long, device=DEV)
    base = _nan(4 * 12 + 1)
    for what, (f, i, out) in {"misaligned out": (feats, idx, base[1:33].view(4, 8)),
                              "B = 0": (feats, idx[:0], base[:0].view(0, 8)),
                              "row not a multiple of 4": (torch.randn(10, 6, device=DEV), idx, base[:24].view(4, 6)),
                              "row mismatch": (feats, idx, base[:48].view(4, 12))}.items():
        with pytest.raises(N.NativeError):
            N.feature_batch(f, labels, i, out, y[:i.numel()])
        torch.cuda.synchronize()
        assert torch.isnan(base).all() and (y == -1).all(), what


def test_loader_contract():
    n, bs = 103, 32
    feats = torch.randn(n, sc.N_MFCC, sc.FRAMES)
    feats[:, 0, 0] = torch.arange(n, dtype=torch.float32)              # sample id
    labels = torch.randint(0, 10, (n,))
    ld = GpuFeatureLoader(feats, labels, bs, DEV, seed=11)
    assert len(ld) == 4 and ld.features.is_cuda
    orders = []
    for _ in range(2):
        batches = list(ld)
        assert len(batches) == len(ld) and [x.shape[0] for x, _ in batches] == [32, 32, 32, 7]
        ids = torch.cat([x[:, 0, 0] for x, _ in batches]).long().cpu()
        assert torch.equal(ids.sort().values, torch.arange(n))
        assert torch.equal(torch.cat([y for _, y in batches]).cpu(), labels[ids])
        assert all(x.is_cuda and x.dtype == torch.float32 and y.dtype == torch.long for x, y in batches)
        orders.append(ids)
    assert not torch.equal(orders[0], orders[1])
    other = torch.cat([x[:, 0, 0] for x, _ in GpuFeatureLoader(feats, labels, bs, DEV, seed=12)]).long().cpu()
    assert not torch.equal(other, orders[0])
    fixed = torch.cat([x[:, 0, 0] for x, _ in GpuFeatureLoader(feats, labels, bs, DEV, shuffle=False)]).long().cpu()
    assert torch.equal(fixed, torch.arange(n))


def test_synthetic_resident_split_is_the_host_synthetic_data():
    gpu = data_loader("SPEECHCOMMANDS", 32, DIST, train=True, synthetic=True, seed=5, device=DEV, gpu_loader=True)
    host = data_loader("SPEECHCOMMANDS", 32, DIST, train=True, synthetic=True, seed=5, device=DEV, gpu_loader=False)
    assert isinstance(gpu, GpuFeatureLoader)
    assert torch.equal(gpu.features.cpu(), host.dataset.data) and torch.equal(gpu.labels.cpu(), host.dataset.labels)
    assert len(gpu) == len(host) and sum(x.shape[0] for x, _ in gpu) == sum(DIST)


def test_real_data_same_samples_as_host_loader(tmp_path):
    tree = make_tree(tmp_path, per_class=3)
    dist = [100] * 10                                                      # every training clip of every class
    gpu = data_loader("SPEECHCOMMANDS", 4, dist, train=True, synthetic=False, root=str(tmp_path), device=DEV,
                      gpu_loader=True)
    host = data_loader("SPEECHCOMMANDS", 4, dist, train=True, synthetic=False, root=str(tmp_path))
    assert isinstance(gpu, GpuFeatureLoader) and len(gpu) == len(host)
    got = [(x.cpu().numpy(), int(y)) for xs, ys in gpu for x, y in zip(xs, ys)]
    ref = [(x.numpy(), int(y)) for xs, ys in host for x, y in zip(xs, ys)]
    assert len(got) == len(ref) == len(tree["train"])
    assert sorted(y for _, y in got) == sorted(y for _, y in ref)
    zero_rows = sum(not x.any() for x, _ in ref)
    assert zero_rows == 1 and sum(not x.any() for x, _ in got) == 1           # the unreadable file
    pool = list(got)
    for x, y in ref:                                                        # match each host sample to one resident sample
        for j, (gx, gy) in enumerate(pool):
            tol = np.spacing(np.abs(x)) + 1e-9 * np.abs(x).max()
            if gy == y and np.all(np.abs(gx.astype(np.float64) - x) <= tol):
                pool.pop(j)
                break
        else:
            raise AssertionError(f"host sample of label {y} has no resident counterpart")


def test_public_api_kwt_gpu_resident_loader(tmp_path, monkeypatch):
    """One KWT round with ``b200.gpu-loader``: the first stage trains from the resident split."""
    import yaml
    monkeypatch.setenv("SLB200_WAIT_SPINS", str(1 << 23))
    from split_learning_b200.checkpoint import load_checkpoint
    from split_learning_b200.config import normalize
    from split_learning_b200.runner import run_inproc
    raw = yaml.safe_load(open("config.yaml"))
    raw["server"].update({"clients": [1, 1], "global-round": 1, "validation": False, "model": "KWT",
                          "data-name": "SPEECHCOMMANDS"})
    raw["server"]["manual"]["no-cluster"]["cut-layers"] = [8]
    raw["server"]["data-distribution"]["num-sample"] = 320
    raw["log_path"] = str(tmp_path)
    raw["learning"].update({"batch-size": 32, "control-count": 3, "learning-rate": 0.001})
    raw["b200"] = {"synthetic-data": True, "gpu-loader": True, "native-tokens": True, "token-graphs": True,
                   "watchdog-seconds": 120}
    srv = run_inproc(normalize(raw), devices=["cuda:0"], workdir=str(tmp_path), timeout=600)
    assert [h["ok"] for h in srv.history] == [True]
    first = [c for c in srv.clients_objs if c.layer_id == 1][0]
    last = [c for c in srv.clients_objs if c.layer_id == 2][0]
    assert isinstance(first.train_loader, GpuFeatureLoader) and first.train_loader.features.is_cuda
    assert tuple(first.train_loader.features.shape) == (320, sc.N_MFCC, sc.FRAMES)
    loss = last.executor.last_loss()
    assert loss is not None and np.isfinite(float(loss))
    sd = load_checkpoint(str(tmp_path / "KWT_SPEECHCOMMANDS.pth"))
    assert all(torch.isfinite(v.float()).all() for v in sd.values())
