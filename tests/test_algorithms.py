import numpy as np
import pytest
import torch

from split_learning_b200.checkpoint import load_checkpoint, merge_stages, save_checkpoint, slice_for_stage
from split_learning_b200.data import label_counts
from split_learning_b200.fedavg import fedasync_merge, fedavg_state_dicts
from split_learning_b200.models import VGG16_CIFAR10
from split_learning_b200.planning import auto_threshold, clustering_algorithm, gmm_1d, kmeans, partition, partition_multi

from oracle_cases import CLUSTER_SEED, PARTITION_CASES, SELECTION_SEED, as_tensor, fedavg_inputs, layout_digest, load_json

# answers of the reference implementation (src/Utils.py, src/Partition.py, src/Cluster.py, src/Selection.py) on the same
# inputs, recorded by tools/make_golden.py
ORACLE = load_json("algorithms.json")


def test_fedavg_matches_reference():
    dicts = fedavg_inputs()
    for w in (None, [3, 1, 7]):
        mine = fedavg_state_dicts(dicts, w)
        oracle = {k: as_tensor(v) for k, v in ORACLE["fedavg"][str(w)].items()}
        assert set(mine) == set(oracle)
        for k in mine:
            assert mine[k].dtype == oracle[k].dtype
            assert torch.allclose(mine[k].float(), oracle[k].float(), atol=1e-6), k


def test_fedavg_int_rounding_and_empty():
    out = fedavg_state_dicts([{"n": torch.tensor(3)}, {"n": torch.tensor(4)}], [1, 1])
    assert out["n"].dtype == torch.int64 and out["n"].item() == 4   # round-half-even of 3.5
    assert fedavg_state_dicts([]) == {}


def test_fedasync():
    g = {"w": torch.ones(3)}
    n = {"w": torch.zeros(3), "x": torch.ones(1)}
    m = fedasync_merge(g, n, 0.25)
    assert torch.allclose(m["w"], torch.full((3,), 0.75)) and "x" in m
    assert torch.equal(fedasync_merge(None, n, 0.5)["w"], n["w"])


def test_partition_matches_reference():
    cases = PARTITION_CASES()
    assert len(cases) == len(ORACLE["partition"]) == 20
    for case, theirs in zip(cases, ORACLE["partition"]):
        assert partition(*case) == theirs


def test_partition_multi():
    e = [[[1.0] * 12], [[1.0] * 12], [[1.0] * 12]]
    cuts = partition_multi(e, [[1e9]] * 3, [1.0] * 12)
    assert cuts == [4, 8]
    assert partition_multi(e[:2], [[1e9]] * 2, [1.0] * 12) == partition(e[0], [1e9], e[1], [1e9], [1.0] * 12)


def test_clustering_matches_reference():
    rng = np.random.RandomState(CLUSTER_SEED)
    a = np.concatenate([rng.dirichlet([10, 1, 1, 1], 6), rng.dirichlet([1, 1, 10, 10], 5)]) * 500
    lm, im = clustering_algorithm(a, 2)
    lt = ORACLE["clustering"]["labels"]
    assert (np.asarray(lm) == np.asarray(lt)).all() and im == ORACLE["clustering"]["infos"]
    # dependency-free path finds the same partition (up to relabelling)
    lk, _ = kmeans(a / a.sum(1, keepdims=True), 2)
    assert len(set(zip(lk.tolist(), np.asarray(lt).tolist()))) == 2


def test_selection_threshold():
    rng = np.random.RandomState(SELECTION_SEED)
    perf = np.concatenate([rng.normal(100, 5, 12), rng.normal(1000, 40, 10)]).clip(1)
    t_mine, t_ref = auto_threshold(perf), ORACLE["selection_threshold"]
    assert abs(np.log(t_mine) - np.log(t_ref)) < 1e-6
    t_own = auto_threshold(perf, backend="own")
    assert 130 < t_own < 800 and abs(np.log(t_own) - np.log(t_ref)) < 0.35
    assert auto_threshold([5.0]) == 0.0
    mu, var, w = gmm_1d(np.log(perf))
    assert abs(w.sum() - 1) < 1e-9


def test_label_counts():
    iid = label_counts(3, 10, 5000)
    assert iid.shape == (3, 10) and (iid == 500).all()
    d1, d2 = label_counts(4, 10, 5000, True, 1.0, seed=7), label_counts(4, 10, 5000, True, 1.0, seed=7)
    assert (d1 == d2).all() and d1.shape == (4, 10) and (d1.sum(1) <= 5000).all() and (d1.sum(1) > 4900).all()
    r = label_counts(2, 10, 1000, True, seed=1, non_iid_rate=0.5)
    assert r.shape == (2, 10) and r.sum() <= 2000 and r.max() > r.min()


def test_checkpoint_slice_merge_roundtrip(tmp_path):
    torch.manual_seed(0)
    full = VGG16_CIFAR10().state_dict()
    p = str(tmp_path / "VGG16_CIFAR10.pth")
    save_checkpoint(full, p, meta={"round": 3})
    loaded = load_checkpoint(p)
    parts = [slice_for_stage(loaded, "VGG16", "CIFAR10", l) for l in ([0, 5], [5, 10], [10, -1])]
    merged = merge_stages(parts)
    assert set(merged) == set(full) and all(torch.equal(merged[k], full[k]) for k in full)
    # the reference's own class can load our checkpoint (layout compatibility): the strict load_state_dict check against
    # the reference model's recorded keys, shapes and dtypes
    theirs = load_json("models.json")["layouts"]["VGG16_CIFAR10"][f"0,{VGG16_CIFAR10.num_layers()}"]
    assert layout_digest(torch.load(p, weights_only=True)) == theirs
    assert load_checkpoint(str(tmp_path / "missing.pth")) is None


def test_variant_label_matrices():
    from split_learning_b200.data.distribution import preset_matrix
    flex = label_counts(9, 4, 5000, True, matrix="flex")
    # other/FLEX/src/Server.py:81-90: 75 % dominant label (0,1,0,1,2,1,2,0,2) + 25 % of the last label
    assert flex.shape == (9, 4) and flex[0].tolist() == [3750, 0, 0, 1250] and flex[4].tolist() == [0, 0, 3750, 1250]
    two = preset_matrix("2ls", 9, 10)
    assert np.allclose(two.sum(1), 1.0) and two[0, :4].tolist() == [0.3, 0.3, 0.3, 0.1]
    explicit = label_counts(3, 2, 100, True, matrix=[[1.0, 0.0], [0.5, 0.5]])
    assert explicit.tolist() == [[100, 0], [50, 50], [100, 0]]


def test_flex_speed_profile(tmp_path):
    """other/FLEX/profiling.py: whole-model samples/s only."""
    from split_learning_b200.profiler import write_speed_profile
    info = write_speed_profile("KWT", 2, str(tmp_path / "profiling.json"), None, rounds=2)
    assert set(info) == {"speed"} and info["speed"] > 0
    info = write_speed_profile("VGG16", 2, str(tmp_path / "p2.json"), "CIFAR10", rounds=1)
    assert info["speed"] > 0


def test_validation_gate_and_heartbeat_pump():
    """``get_val``: the main tree always passes (src/val/get_val.py), the Vanilla_SL gate fails the round on a NaN / huge
    loss (other/Vanilla_SL/src/Validation.py:46,55-56); ``pump`` is called every 5 batches (DCSL's heartbeat hook)."""
    import math
    import torch
    from split_learning_b200.models import get_model_class
    from split_learning_b200.validation import get_val
    torch.manual_seed(0)
    sd = get_model_class("KWT", "SPEECHCOMMANDS")().state_dict()
    beats = []
    ok, m = get_val("KWT", "SPEECHCOMMANDS", sd, strict=True, device="cpu", pump=lambda: beats.append(1), synthetic=True)
    assert ok and m["val_total"] > 0 and 0.0 <= m["val_acc"] <= 100.0 and len(beats) == (m["val_total"] // 20) // 5
    bad = {k: v.clone() for k, v in sd.items()}
    bad["layer1.weight"][0, 0] = float("nan")
    ok_main, m_main = get_val("KWT", "SPEECHCOMMANDS", bad, strict=False, device="cpu", synthetic=True)
    ok_strict, _ = get_val("KWT", "SPEECHCOMMANDS", bad, strict=True, device="cpu", synthetic=True)
    assert ok_main and math.isnan(m_main["val_loss"]) and not ok_strict
    assert get_val("NOPE", "CIFAR10", {}, device="cpu") == (False, {})


def test_batched_tensor_loader_contract():
    """``BatchedTensorLoader`` = ``DataLoader(ds, batch_size, shuffle, drop_last=False)`` for an in-memory dataset: every sample
    exactly once per epoch, the short batch last, a new permutation every epoch, per-client seeds, exact per-label counts;
    pinned staging is capped (long epochs yield pageable tensors and the consumer stages through its own bounded ring)."""
    from split_learning_b200.data.loaders import BatchedTensorLoader, SyntheticDataset, data_loader
    counts = [7, 0, 13, 5, 0, 0, 9, 1, 0, 3]
    ds = SyntheticDataset("CIFAR10", counts, seed=3)
    assert len(ds) == sum(counts) and torch.bincount(ds.labels, minlength=10).tolist() == counts
    ld = BatchedTensorLoader(ds, 8, shuffle=True, pin=False, seed=3)
    assert len(ld) == 5 and ld.batch_size == 8 and ld.drop_last is False
    epochs = []
    for _ in range(2):
        xs, ys, sizes = [], [], []
        for x, y in ld:
            assert x.shape[1:] == (3, 32, 32) and x.dtype == torch.float32 and y.dtype == torch.long
            xs.append(x), ys.append(y), sizes.append(x.shape[0])
        assert sizes == [8, 8, 8, 8, 6]                                   # the short batch comes last
        x, y = torch.cat(xs), torch.cat(ys)
        assert torch.bincount(y, minlength=10).tolist() == counts            # every sample once
        key = x.flatten(1).sum(1)
        assert torch.allclose(key.sort().values, ds.data.flatten(1).sum(1).sort().values)
        epochs.append(y)
    assert not torch.equal(epochs[0], epochs[1])                              # reshuffled
    fixed = BatchedTensorLoader(ds, 8, shuffle=False)
    assert torch.equal(torch.cat([y for _, y in fixed]), ds.labels)
    # different clients draw different samples; validation never re-draws the training stream
    a = data_loader("CIFAR10", 8, counts, train=True, synthetic=True, seed=1).dataset.data
    b = data_loader("CIFAR10", 8, counts, train=True, synthetic=True, seed=2).dataset.data
    v = data_loader("CIFAR10", 8, counts, train=False, synthetic=True, seed=1).dataset.data
    assert not torch.equal(a, b) and not torch.equal(a[: len(v)], v[: len(a)])
    long_epoch = BatchedTensorLoader(SyntheticDataset("MNIST", [60] * 10, seed=0), 1, pin=True)
    assert len(long_epoch) == 600 > BatchedTensorLoader.MAX_PINNED_BATCHES and long_epoch.pin is False
