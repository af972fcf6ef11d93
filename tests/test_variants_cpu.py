"""The five ``other/*`` algorithm variants end to end on CPU (in-process broker)."""
import os

import pytest
import torch
import yaml

from split_learning_b200.algorithms import ALGORITHMS, client_class, server_class
from split_learning_b200.checkpoint import load_checkpoint
from split_learning_b200.config import normalize
from split_learning_b200.runner import run_variant


def _base(tmp, algo, clients, **server):
    raw = {"server": {"global-round": 1, "clients": list(clients), "no-cluster": {"cut-layers": [7]}, "model": "VGG16",
                      "data-name": "CIFAR10", "parameters": {"load": False, "save": True}, "validation": True,
                      "data-distribution": {"non-iid": False, "num-sample": 32, "num-label": 10, "dirichlet": {"alpha": 1}},
                      "random-seed": 1},
           "log_path": str(tmp), "debug_mode": False,
           "learning": {"learning-rate": 0.01, "momentum": 0.5, "batch-size": 8, "control-count": 2, "clip-grad-norm": 1.0},
           "b200": {"algorithm": algo, "synthetic-data": True, "watchdog-seconds": 60}}
    raw["server"].update(server)
    return raw


def test_registry():
    for a in ALGORITHMS:
        assert server_class(a).ALGORITHM in (a, "main") or a == "main"
        assert client_class(a) is not None


def test_vanilla_sl_sequential_handoff(tmp_path):
    cfg = normalize(_base(tmp_path, "vanilla_sl", (2, 1)))
    srv = run_variant(cfg, [dict(layer_id=1), dict(layer_id=1), dict(layer_id=2)], workdir=str(tmp_path))
    assert srv.history and srv.history[0]["ok"] and len(srv.groups) == 2
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97


def test_cluster_fsl(tmp_path):
    cfg = normalize(_base(tmp_path, "cluster_fsl", (2, 1), **{"manual-cluster": {"num-cluster": 2, "cut-layers": [[7], [7]]}}))
    srv = run_variant(cfg, [dict(layer_id=1, cluster=0), dict(layer_id=1, cluster=1), dict(layer_id=2, cluster=0)],
                      workdir=str(tmp_path))
    assert srv.history[0]["ok"] and [len(g) for g in srv.groups] == [1, 1]


def test_dcsl_sda_and_local_round(tmp_path):
    cfg = normalize(_base(tmp_path, "dcsl", (2, 1), **{"local-round": 2}))
    srv = run_variant(cfg, [dict(layer_id=1, cluster=0), dict(layer_id=1, cluster=0), dict(layer_id=2, cluster=0)],
                      workdir=str(tmp_path))
    assert srv.history[0]["ok"]
    sd = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    # 2 local epochs x 4 batches per client, SDA concatenates the two clients' batches on the last stage
    assert int(sd["layer9.num_batches_tracked"]) == 2 * 4


def test_flex_multirate(tmp_path):
    raw = _base(tmp_path, "flex", (2, 2), **{"global-round": 2, "t-g": 2, "t-c": 1, "num-cluster": 2, "cut-layer": [7, 4]})
    del raw["server"]["no-cluster"]
    cfg = normalize(raw)
    assert cfg.cluster_cut_layers == [[7], [4]]
    srv = run_variant(cfg, [dict(layer_id=1, cluster=0, select=1), dict(layer_id=1, cluster=1, select=1),
                            dict(layer_id=2, cluster=0), dict(layer_id=2, cluster=1)], workdir=str(tmp_path))
    assert len(srv.history) == 2 and all(h["ok"] for h in srv.history)
    assert "val_acc" in srv.history[1] and "val_acc" not in srv.history[0]      # edges upload every t-g = 2 rounds
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97


def test_two_ls_fedasync(tmp_path):
    raw = _base(tmp_path, "2ls", (2, 1), **{"num-cluster": 1, "cut-layer": 7, "info-cluster": [[2, 1]]})
    del raw["server"]["no-cluster"]
    cfg = normalize(raw)
    srv = run_variant(cfg, [dict(layer_id=1, idx=0, in_cluster=0, out_cluster=0),
                            dict(layer_id=1, idx=0, in_cluster=0, out_cluster=1),
                            dict(layer_id=2, idx=0, in_cluster=0, out_cluster=0)], workdir=str(tmp_path))
    assert srv.history[0]["ok"] and sorted(srv.out_ids) == [0, 1]
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97


def test_vanilla_sl_limited_time_mode(tmp_path):
    """``limited-time``: the first stage keeps looping epochs until the wall-clock budget is spent
    (other/Vanilla_SL/src/Scheduler.py:68-69,77,108-115), instead of exactly one pass."""
    raw = _base(tmp_path, "vanilla_sl", (1, 1), **{"limited-time": {"enable": True, "epoch": 50, "time": 4.0}})
    raw["server"]["validation"] = False
    cfg = normalize(raw)
    assert cfg.limited_time == {"enable": True, "epoch": 50, "time": 4.0}
    srv = run_variant(cfg, [dict(layer_id=1), dict(layer_id=2)], workdir=str(tmp_path))
    assert srv.history[0]["ok"]
    sd = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    one_epoch = 32 // 8                                   # 32 samples / batch 8
    assert int(sd["layer9.num_batches_tracked"]) > one_epoch          # more than one pass fitted into the budget
    assert int(sd["layer9.num_batches_tracked"]) % one_epoch == 0     # the budget is checked at epoch boundaries


def test_flex_unselected_device_is_dropped(tmp_path):
    """FLEX ``--s 0``: an un-selected first-stage device is rejected at registration (other/FLEX/src/Server.py:270-285);
    the round runs with the remaining devices."""
    raw = _base(tmp_path, "flex", (2, 1), **{"t-g": 1, "t-c": 1, "num-cluster": 1, "cut-layer": [7]})
    del raw["server"]["no-cluster"]
    cfg = normalize(raw)
    srv = run_variant(cfg, [dict(layer_id=1, cluster=0, select=1), dict(layer_id=1, cluster=0, select=0),
                            dict(layer_id=2, cluster=0)], workdir=str(tmp_path))
    assert srv.history and srv.history[0]["ok"]
    assert srv.total_clients[0] == 1
    trained = [c for c in srv.clients if c.layer_id == 1 and c.train]
    assert len(trained) == 1 and sum(trained[0].label_counts) > 0
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97
