"""``config.yaml`` loader / normaliser.

Accepts the *actual* main-tree schema (reference config.yaml:1-55), the README-era keys
(README.md:75-132: ``no-cluster``/``cluster`` at server level, ``non-iid-rate``,
``local-round``) and the per-variant keys (SURVEY §5: ``limited-time.*``, ``clip-grad-norm``,
``local-round``, ``manual-cluster.*``, ``t-g``, ``t-c``, ``select-ratio``, ``cut-layer``,
``info-cluster``, ``lr-decay``, ``lr-step``, ``refresh-each-round``), and produces one
canonical ``Config`` object.  ``rabbit.*`` is tolerated and ignored: the transport here is
an in-box broker, not RabbitMQ.  A ``b200:`` section carries engine-specific knobs.
"""
from __future__ import annotations

import copy
import os
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import yaml

DEFAULT_LEARNING = {
    "learning-rate": 0.0005, "weight-decay": 0.01, "momentum": 0.5,
    "batch-size": 32, "control-count": 3, "clip-grad-norm": 0.0,
}

DEFAULT_B200 = {
    # "auto" → sm_90a kernels on CUDA, reference-math torch executor on CPU
    "executor": "auto",
    # faithful = recompute forward at backward time on non-last stages (reference semantics,
    # src/train/VGG16.py:89-92); "stash" keeps activations instead
    "recompute": True,
    "wire-dtype": "bf16",          # cut-edge payload dtype on the device data plane
    "compute-dtype": "bf16",
    "algorithm": "main",           # main | vanilla_sl | cluster_fsl | dcsl | flex | 2ls
    "transport": "auto",           # inproc | tcp | auto
    "port": 29777,
    "watchdog-seconds": 120.0,     # replaces the reference's silent deadlock
    "synthetic-data": False,
    "routing": "round-robin",      # competing-consumer emulation on the device plane
    "data-plane": "host",          # host = broker queues (any device) | device = peer-memory mailboxes (CUDA)
}


def _get(d: Dict, *path, default=None):
    cur = d
    for p in path:
        if not isinstance(cur, dict) or p not in cur:
            return default
        cur = cur[p]
    return cur


@dataclass
class Config:
    raw: Dict[str, Any]
    # ---- server ----
    global_round: int = 1
    clients: List[int] = field(default_factory=lambda: [1, 1])
    auto_mode: bool = False
    model: str = "VGG16"
    data_name: str = "CIFAR10"
    load_parameters: bool = True
    save_parameters: bool = True
    validation: bool = True
    # data distribution
    non_iid: bool = False
    num_sample: int = 5000
    num_label: int = 10
    dirichlet_alpha: float = 1.0
    non_iid_rate: Optional[float] = None
    label_matrix: Any = None            # explicit per-client label probabilities, or a preset name ("flex" / "2ls")
    refresh: bool = True
    random_seed: Optional[int] = 1
    # topology
    cluster_mode: bool = False
    no_cluster_cut_layers: List[int] = field(default_factory=lambda: [7])
    num_cluster: int = 1
    cluster_cut_layers: List[List[int]] = field(default_factory=lambda: [[7]])
    infor_cluster: List[List[int]] = field(default_factory=lambda: [[1, 1]])
    infor_cluster_given: bool = False   # False → membership comes from client --cluster flags
    # auto mode
    sel_num_cluster: int = 1
    algorithm_cluster: str = "KMeans"
    selection_mode: bool = False
    # variants
    limited_time: Dict[str, Any] = field(default_factory=lambda: {"enable": False, "epoch": 10, "time": 10})
    local_round: int = 1
    t_g: int = 1
    t_c: int = 1
    select_ratio: Optional[float] = None
    lr_decay: Optional[float] = None
    lr_step: Optional[int] = None
    # misc
    log_path: str = "."
    debug_mode: bool = True
    learning: Dict[str, Any] = field(default_factory=lambda: dict(DEFAULT_LEARNING))
    b200: Dict[str, Any] = field(default_factory=lambda: dict(DEFAULT_B200))
    warnings: List[str] = field(default_factory=list)

    # ------------------------------------------------------------------
    @property
    def num_stages(self) -> int:
        return len(self.clients)

    @property
    def total_clients(self) -> int:
        return sum(self.clients)

    def cut_layers_for_cluster(self, c: int) -> List[int]:
        if self.cluster_mode:
            return list(self.cluster_cut_layers[c])
        return list(self.no_cluster_cut_layers)

    def to_dict(self) -> Dict[str, Any]:
        """Round-trip to the main-tree YAML schema."""
        return {
            "name": self.raw.get("name", "Split Learning"),
            "server": {
                "global-round": self.global_round, "clients": list(self.clients),
                "auto-mode": self.auto_mode, "model": self.model, "data-name": self.data_name,
                "parameters": {"load": self.load_parameters, "save": self.save_parameters},
                "validation": self.validation,
                "data-distribution": {
                    "non-iid": self.non_iid, "num-sample": self.num_sample, "num-label": self.num_label,
                    "dirichlet": {"alpha": self.dirichlet_alpha}, "refresh": self.refresh},
                "random-seed": self.random_seed,
                "manual": {
                    "cluster-mode": self.cluster_mode,
                    "no-cluster": {"cut-layers": list(self.no_cluster_cut_layers)},
                    "cluster": dict(
                        {"num-cluster": self.num_cluster,
                         "cut-layers": copy.deepcopy(self.cluster_cut_layers)},
                        **({"infor-cluster": copy.deepcopy(self.infor_cluster)}
                           if self.infor_cluster_given else {}))},
                "cluster-selection": {"num-cluster": self.sel_num_cluster,
                                      "algorithm-cluster": self.algorithm_cluster,
                                      "selection-mode": self.selection_mode},
            },
            "rabbit": self.raw.get("rabbit", {"address": "127.0.0.1", "username": "admin",
                                              "password": "admin", "virtual-host": "/"}),
            "log_path": self.log_path, "debug_mode": self.debug_mode,
            "learning": dict(self.learning), "b200": dict(self.b200),
        }


def normalize(raw: Dict[str, Any]) -> Config:
    raw = copy.deepcopy(raw or {})
    s = raw.get("server", {}) or {}
    cfg = Config(raw=raw)
    cfg.global_round = int(s.get("global-round", 1))
    cfg.clients = [int(x) for x in s.get("clients", [1, 1])]
    cfg.auto_mode = bool(s.get("auto-mode", False))
    cfg.model = s.get("model", "VGG16")
    cfg.data_name = s.get("data-name", "CIFAR10")
    cfg.load_parameters = bool(_get(s, "parameters", "load", default=True))
    cfg.save_parameters = bool(_get(s, "parameters", "save", default=True))
    cfg.validation = bool(s.get("validation", True))

    dd = s.get("data-distribution", {}) or {}
    cfg.non_iid = bool(dd.get("non-iid", False))
    cfg.num_sample = int(dd.get("num-sample", 5000))
    cfg.num_label = int(dd.get("num-label", 10))
    cfg.dirichlet_alpha = float(_get(dd, "dirichlet", "alpha", default=1))
    cfg.non_iid_rate = dd.get("non-iid-rate", s.get("non-iid-rate"))
    cfg.label_matrix = dd.get("label-matrix")
    cfg.refresh = bool(dd.get("refresh", dd.get("refresh-each-round", True)))
    cfg.random_seed = s.get("random-seed", 1)

    # topology: main tree 'manual', README-era / variant top-level keys
    manual = s.get("manual") or {}
    mc = s.get("manual-cluster") or {}          # Cluster_FSL / DCSL
    n_cut = len(cfg.clients) - 1
    cfg.cluster_mode = bool(manual.get("cluster-mode", False))
    nc = manual.get("no-cluster") or s.get("no-cluster") or {}
    cut = nc.get("cut-layers", s.get("cut-layers", s.get("cut-layer")))
    if cut is None:
        cut = [7] * n_cut if n_cut == 1 else []
    if isinstance(cut, int):
        cut = [cut] * max(n_cut, 1)             # 2LS: one scalar cut for every cluster
    cl = dict(manual.get("cluster") or mc or (s.get("cluster") if isinstance(s.get("cluster"), dict) else {}) or {})
    top_nc = s.get("num-cluster")
    per_cluster = None
    if cut and isinstance(cut[0], (list, tuple)):
        per_cluster = [list(map(int, c)) for c in cut]
    elif top_nc and len(cut) == int(top_nc) and len(cut) != n_cut:
        per_cluster = [[int(c)] for c in cut]   # FLEX: one scalar cut per cluster
    if per_cluster is not None:
        cl.setdefault("cut-layers", per_cluster)
        cl.setdefault("num-cluster", len(per_cluster))
        cut = per_cluster[0]
    if top_nc and "num-cluster" not in cl:
        cl["num-cluster"] = int(top_nc)
    cfg.no_cluster_cut_layers = [int(c) for c in cut]
    cfg.num_cluster = int(cl.get("num-cluster", 1))
    if (mc or top_nc or per_cluster is not None) and "cluster-mode" not in manual:
        cfg.cluster_mode = cfg.num_cluster > 1 or per_cluster is not None
    ccl = cl.get("cut-layers") or [cfg.no_cluster_cut_layers] * cfg.num_cluster
    cfg.cluster_cut_layers = [list(map(int, c)) if isinstance(c, (list, tuple)) else [int(c)] for c in ccl]
    if len(cfg.cluster_cut_layers) == 1 and cfg.num_cluster > 1:
        cfg.cluster_cut_layers = cfg.cluster_cut_layers * cfg.num_cluster
    info = cl.get("infor-cluster", cl.get("info-cluster", s.get("info-cluster", s.get("infor-cluster"))))
    cfg.infor_cluster_given = bool(info)
    cfg.infor_cluster = [list(map(int, c)) for c in info] if info else [list(cfg.clients)]
    if not cfg.cluster_mode:
        cfg.num_cluster = 1

    sel = s.get("cluster-selection", {}) or {}
    cfg.sel_num_cluster = int(sel.get("num-cluster", 1))
    cfg.algorithm_cluster = sel.get("algorithm-cluster", "KMeans")
    cfg.selection_mode = bool(sel.get("selection-mode", False))

    lt = s.get("limited-time")
    if isinstance(lt, dict):
        cfg.limited_time = {"enable": bool(lt.get("enable", False)), "epoch": int(lt.get("epoch", 10)),
                            "time": float(lt.get("time", 10))}
    cfg.local_round = int(s.get("local-round", raw.get("learning", {}).get("local-round", 1)))
    cfg.t_g = int(s.get("t-g", 1))
    cfg.t_c = int(s.get("t-c", 1))
    cfg.select_ratio = s.get("select-ratio")
    cfg.lr_decay = s.get("lr-decay")
    cfg.lr_step = s.get("lr-step")

    cfg.log_path = raw.get("log_path", ".")
    cfg.debug_mode = bool(raw.get("debug_mode", True))
    learning = dict(DEFAULT_LEARNING)
    learning.update(raw.get("learning", {}) or {})
    cfg.learning = learning
    b = dict(DEFAULT_B200)
    b.update(raw.get("b200", {}) or {})
    if os.environ.get("SLB200_ALGORITHM"):
        b["algorithm"] = os.environ["SLB200_ALGORITHM"]
    cfg.b200 = b
    _validate(cfg)
    return cfg


def _validate(cfg: Config) -> None:
    if len(cfg.clients) < 1 or any(c < 0 for c in cfg.clients):
        raise ValueError(f"server.clients must be a list of non-negative ints, got {cfg.clients}")
    n_cut = len(cfg.clients) - 1
    cuts = cfg.cluster_cut_layers if cfg.cluster_mode else [cfg.no_cluster_cut_layers]
    if not cfg.auto_mode:
        for c in cuts:
            if len(c) != n_cut and not (len(c) == 1 and c[0] == 0):
                raise ValueError(f"{len(cfg.clients)} layers need {n_cut} cut points, got {c}")
            if any(b <= a for a, b in zip(c, c[1:])):
                raise ValueError(f"cut layers must be increasing: {c}")
    if cfg.cluster_mode:
        if len(cfg.cluster_cut_layers) != cfg.num_cluster:
            raise ValueError("cluster.cut-layers must have num-cluster entries")
    if cfg.cluster_mode and cfg.infor_cluster_given:
        if len(cfg.infor_cluster) != cfg.num_cluster:
            raise ValueError("infor-cluster must have num-cluster entries")
        per_stage = [sum(ic[i] for ic in cfg.infor_cluster) for i in range(len(cfg.clients))]
        if per_stage != list(cfg.clients):
            # the reference ships such a file (other/2LS/config.yaml: clients [9,3] vs 3x[2,1]);
            # tolerate it like the reference does and let registration counts decide.
            cfg.warnings.append(f"infor-cluster sums {per_stage} != clients {cfg.clients}")


def load_config(path: str = "config.yaml") -> Config:
    with open(path, "r") as f:
        return normalize(yaml.safe_load(f))


def dump_config(cfg: Config, path: str) -> None:
    with open(path, "w") as f:
        yaml.safe_dump(cfg.to_dict(), f, sort_keys=False)
