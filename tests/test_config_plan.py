import pytest
import yaml

from split_learning_b200.config import load_config, normalize
from split_learning_b200.plan import rank_assignment, resolve_range, stage_layers

from oracle_cases import reference_config

# the reference's config.yaml and other/<variant>/config.yaml, stored under tests/golden/reference_configs


@pytest.mark.parametrize("name", ["main", "2LS", "Cluster_FSL", "DCSL", "FLEX", "Vanilla_SL"])
def test_reference_configs_load_and_roundtrip(name):
    cfg = load_config(reference_config(name))
    again = normalize(cfg.to_dict())
    assert again.to_dict() == cfg.to_dict()
    assert cfg.learning["batch-size"] > 0 and "control-count" in cfg.learning


def test_variant_keys():
    flex = load_config(reference_config("FLEX"))
    assert flex.cluster_mode and flex.num_cluster == 3 and flex.cluster_cut_layers == [[7], [7], [4]]
    assert (flex.t_g, flex.t_c, flex.select_ratio) == (4, 2, 0.5)
    two = load_config(reference_config("2LS"))
    assert two.cluster_cut_layers == [[2]] * 3 and two.infor_cluster == [[2, 1]] * 3 and two.warnings
    dcsl = load_config(reference_config("DCSL"))
    assert dcsl.local_round == 1 and dcsl.no_cluster_cut_layers == [7]
    van = load_config(reference_config("Vanilla_SL"))
    assert van.limited_time == {"enable": False, "epoch": 10, "time": 10.0}
    assert van.learning["clip-grad-norm"] == 0.0


def test_readme_era_schema():
    raw = {"server": {"clients": [2, 2], "no-cluster": {"cut-layers": [14]}, "model": "VGG16",
                      "data-distribution": {"non-iid": True, "non-iid-rate": 0.5, "num-sample": 100, "num-label": 10}},
           "learning": {"batch-size": 8}}
    cfg = normalize(raw)
    assert cfg.no_cluster_cut_layers == [14] and cfg.non_iid_rate == 0.5
    assert cfg.learning["control-count"] == 3          # defaults filled in


def test_validation_errors():
    with pytest.raises(ValueError):
        normalize({"server": {"clients": [1, 1, 1], "manual": {"cluster-mode": False, "no-cluster": {"cut-layers": [7]}}}})
    with pytest.raises(ValueError):
        normalize({"server": {"clients": [1, 1, 1], "manual": {"cluster-mode": False, "no-cluster": {"cut-layers": [10, 5]}}}})


def test_stage_layers_matches_reference_arithmetic():
    # src/Server.py:222-228
    assert stage_layers(1, 2, [7]) == [0, 7]
    assert stage_layers(2, 2, [7]) == [7, -1]
    assert [stage_layers(i, 3, [5, 10]) for i in (1, 2, 3)] == [[0, 5], [5, 10], [10, -1]]
    assert resolve_range([0, 0], 52) == (0, 52)
    assert resolve_range([7, -1], 52) == (7, 52)


def test_rank_assignment():
    assert rank_assignment([1, 1]) == [(1, 0, 0), (2, 0, 0)]
    r = rank_assignment([4, 4], [[2, 2], [2, 2]])
    assert len(r) == 8 and r[0] == (1, 0, 0) and r[2] == (2, 0, 0) and r[4] == (1, 1, 0)


def test_shipped_example_configs_normalise():
    """configs/*.yaml: one example per algorithm variant / model family / topology."""
    import glob
    import os
    import yaml
    from split_learning_b200.config import normalize
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    files = sorted(glob.glob(os.path.join(root, "configs", "*.yaml")))
    assert len(files) >= 12
    algos = set()
    for f in files:
        cfg = normalize(yaml.safe_load(open(f)))
        algos.add(cfg.b200.get("algorithm", "main"))
        assert sum(cfg.clients) >= 2
    assert algos == {"main", "vanilla_sl", "cluster_fsl", "dcsl", "flex", "2ls"}


def test_fedavg_allreduce_segments_two_clusters_cut_7_and_14():
    """The device FedAvg all-reduce (``parallel/allreduce.py``) cuts the model into segments = maximal key ranges held by the
    same set of replicas.  BASELINE config #4 (cluster 0 cut at 7, cluster 1 cut at 14): layers 1-7 live in both first
    stages, 8-14 in stage 2 of cluster 0 and stage 1 of cluster 1, 15-52 in both last stages — for parameters, BN running
    statistics and the integer counters alike — and every replica derives the same list from (model, layers) alone."""
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.parallel.allreduce import KINDS, Member, build_segments, model_key_order
    from split_learning_b200.train.b200_executor import flat_layouts
    spans = [(0, 7, 0), (7, 52, 0), (0, 14, 1), (14, 52, 1)]                 # (start, end, cluster)
    members = sorted((Member(f"m{i}", cl, a, b, {}, {}) for i, (a, b, cl) in enumerate(spans)), key=lambda m: m.uid)
    layouts = [flat_layouts(VGG16_CIFAR10, m.start_layer, m.end_layer) for m in members]
    order = model_key_order(VGG16_CIFAR10)
    segs = build_segments(members, layouts, order)
    assert [s.index for s in segs] == list(range(len(segs)))
    by_kind = {k: [s for s in segs if s.kind == k] for k in KINDS}
    for kind in KINDS:
        assert [s.holders for s in by_kind[kind]] == [[0, 2], [1, 2], [1, 3]], kind
    p = by_kind["P"]
    assert p[0].first_key == "layer1.weight" and p[1].first_key == "layer8.weight" and p[2].first_key == "layer15.weight"
    # a segment starts where the holder's own flat layout puts its first key, and the three segments tile every stage buffer
    for s in segs:
        for q, off in zip(s.holders, s.offs):
            assert off == layouts[q][s.kind][s.first_key][0]
    for q in range(4):
        for kind in KINDS:
            mine = sorted((s.offs[s.holders.index(q)], s.n) for s in by_kind[kind] if q in s.holders)
            total = sum(n for _, n in layouts[q][kind].values())
            assert mine[0][0] == 0 and all(a + n == b for (a, n), (b, _) in zip(mine, mine[1:])) and sum(n for _, n in mine) == total
    # every parameter of the model is covered exactly once per kind
    covered = sum(s.n for s in p if 0 in s.holders) + sum(s.n for s in p if 1 in s.holders)
    full = flat_layouts(VGG16_CIFAR10, 0, VGG16_CIFAR10.num_layers())
    assert covered == sum(n for _, n in full["P"].values())
    # one cluster, one replica per stage: a single segment per kind and holder — the degenerate case the main tests use
    solo = build_segments(members[:2], layouts[:2], order)
    assert [(s.kind, s.holders) for s in solo] == [(k, [q]) for k in KINDS for q in (0, 1)]
