"""Inputs shared by the tests that compare with the reference implementation and by ``tools/make_golden.py``, which ran
the reference on exactly these inputs and stored its answers under ``tests/golden/``."""
import hashlib
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_path(*parts):
    return os.path.join(GOLDEN, *parts)


def load_json(name):
    with open(golden_path(name)) as f:
        return json.load(f)


def reference_config(name="main"):
    """A reference config file (``config.yaml`` or ``other/<name>/config.yaml``), stored as JSON (valid YAML)."""
    return golden_path("reference_configs", name + ".json")


def layout_digest(state_dict):
    """Entry count and sha256 of a state dict's (key, shape, dtype) list: what ``load_state_dict`` checks."""
    layout = [[k, list(v.shape), str(v.dtype)] for k, v in state_dict.items()]
    return {"entries": len(layout), "sha256": hashlib.sha256(json.dumps(layout).encode()).hexdigest()}


def as_tensor(d):
    return torch.tensor(d["values"], dtype=getattr(torch, d["dtype"])).reshape(d["shape"])


# ---- FedAvg / planning oracles
def rand_sd(seed, keys=("a", "b", "n"), nan=False):
    g = torch.Generator().manual_seed(seed)
    sd = {"a": torch.randn(4, 3, generator=g), "b": torch.randn(5, generator=g),
          "n": torch.tensor(seed * 3 + 1, dtype=torch.int64)}
    if nan:
        sd["a"][0, 0] = float("nan")
    return {k: sd[k] for k in keys}


def fedavg_inputs():
    return [rand_sd(1), rand_sd(2, nan=True), rand_sd(3, keys=("a", "n"))]


def PARTITION_CASES():
    rng = np.random.RandomState(0)
    cases = []
    for _ in range(20):
        L = rng.randint(3, 30)
        e1 = [list(rng.rand(L) + 0.01) for _ in range(rng.randint(1, 4))]
        e2 = [list(rng.rand(L) * 0.3 + 0.01) for _ in range(rng.randint(1, 4))]
        n1, n2 = list(rng.rand(len(e1)) + 0.1), list(rng.rand(len(e2)) + 0.1)
        size = list(rng.rand(L) * 5)
        cases.append((e1, n1, e2, n2, size))
    return cases


CLUSTER_SEED, SELECTION_SEED = 1, 2


def model_cases():
    """(our class, reference module, reference class, reference sub-directory, forward outputs stored)"""
    from split_learning_b200.models import (BERT_AGNEWS, BERT_EMOTION, KWT_SPEECHCOMMANDS, MobileNetv1_CIFAR10,
                                            VGG16_CIFAR10, VGG16_MNIST, ViT_CIFAR10, ViT_MNIST)
    van = os.path.join("other", "Vanilla_SL")
    return [(VGG16_CIFAR10, "src.model.VGG16_CIFAR10", "VGG16_CIFAR10", "", True),
            (KWT_SPEECHCOMMANDS, "src.model.KWT_SPEECHCOMMANDS", "KWT_SPEECHCOMMANDS", "", True),
            (BERT_AGNEWS, "src.model.BERT_AGNEWS", "BERT_AGNEWS", "", False),
            (VGG16_MNIST, "src.model.VGG16_MNIST", "VGG16_MNIST", van, False),
            (MobileNetv1_CIFAR10, "src.model.MobileNetv1_CIFAR10", "MobileNetv1_CIFAR10", van, False),
            (ViT_CIFAR10, "src.model.ViT_CIFAR10", "ViT_CIFAR10", van, True),
            (ViT_MNIST, "src.model.ViT_MNIST", "ViT_MNIST", van, False),
            (BERT_EMOTION, "src.model.BERT_EMOTION", "BERT_EMOTION", van, False)]


# ---- golden parity of the VGG16 / CIFAR10 training loop (cut after layer 7)
STEPS, B, CUT = 20, 32, 7
PARITY_LEARNING = {"learning-rate": 0.0005, "momentum": 0.5, "batch-size": B, "control-count": 1, "weight-decay": 0.01}
PARITY_SAMPLES = 2048            # fixed random elements of each cut activation / gradient that are stored
PARITY_KEYS = ("layer1.weight", "layer4.weight", "layer5.running_mean", "layer8.weight", "layer41.weight", "layer50.weight",
               "layer52.bias")


def parity_batches():
    g = torch.Generator().manual_seed(5)
    return [(torch.randn(B, 3, 32, 32, generator=g), torch.randint(0, 10, (B,), generator=g)) for _ in range(STEPS)]


def parity_initial_stages(cls):
    """Both stages built under the seed the reference run used (same construction order -> same initial weights)."""
    torch.manual_seed(11)
    return cls(0, CUT), cls(CUT, 52)
