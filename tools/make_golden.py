"""Regenerate the stored oracle data under ``tests/golden/`` from the original (reference) project.

The tests compare this engine with the reference implementation it reproduces; they read these files instead of the
reference tree, so the suite runs from a plain checkout.

    python tools/make_golden.py cpu REFERENCE_DIR        # configs, planning / FedAvg oracles, model layouts and outputs
    SLB200_REFERENCE_DIR=REFERENCE_DIR python baseline/install_reference.py   # reference trainers -> baseline/_ref
    python tools/make_golden.py parity [OUT_DIR]         # reference trainers on a GPU: TF32 run + fp32 oracle (CUDA)
"""
import contextlib
import io
import json
import os
import pickle
import sys
import threading
import time
import uuid

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _import_from(root, module):
    import importlib
    for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
        del sys.modules[k]
    sys.path.insert(0, root)
    try:
        return importlib.import_module(module)
    finally:
        sys.path.remove(root)


def _tensor_json(t):
    return {"dtype": str(t.dtype).replace("torch.", ""), "shape": list(t.shape), "values": t.flatten().tolist()}


def cpu(ref):
    import types
    import yaml
    from oracle_cases import PARTITION_CASES, CLUSTER_SEED, SELECTION_SEED, fedavg_inputs, layout_digest, model_cases
    os.makedirs(os.path.join(GOLDEN, "reference_configs"), exist_ok=True)
    configs = {"main": os.path.join(ref, "config.yaml")}
    for d in sorted(os.listdir(os.path.join(ref, "other"))):
        p = os.path.join(ref, "other", d, "config.yaml")
        if os.path.exists(p):
            configs[d] = p
    for name, p in configs.items():
        with open(os.path.join(GOLDEN, "reference_configs", name + ".json"), "w") as f:
            json.dump(yaml.safe_load(open(p)), f, indent=1)

    out = {}
    sys.modules.setdefault("pika", types.ModuleType("pika"))
    fedavg = _import_from(ref, "src.Utils").fedavg_state_dicts
    out["fedavg"] = {str(w): {k: _tensor_json(v) for k, v in fedavg(fedavg_inputs(), w).items()} for w in (None, [3, 1, 7])}
    partition = _import_from(ref, "src.Partition").partition
    out["partition"] = [partition(*case) for case in PARTITION_CASES()]
    rng = np.random.RandomState(CLUSTER_SEED)
    a = np.concatenate([rng.dirichlet([10, 1, 1, 1], 6), rng.dirichlet([1, 1, 10, 10], 5)]) * 500
    labels, infos = _import_from(ref, "src.Cluster").clustering_algorithm(a, 2)
    out["clustering"] = {"labels": np.asarray(labels).tolist(), "infos": [[int(x[0])] for x in infos]}
    rng = np.random.RandomState(SELECTION_SEED)
    perf = np.concatenate([rng.normal(100, 5, 12), rng.normal(1000, 40, 10)]).clip(1)
    out["selection_threshold"] = float(_import_from(ref, "src.Selection").auto_threshold(perf))
    with open(os.path.join(GOLDEN, "algorithms.json"), "w") as f:
        json.dump(out, f)

    layouts, forwards = {}, {}
    for mine, mod, cls, sub, forward in model_cases():
        theirs = getattr(_import_from(os.path.join(ref, sub), mod), cls)
        n = mine.num_layers()
        layouts[cls] = {f"{a},{b}": layout_digest(theirs(start_layer=a, end_layer=b).state_dict()) for a, b in [(0, n), (0, 3), (3, n), (2, 5)]}
        if forward:
            torch.manual_seed(0)
            m, t = mine().eval(), theirs().eval()
            t.load_state_dict(m.state_dict())
            torch.manual_seed(1)
            x = mine.example_input(2)
            with torch.no_grad():
                forwards[cls] = t(x).tolist()
    with open(os.path.join(GOLDEN, "models.json"), "w") as f:
        json.dump({"layouts": layouts, "forward": forwards}, f, indent=0)
    print("wrote", GOLDEN)


def _reference_run(batches, device, cut, learning, tf32):
    """Losses, cut activations, cut gradients and the initial / final state dicts of the unmodified reference trainers
    (first-layer and last-layer loops over the in-process pika shim), dropout off."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = bool(tf32)
    try:
        sys.path.insert(0, os.path.join(ROOT, "baseline"))
        from run_reference import _prepare_imports
        _prepare_imports()
        import pika
        from src.model.VGG16_CIFAR10 import VGG16_CIFAR10 as RefVGG
        from src.train.VGG16 import Train_VGG16
        pika._REMOTE = None
        torch.manual_seed(11)
        m1, m2 = RefVGG(start_layer=0, end_layer=cut), RefVGG(start_layer=cut)
        for m in m2.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        init = ({k: v.clone() for k, v in m1.state_dict().items()}, {k: v.clone() for k, v in m2.state_dict().items()})
        acts, grads = [], []

        def hook(queue, body):
            if queue.startswith("intermediate_queue_"):
                acts.append(torch.from_numpy(pickle.loads(body)["data"]).clone())
            elif queue.startswith("gradient_queue_"):
                grads.append(torch.from_numpy(pickle.loads(body)["data"]).clone())
        pika.on_get.append(hook)
        ids = (uuid.uuid4(), uuid.uuid4())
        ch = lambda: pika.BlockingConnection(pika.ConnectionParameters("127.0.0.1")).channel()
        t1, t2 = Train_VGG16(ids[0], 1, ch(), device), Train_VGG16(ids[1], 2, ch(), device)
        errs = []

        def guard(fn):
            def run():
                try:
                    fn()
                except Exception as e:            # noqa
                    errs.append(e)
            return run
        th = [threading.Thread(target=guard(lambda: t1.train_on_first_layer(m1, learning, batches, 0)), daemon=True),
              threading.Thread(target=guard(lambda: t2.train_on_last_layer(m2, learning, 0)), daemon=True)]
        server, out = ch(), io.StringIO()
        with contextlib.redirect_stdout(out):
            for t in th:
                t.start()
            deadline = time.time() + 300
            while time.time() < deadline and not errs:           # the "server": NOTIFY -> PAUSE to both clients
                _, _, body = server.basic_get(queue="rpc_queue")
                if body and pickle.loads(body).get("action") == "NOTIFY":
                    for cid in ids:
                        server.basic_publish(routing_key=f"reply_{cid}", body=pickle.dumps({"action": "PAUSE", "message": "", "parameters": None}))
                    break
            for t in th:
                t.join(60)
        pika.on_get.remove(hook)
        assert not errs and not any(t.is_alive() for t in th), errs
        losses = [float(l.split("Loss:")[1]) for l in out.getvalue().splitlines() if l.startswith("Loss:")]
        final = ({k: v.detach().cpu().clone() for k, v in m1.state_dict().items()}, {k: v.detach().cpu().clone() for k, v in m2.state_dict().items()})
        return losses, acts, grads, init, final
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def parity(out_dir):
    import oracle_cases as G
    from split_learning_b200.models import VGG16_CIFAR10
    batches = G.parity_batches()
    tf = _reference_run(batches, "cuda:0", G.CUT, G.PARITY_LEARNING, tf32=True)
    fp = _reference_run(batches, "cuda:0", G.CUT, G.PARITY_LEARNING, tf32=False)
    # the engine starts from the same weights by building its own stages under the same seed
    m1, m2 = G.parity_initial_stages(VGG16_CIFAR10)
    for mine, theirs in ((m1.state_dict(), tf[3][0]), (m2.state_dict(), tf[3][1])):
        assert list(mine) == list(theirs) and all(torch.equal(mine[k], theirs[k]) for k in mine)
    rng = np.random.default_rng(0)
    # the first PARITY_SAMPLES of 4096 draws (the stored file was cut down to stay under 1 MB)
    act_idx = rng.choice(tf[1][0].numel(), 4096, replace=False)[:G.PARITY_SAMPLES]
    grad_idx = rng.choice(tf[2][0].numel(), 4096, replace=False)[:G.PARITY_SAMPLES]
    pick = lambda ts, idx: np.stack([t.flatten().float().numpy()[idx] for t in ts])
    data = {"loss_tf32": np.array(tf[0]), "loss_fp32": np.array(fp[0]), "act_idx": act_idx, "grad_idx": grad_idx,
            "act_tf32": pick(tf[1], act_idx), "act_fp32": pick(fp[1], act_idx),
            "grad_tf32": pick(tf[2], grad_idx), "grad_fp32": pick(fp[2], grad_idx),
            "nbt": np.array(int(tf[4][0]["layer2.num_batches_tracked"]))}
    for k in G.PARITY_KEYS:
        which = 0 if k in tf[3][0] else 1
        n = tf[3][which][k].numel()
        idx = rng.choice(n, min(n, 2048), replace=False)
        data[f"{k}:idx"] = idx
        data[f"{k}:tf32"] = tf[4][which][k].flatten().float().numpy()[idx]
        data[f"{k}:fp32"] = fp[4][which][k].flatten().float().numpy()[idx]
    os.makedirs(out_dir, exist_ok=True)
    np.savez(os.path.join(out_dir, "parity_vgg16_cut7.npz"), **data)
    print("wrote", out_dir, {k: v.shape for k, v in data.items()})


if __name__ == "__main__":
    if sys.argv[1] == "cpu":
        cpu(sys.argv[2])
    else:
        parity(sys.argv[2] if len(sys.argv) > 2 else GOLDEN)
