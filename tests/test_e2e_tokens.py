"""Token-model families (and MobileNetv1) through the full control plane (REGISTER .. STOP): KWT / ViT with AdamW, BERT with LoRA
wrapping + merge before upload (reference src/RpcClient.py:61-66,99-103,121-122).  CPU: torch executor; GPU: the
native sm_90a blocks (``train/token_native.py``) — same config, same checkpoint layout."""
import os

import pytest
import torch
import yaml

from split_learning_b200.checkpoint import load_checkpoint
from split_learning_b200.config import normalize
from split_learning_b200.runner import run_inproc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [("KWT", "SPEECHCOMMANDS", 8, 10, 4, 152), ("ViT", "CIFAR10", 6, 10, 4, 80), ("BERT", "AGNEWS", 6, 4, 2, 201),
         ("MobileNetv1", "CIFAR10", 15, 10, 4, 191)]


def _raw(tmp, model, data, cut, labels, bs, **b200):
    raw = yaml.safe_load(open(os.path.join(ROOT, "config.yaml")))
    raw["server"].update({"clients": [1, 1], "global-round": 1, "validation": True, "model": model, "data-name": data})
    raw["server"]["manual"]["no-cluster"]["cut-layers"] = [cut]
    raw["server"]["data-distribution"].update({"num-sample": 2 * bs * labels, "num-label": labels})
    raw["log_path"] = str(tmp)
    raw["learning"]["batch-size"] = bs
    raw["b200"] = {"synthetic-data": True, "watchdog-seconds": 120, **b200}
    return raw


@pytest.mark.parametrize("model,data,cut,labels,bs,n_keys", CASES, ids=[c[0] for c in CASES])
def test_token_family_round_cpu(tmp_path, model, data, cut, labels, bs, n_keys):
    srv = run_inproc(normalize(_raw(tmp_path, model, data, cut, labels, bs)), workdir=str(tmp_path), timeout=600)
    assert srv.history and srv.history[0]["ok"] and srv.history[0]["val_total"] > 0
    sd = load_checkpoint(str(tmp_path / f"{model}_{data}.pth"))
    assert len(sd) == n_keys and all("lora" not in k for k in sd)
    assert all(torch.isfinite(v.float()).all() for v in sd.values())


@pytest.mark.gpu
@pytest.mark.parametrize("model,data,cut,labels,bs,n_keys", CASES, ids=[c[0] for c in CASES])
def test_token_family_round_native_gpu(tmp_path, model, data, cut, labels, bs, n_keys, monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.ops import native as N
    from split_learning_b200.train import executor as E
    made = []
    real = E.TorchExecutor.__init__

    def spy(self, *a, **k):
        real(self, *a, **k)
        made.append(self.native)
    monkeypatch.setattr(E.TorchExecutor, "__init__", spy)
    before = N.LAUNCHES
    srv = run_inproc(normalize(_raw(tmp_path, model, data, cut, labels, 32 if model == "MobileNetv1" else 8)),
                     devices=["cuda:0"], workdir=str(tmp_path), timeout=600)
    assert srv.history and srv.history[0]["ok"]
    assert made and all(made), made                      # every stage ran the native blocks
    assert N.LAUNCHES - before > 100
    sd = load_checkpoint(str(tmp_path / f"{model}_{data}.pth"))
    assert len(sd) == n_keys and all(torch.isfinite(v.float()).all() for v in sd.values())


@pytest.mark.gpu
def test_cuda_wire_in_process(tmp_path):
    """``b200.wire: cuda``: cut activations / gradients of the host data plane never leave the GPU (thread hand-off)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.train.dataplane import _LOCAL, HostDataPlane
    before = dict(HostDataPlane.sent)
    srv = run_inproc(normalize(_raw(tmp_path, "KWT", "SPEECHCOMMANDS", 8, 10, 8, wire="cuda")), devices=["cuda:0"],
                     workdir=str(tmp_path), timeout=600)
    assert srv.history and srv.history[0]["ok"]
    assert HostDataPlane.sent["cuda_local"] - before["cuda_local"] >= 2 * 20 and HostDataPlane.sent["host"] == before["host"]
    assert not _LOCAL                                                  # every handed-over tensor was consumed


@pytest.mark.gpu
def test_cuda_wire_across_processes(tmp_path):
    """Same through ``launch.py`` (one OS process per client): CUDA-IPC handles in the broker messages."""
    import subprocess
    import sys
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    raw = _raw(tmp_path, "KWT", "SPEECHCOMMANDS", 8, 10, 8, wire="cuda", port=29941)
    raw["server"]["validation"] = False
    cfg = tmp_path / "config.yaml"
    yaml.safe_dump(raw, open(cfg, "w"))
    env = dict(os.environ, SLB200_QUIET="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "launch.py"), "--config", str(cfg), "--timeout", "280"],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    assert "payloads stay on the GPU" in r.stdout + r.stderr
    sd = load_checkpoint(str(tmp_path / "KWT_SPEECHCOMMANDS.pth"))
    assert len(sd) == 152 and all(torch.isfinite(v.float()).all() for v in sd.values())
