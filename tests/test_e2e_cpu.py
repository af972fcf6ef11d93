"""BASELINE config #1: VGG16/CIFAR10 2-layer split cut=[7], 1 client/layer, CPU world_size=2
— the full REGISTER→START→READY→SYN→NOTIFY→PAUSE→UPDATE→STOP cycle with no GPU."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import yaml

from split_learning_b200.checkpoint import load_checkpoint
from split_learning_b200.config import normalize
from split_learning_b200.models import VGG16_CIFAR10
from split_learning_b200.runner import run_inproc

from oracle_cases import reference_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _raw(tmp, clients=(1, 1), cut=(7,), rounds=1, samples=64, **server):
    raw = yaml.safe_load(open(reference_config()))
    raw["server"].update({"clients": list(clients), "global-round": rounds, "validation": True})
    raw["server"]["manual"]["no-cluster"]["cut-layers"] = list(cut)
    raw["server"]["data-distribution"]["num-sample"] = samples
    raw["server"].update(server)
    raw["log_path"] = str(tmp)
    raw["learning"]["batch-size"] = 8
    raw["b200"] = {"synthetic-data": True, "watchdog-seconds": 60}
    return raw


def test_two_stage_inproc(tmp_path):
    srv = run_inproc(normalize(_raw(tmp_path, rounds=2)), workdir=str(tmp_path), timeout=300)
    assert [h["ok"] for h in srv.history] == [True, True]
    assert srv.topology.cut_layers() == [[7]] and srv.topology.infor_cluster() == [[1, 1]]
    sd = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    m = VGG16_CIFAR10()
    m.load_state_dict(sd)                       # flat full-model layout, 97 entries
    assert len(sd) == 97
    # BN counters advanced: stage 1 recomputes forward (2 per microbatch), stage 2 once
    nb = 6 * 8 // 8 if False else None
    assert sd["layer2.num_batches_tracked"].item() == 2 * sd["layer9.num_batches_tracked"].item() > 0


def test_three_stage_two_first_clients(tmp_path):
    srv = run_inproc(normalize(_raw(tmp_path, clients=(2, 1, 1), cut=(5, 10))), workdir=str(tmp_path), timeout=300)
    assert srv.history[0]["ok"] and srv.topology.infor_cluster() == [[2, 1, 1]]
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97


def test_cluster_mode(tmp_path):
    raw = _raw(tmp_path, clients=(2, 2))
    raw["server"]["manual"] = {"cluster-mode": True, "no-cluster": {"cut-layers": [7]},
                               "cluster": {"num-cluster": 2, "cut-layers": [[7], [14]], "infor-cluster": [[1, 1], [1, 1]]}}
    srv = run_inproc(normalize(raw), workdir=str(tmp_path), timeout=300)
    assert srv.history[0]["ok"] and srv.topology.cut_layers() == [[7], [14]]
    assert len(load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))) == 97


def test_resume_from_checkpoint(tmp_path):
    run_inproc(normalize(_raw(tmp_path)), workdir=str(tmp_path), timeout=300)
    first = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    raw = _raw(tmp_path)
    raw["learning"]["learning-rate"] = 0.0         # resumed weights must come back unchanged
    raw["learning"]["momentum"] = 0.0
    run_inproc(normalize(raw), workdir=str(tmp_path), timeout=300)
    second = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    assert torch.equal(first["layer52.weight"], second["layer52.weight"])
    assert torch.equal(first["layer1.weight"], second["layer1.weight"])


def test_watchdog_instead_of_deadlock(tmp_path):
    """Kill-a-stage fault test: with no last stage the first stage must time out, not hang."""
    from split_learning_b200.client import RpcClient
    from split_learning_b200.server import Server
    from split_learning_b200.transport import InProcBroker
    import threading
    raw = _raw(tmp_path)
    raw["b200"]["watchdog-seconds"] = 1.0
    cfg = normalize(raw)
    broker = InProcBroker()
    srv = Server(cfg, broker, workdir=str(tmp_path))
    threading.Thread(target=lambda: srv.start(idle_timeout=20), daemon=True).start()
    ghost = RpcClient("ghost", 2, broker, b200_opts=cfg.b200)
    ghost.register({"speed": 1})                  # registers, then never serves its queue

    def ghost_ack():                              # acknowledges START so SYN is released, then dies
        m = broker.get_obj("reply_ghost", 20)
        ghost.on_start(m)
    threading.Thread(target=ghost_ack, daemon=True).start()
    c1 = RpcClient("c1", 1, broker, b200_opts=cfg.b200)
    c1.register({"speed": 1})
    with pytest.raises(TimeoutError):
        c1.wait_response(idle_timeout=30)
    srv.done = True


@pytest.mark.slow
def test_world_size_2_processes_tcp(tmp_path):
    """One OS process per role over the loopback TCP broker (server.py / client.py CLIs)."""
    cfg_path = tmp_path / "config.yaml"
    raw = _raw(tmp_path)
    raw["b200"]["port"] = 29911
    yaml.safe_dump(raw, open(cfg_path, "w"))
    env = dict(os.environ, PYTHONPATH=ROOT, SLB200_QUIET="1")
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "server.py"), "--config", str(cfg_path)],
                              cwd=tmp_path, env=env)]
    for layer in (1, 2):
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "client.py"), "--layer_id", str(layer),
                                       "--device", "cpu", "--config", str(cfg_path)], cwd=tmp_path, env=env))
    try:
        for p in procs:
            assert p.wait(timeout=300) == 0
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    assert (tmp_path / "VGG16_CIFAR10.pth").exists()


def test_nan_round_is_counted_but_not_aggregated(tmp_path, monkeypatch):
    """Reference semantics (src/Server.py:162-170,195-196): a round in which a client saw a NaN loss is not aggregated
    or checkpointed, yet it still consumes one of the global rounds."""
    from split_learning_b200.train import executor as E
    calls = {"n": 0}
    real = E.TorchExecutor.nan_detected

    def flaky(self):
        if self.is_last:
            calls["n"] += 1
            if calls["n"] == 1:              # last stage reports a NaN loss in round 1 only
                return True
        return real(self)
    monkeypatch.setattr(E.TorchExecutor, "nan_detected", flaky)
    raw = _raw(tmp_path, rounds=2)
    raw["server"]["validation"] = False
    srv = run_inproc(normalize(raw), workdir=str(tmp_path), timeout=300)
    assert [h["ok"] for h in srv.history] == [False, True]
    assert load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))          # written by the good round


def test_duplicate_register_is_ignored(tmp_path):
    """A client that REGISTERs twice is listed once (src/Server.py:119-120)."""
    import uuid
    from split_learning_b200 import messages as M
    from split_learning_b200.server import Server
    from split_learning_b200.transport import InProcBroker
    cfg = normalize(_raw(tmp_path, clients=(2, 1)))
    srv = Server(cfg, InProcBroker(), workdir=str(tmp_path))
    cid = uuid.uuid4()
    msg = M.register(cid, 1, {"speed": 1.0, "exe_time": [1.0] * 52, "size_data": [1.0] * 52, "network": 1.0}, -1)
    srv.on_request(msg)
    srv.on_request(msg)
    assert len(srv.clients) == 1


def test_dead_client_becomes_an_error_not_a_deadlock(tmp_path, monkeypatch):
    """Failure detection: the reference dead-locks when a client dies mid-round (no heartbeat / timeouts, SURVEY §5).
    Here the peers' watchdogs turn the silence into a TimeoutError within ``watchdog-seconds``."""
    import time
    from split_learning_b200 import client as C
    real = C.RpcClient.run_stage

    def dying(self):
        if self.layer_id == 2:
            raise RuntimeError("simulated crash of the last-stage client")
        return real(self)
    monkeypatch.setattr(C.RpcClient, "run_stage", dying)
    raw = _raw(tmp_path)
    raw["server"]["validation"] = False
    raw["b200"]["watchdog-seconds"] = 3
    t0 = time.monotonic()
    with pytest.raises((RuntimeError, TimeoutError)):
        run_inproc(normalize(raw), workdir=str(tmp_path), timeout=60)
    assert time.monotonic() - t0 < 60


def test_async_checkpoint_protocol_resident_rounds(tmp_path):
    """The device plane's round end, replayed with scripted clients on the CPU: UPDATEs without parameters (``resident``,
    ``checkpoint_follows``), the stage state-dicts arriving later as CHECKPOINT messages on their own queue (out of order,
    the older round last) — the server must not wait for them inside the round, must write exactly the newest round, and
    must not send parameters in the next START."""
    import threading
    import time
    from split_learning_b200 import messages as M
    from split_learning_b200.checkpoint import load_meta
    from split_learning_b200.server import Server
    from split_learning_b200.transport import InProcBroker
    raw = _raw(tmp_path, rounds=2)
    raw["server"]["validation"] = False
    cfg = normalize(raw)
    br = InProcBroker()
    srv = Server(cfg, br, workdir=str(tmp_path))
    th = threading.Thread(target=lambda: srv.start(idle_timeout=60), daemon=True)
    th.start()
    full = VGG16_CIFAR10().state_dict()
    parts = {1: {k: v for k, v in full.items() if int(k.split(".")[0][5:]) <= 7},
             2: {k: v for k, v in full.items() if int(k.split(".")[0][5:]) > 7}}
    ids = {1: "c-one", 2: "c-two"}
    for lid, cid in ids.items():
        br.publish_obj(M.RPC_QUEUE, M.register(cid, lid, {"speed": 1.0}, -1, rank=lid - 1))

    def expect(cid, action, timeout=30):
        t0 = time.monotonic()
        while time.monotonic() - t0 < timeout:
            m = br.get_obj(M.reply_queue(cid), 0.5)
            if m is not None and m.get("action") != M.HEARTBEAT:
                assert m["action"] == action, (m["action"], action)
                return m
        raise AssertionError(f"{cid}: no {action}")
    starts = []
    for rnd in (1, 2):
        for lid, cid in ids.items():
            starts.append(expect(cid, M.START))
            br.publish_obj(M.RPC_QUEUE, M.ready(cid, lid))
        for cid in ids.values():
            expect(cid, M.SYN)
        br.publish_obj(M.RPC_QUEUE, M.notify(ids[1], 1, 0))
        for cid in ids.values():
            expect(cid, M.PAUSE)
        for lid, cid in ids.items():
            br.publish_obj(M.RPC_QUEUE, M.update(cid, lid, True, 4, 0, None, resident=True, checkpoint_follows=rnd,
                                                 device_ms=12.5, loss=2.0, timing={"fedavg": 0.4, "at_update": time.monotonic()}))
    for cid in ids.values():
        expect(cid, M.STOP)
    assert starts[0]["parameters"] is None and all(s["parameters"] is None and s["resident"] for s in starts[2:])
    # round 2's parts arrive first, round 1's afterwards: the stale round must not overwrite the newer checkpoint
    tag = lambda sd, v: {k: (t.clone().float().fill_(v) if t.is_floating_point() else t.clone()) for k, t in sd.items()}
    for rnd in (2, 1):
        for lid, cid in ids.items():
            br.publish_obj(M.CKPT_QUEUE, M.checkpoint(cid, lid, 0, rnd, tag(parts[lid], float(rnd))))
        time.sleep(0.3)
    th.join(30)
    assert not th.is_alive(), "server must finish once every announced checkpoint part has arrived"
    sd = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))
    assert len(sd) == 97 and float(sd["layer1.weight"].flatten()[0]) == 2.0 and float(sd["layer50.weight"].flatten()[0]) == 2.0
    assert load_meta(str(tmp_path / "VGG16_CIFAR10.pth")).get("round") == 2
    assert [h["ok"] for h in srv.history] == [True, True]
    assert srv.history[0]["device_ms"] == 12.5 and "updates_in" in srv.history[0]["phases_ms"]
    assert srv.history[1]["first_stage_microbatches"] == 4
