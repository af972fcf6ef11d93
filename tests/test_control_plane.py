"""Transport, messages, auto-mode planning and mailbox geometry (CPU)."""
import threading
import time

import numpy as np
import pytest
import yaml

from split_learning_b200 import messages as M
from split_learning_b200.config import normalize
from split_learning_b200.runner import DEFAULT_PROFILE, run_inproc
from split_learning_b200.transport import InProcBroker, TcpBroker, TcpChannel
from split_learning_b200.transport.broker import delete_old_queues

from oracle_cases import reference_config


def test_inproc_broker_fifo_and_blocking_get():
    b = InProcBroker()
    assert b.basic_get("q") is None
    threading.Timer(0.05, lambda: b.publish_obj("q", {"k": 1})).start()
    t0 = time.monotonic()
    assert b.get_obj("q", 2.0) == {"k": 1} and time.monotonic() - t0 < 1.0
    for i in range(5):
        b.publish_obj("q", i)
    assert [b.get_obj("q") for _ in range(5)] == list(range(5))


@pytest.mark.parametrize("kind", ["native", "python"])
def test_tcp_broker_roundtrip_and_hygiene(kind):
    """Both brokers — the C++ daemon (transport/csrc/slb_broker.cpp) and the Python fallback — behind one protocol."""
    from split_learning_b200.transport import NativeBroker
    srv = NativeBroker(port=0) if kind == "native" else TcpBroker(port=0)
    try:
        c1, c2 = TcpChannel(port=srv.port), TcpChannel(port=srv.port)
        payload = b"x" * (3 << 20)                         # multi-MB frames (a state-dict sized message)
        c1.basic_publish("rpc_queue", payload)
        c1.publish_obj("reply_abc", {"action": "START"})
        c1.publish_obj("keepme", 1)
        assert c2.basic_get("rpc_queue", 2.0) == payload
        assert c2.get_obj("reply_abc", 2.0)["action"] == "START"
        assert c2.queue_depth("keepme") == 1
        delete_old_queues(c2)                              # reply*/rpc_queue* deleted, everything else purged
        assert c2.queue_depth("keepme") == 0 and "reply_abc" not in c2.list_queues()
        # blocking get: times out empty-handed, wakes up as soon as another connection publishes
        t0 = time.monotonic()
        assert c2.basic_get("later", 0.2) is None and 0.15 < time.monotonic() - t0 < 2.0
        threading.Timer(0.1, lambda: c1.publish_obj("later", "hello")).start()
        t0 = time.monotonic()
        assert c2.get_obj("later", 5.0) == "hello" and time.monotonic() - t0 < 2.0
        assert c1.ping()
        own = srv.channel()                                # the server's own channel
        own.publish_obj("fifo", 1), own.publish_obj("fifo", 2)
        assert [c2.get_obj("fifo", 1.0), c2.get_obj("fifo", 1.0)] == [1, 2]
        c1.close(), c2.close()
    finally:
        srv.close()


def test_message_schemas_match_reference_fields():
    # SURVEY Appendix A
    assert set(M.register("id", 1, {"speed": 1}, -1)) >= {"action", "client_id", "layer_id", "profile", "cluster", "message"}
    s = M.start(None, [0, 7], "VGG16", "CIFAR10", {"batch-size": 32}, [500] * 10, True, 0)
    assert set(s) >= {"action", "message", "parameters", "layers", "model_name", "data_name", "learning", "label_count",
                      "refresh", "cluster"}
    assert M.pause()["parameters"] is None and M.stop()["action"] == "STOP"
    u = M.update("id", 2, True, 17, 0, {})
    assert set(u) >= {"action", "client_id", "layer_id", "result", "size", "cluster", "message", "parameters"}
    assert M.notify("id", 1, 0)["action"] == "NOTIFY" and M.reply_queue("x") == "reply_x"


def _auto_cfg(tmp_path, selection):
    raw = yaml.safe_load(open(reference_config()))
    raw["server"].update({"clients": [4, 2], "auto-mode": True, "validation": False, "global-round": 1})
    raw["server"]["data-distribution"].update({"non-iid": True, "num-sample": 64})
    raw["server"]["cluster-selection"] = {"num-cluster": 2, "algorithm-cluster": "KMeans", "selection-mode": selection}
    raw["log_path"] = str(tmp_path)
    raw["learning"]["batch-size"] = 8
    raw["b200"] = {"synthetic-data": True, "watchdog-seconds": 60}
    return normalize(raw)


def test_auto_mode_partition_and_clusters(tmp_path):
    """auto-mode: KMeans over label histograms -> per-cluster cut search from the clients' profiles
    (reference src/Server.py:300-362).  Profiles make layer 7 the balanced cut."""
    exe = [1.0] * 52
    size = [8e6] * 52
    size[6] = 1e3                                           # tiny activation after layer 7 -> best cut = 7
    prof = dict(DEFAULT_PROFILE, exe_time=exe, size_data=size, network=1.0, speed=10.0)
    profiles = [dict(prof) for _ in range(6)]
    cfg = _auto_cfg(tmp_path, selection=False)
    srv = run_inproc(cfg, profiles=profiles, workdir=str(tmp_path), timeout=600)
    assert srv.history[0]["ok"]
    assert len(srv.topology.clusters) == 2
    for cl in srv.topology.clusters:
        if cl.members[0] and cl.members[1]:
            assert cl.cut_layers == [7]
    assert sum(len(c.members[0]) for c in srv.topology.clusters) == 4


def test_broker_comm_allgather_and_barrier():
    """FedAvg group primitives over the control-plane broker (used when clients have no torch.distributed)."""
    from split_learning_b200.parallel.fedavg import BrokerComm
    b = InProcBroker()
    members = ["c", "a", "b"]
    out = {}

    def run(me):
        comm = BrokerComm(b, "g", members, me, timeout=10)
        r1 = comm.all_gather_object({"me": me})
        comm.barrier()
        r2 = comm.all_gather_object(me.upper())
        out[me] = (r1, r2, comm.me)
    ts = [threading.Thread(target=run, args=(m,)) for m in members]
    [t.start() for t in ts]
    [t.join(20) for t in ts]
    assert set(out) == set(members)
    for me, (r1, r2, idx) in out.items():
        assert [d["me"] for d in r1] == ["a", "b", "c"] and r2 == ["A", "B", "C"] and sorted(members)[idx] == me


def test_device_plane_lane_mapping():
    """Lane i (first-stage client i) is served at stage s by member i % n_s.  ``dynamic-consumers`` turns the last edge into a
    ticket ring: every last-stage replica may serve every lane, producers have no fixed partner — also for a last stage that
    does not divide its predecessor.  Without the flag non-dividing stages are refused (-> host data plane)."""
    import pytest
    from split_learning_b200.parallel.device_client import DeviceRpcClient

    def lanes(counts, layer, member, **opts):
        members = {s + 1: [(f"c{s + 1}_{j}", 0) for j in range(n)] for s, n in enumerate(counts)}
        c = DeviceRpcClient.__new__(DeviceRpcClient)
        c.client_id, c.layer_id, c.num_layers, c.opts = f"c{layer}_{member}", layer, len(counts), opts
        return c._lanes({"peers": {"members": members}})

    assert lanes([4, 2, 1], 1, 3) == [(3, None, "c2_1")]
    assert lanes([4, 2, 1], 2, 1) == [(1, "c1_1", "c3_0"), (3, "c1_3", "c3_0")]
    assert [l for l, _, _ in lanes([4, 2, 1], 3, 0)] == [0, 1, 2, 3]
    assert lanes([4, 2, 1], 3, 0)[2] == (2, "c2_0", None)
    assert lanes([2, 2], 2, 1) == [(1, "c1_1", None)]
    # competing consumers (opt-in): [3, 2] cannot be cut into static lanes -> both last-stage replicas serve all three lanes
    dyn = {"dynamic-consumers": True}
    assert lanes([3, 2], 1, 2, **dyn) == [(2, None, None)]
    assert lanes([3, 2], 2, 1, **dyn) == [(0, "c1_0", None), (1, "c1_1", None), (2, "c1_2", None)]
    assert lanes([1, 2], 2, 0, **dyn) == [(0, "c1_0", None)]
    assert lanes([4, 2], 2, 0, **dyn) == [(l, f"c1_{l}", None) for l in range(4)]
    with pytest.raises(RuntimeError):                       # without the flag a non-dividing last stage keeps the host plane
        lanes([3, 2], 1, 0)
    assert lanes([4, 2, 2], 2, 1, **{"dynamic-consumers": True}) == [(1, "c1_1", None), (3, "c1_3", None)]
    with pytest.raises(RuntimeError):
        lanes([3, 2, 1], 1, 0)


@pytest.mark.parametrize("kind", ["native", "python"])
def test_broker_competing_consumers_exactly_once(kind):
    """N producers, M competing consumers on one queue (the reference's layer-2 load balancing, src/train/VGG16.py:143-154):
    every message is delivered exactly once, per-producer FIFO order is preserved for each consumer."""
    from split_learning_b200.transport import NativeBroker
    srv = NativeBroker(port=0) if kind == "native" else TcpBroker(port=0)
    try:
        n_prod, n_cons, per = 4, 3, 300
        got = [[] for _ in range(n_cons)]

        def produce(p):
            ch = TcpChannel(port=srv.port)
            for i in range(per):
                ch.publish_obj("intermediate_queue_1_0", (p, i))
            ch.close()

        def consume(c):
            ch = TcpChannel(port=srv.port)
            while True:
                m = ch.get_obj("intermediate_queue_1_0", 1.0)
                if m is None:
                    break
                got[c].append(m)
            ch.close()
        ts = [threading.Thread(target=produce, args=(p,)) for p in range(n_prod)]
        ts += [threading.Thread(target=consume, args=(c,)) for c in range(n_cons)]
        [t.start() for t in ts]
        [t.join(60) for t in ts]
        flat = [m for g in got for m in g]
        assert len(flat) == n_prod * per and len(set(flat)) == n_prod * per
        for g in got:
            for p in range(n_prod):
                seq = [i for q, i in g if q == p]
                assert seq == sorted(seq)
    finally:
        srv.close()


def test_fedavg_control_messages_over_gloo_two_processes():
    """world_size = 2 on CPU (gloo): the torch.distributed side of the peer-memory FedAvg (object all-gather, barrier,
    rounded integer-state average)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29611", os.path.join(root, "tools", "check_dist_cpu.py")],
                       capture_output=True, text=True, timeout=240, cwd=root, env=dict(os.environ, PYTHONPATH=root))
    assert r.returncode == 0 and "DIST_CPU_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


def test_queue_grammar_of_every_variant():
    """SURVEY Appendix B: forward / gradient queue names per algorithm variant, and a host data-plane round trip
    (forward message -> gradient routed back to the originating client through ``trace``)."""
    import torch
    from split_learning_b200.train.dataplane import HostDataPlane, QueueGrammar
    assert QueueGrammar("main").forward_queue(1, 0) == "intermediate_queue_1_0"
    assert QueueGrammar("flex").forward_queue(1, 2) == "intermediate_queue_1_2"
    assert QueueGrammar("vanilla_sl").forward_queue(1, 0) == QueueGrammar("cluster_fsl").forward_queue(1, 3) == "intermediate_queue_1"
    assert QueueGrammar("dcsl").forward_queue(1, 0, target="dev7") == "intermediate_queue_dev7"
    assert QueueGrammar("dcsl").forward_queue(1, 0) == "intermediate_queue_1"
    assert QueueGrammar("2ls").forward_queue(1, 0, target=3) == "intermediate_queue_1_3"
    for v in ("main", "vanilla_sl", "dcsl", "2ls", "flex"):
        assert QueueGrammar(v).gradient_queue(1, "abc") == "gradient_queue_1_abc"
    b = InProcBroker()
    first = HostDataPlane(b, "c1", 1, cluster=0)
    last = HostDataPlane(b, "c2", 2, cluster=0)
    first.send_forward("id0", torch.arange(6.0).view(2, 3), torch.tensor([1, 0]))
    m = last.recv_forward(1.0)
    assert m["data_id"] == "id0" and m["trace"] == ["c1"] and m["data"].shape == (2, 3) and m["label"].tolist() == [1, 0]
    last.send_gradient(m["data_id"], torch.ones(2, 3), m["trace"])
    g = first.recv_gradient(1.0)
    assert g["data_id"] == "id0" and g["trace"] == [] and torch.equal(g["data"], torch.ones(2, 3))
    assert last.recv_forward(0.0) is None and first.recv_gradient(0.0) is None
