"""In-box stand-in for the ``pika`` AMQP client so the UNMODIFIED reference (baseline/_ref)
can run without a RabbitMQ server.  Implements exactly the API surface the reference touches
(BlockingConnection/channel: queue_declare, basic_qos, basic_consume, start_consuming,
basic_publish, basic_get, basic_ack, queue_delete/purge; PlainCredentials,
ConnectionParameters, BasicProperties).  Queues live in one broker: in-process when every
role runs in this process, else a loopback TCP broker hosted by rank 0 (``serve``).
Nothing of split_learning_b200 is imported here.

Message-completion hook: ``on_get`` callbacks let the benchmark harness observe deliveries
(to time K pipeline steps) without touching the reference's code.

NCCL mode (``use_nccl``; ``bench.py --impl reference-nccl``) — the "reference's own NCCL build" that BASELINE.json names as
the competitor: the tensors of the two HOT queues (``intermediate_queue_*`` activations, ``gradient_queue_*`` gradients,
reference src/train/VGG16.py:20-53) travel GPU -> GPU with ``torch.distributed`` NCCL ``isend`` / ``recv``; only a small
header (data_id, label, trace, shape) goes through the broker, and the control verbs stay on the broker as before.  The
reference trainers are untouched: they still hand the shim a pickled dict with a CPU NumPy array and get one back, so the
D2H / H2D copies at the trainer boundary remain (they are part of the reference's code), but the wire itself is NCCL p2p
over NVLink instead of pickle-over-TCP.  Routing is static (first-stage rank r -> last-stage rank n_first + r % n_last; the
gradient returns to the rank the activation came from), forward and backward use separate communicators so the 1F1B
schedule cannot dead-lock on NCCL's per-communicator ordering.
"""
import collections
import os
import pickle
import socket
import struct
import threading
import time

_EMPTY_WAIT = 2e-4          # a fast broker round trip; keeps busy-polling loops from hogging the GIL


class _Store:
    def __init__(self):
        self.q = collections.defaultdict(collections.deque)
        self.cv = threading.Condition()

    def publish(self, key, body):
        with self.cv:
            self.q[key].append(body)
            self.cv.notify_all()

    def get(self, key, wait=_EMPTY_WAIT):
        with self.cv:
            d = self.q[key]
            if not d and wait:
                self.cv.wait(wait)
            return d.popleft() if d else None

    def delete(self, key):
        with self.cv:
            self.q.pop(key, None)


_NCCL = None                # dict(rank, n_first, n_last, fwd, bwd, device, origin, pending) in NCCL mode


def use_nccl(rank, n_first, n_last, device):
    """Route the payload of the two hot queues over NCCL p2p.  Collective: every rank must call (creates two groups)."""
    global _NCCL
    import torch.distributed as dist
    world = dist.get_world_size()
    fwd = dist.new_group(list(range(world)))
    bwd = dist.new_group(list(range(world)))
    _NCCL = {"rank": rank, "n_first": n_first, "n_last": n_last, "fwd": fwd, "bwd": bwd, "device": device,
             "origin": {}, "pending": [], "sent": 0, "received": 0, "bytes": 0}


def nccl_stats():
    return None if _NCCL is None else {k: _NCCL[k] for k in ("sent", "received", "bytes")}


def _nccl_publish(chan, routing_key, body):
    import torch
    import torch.distributed as dist
    st = _NCCL
    msg = pickle.loads(body)
    arr = msg.pop("data")
    t = torch.from_numpy(arr).to(st["device"])
    if routing_key.startswith("intermediate_queue_"):
        dst = st["n_first"] + st["rank"] % st["n_last"]
        key, group = f"{routing_key}@{dst}", st["fwd"]
    else:                                   # gradient_queue_{layer}_{client_id}: back to where the activation came from
        dst = st["origin"][routing_key.split("_", 3)[3]]
        key, group = routing_key, st["bwd"]
    header = {"__nccl__": 1, "src": st["rank"], "shape": tuple(arr.shape), "dtype": str(arr.dtype), "rest": msg}
    chan._pub(key, pickle.dumps(header, protocol=pickle.HIGHEST_PROTOCOL))
    work = dist.isend(t, dst, group=group)
    st["pending"].append((work, t))
    st["pending"] = [(w, x) for (w, x) in st["pending"] if not w.is_completed()][-64:]
    st["sent"] += 1
    st["bytes"] += arr.nbytes


def _nccl_receive(queue, body):
    import numpy as np
    import torch
    import torch.distributed as dist
    st = _NCCL
    h = pickle.loads(body)
    if not (isinstance(h, dict) and h.get("__nccl__")):
        return body
    fwd = queue.startswith("intermediate_queue_")
    buf = torch.empty(h["shape"], dtype=getattr(torch, h["dtype"]), device=st["device"])
    dist.recv(buf, src=h["src"], group=st["fwd"] if fwd else st["bwd"])
    msg = h["rest"]
    if fwd and msg.get("trace"):
        st["origin"][str(msg["trace"][-1])] = h["src"]
    msg["data"] = buf.cpu().numpy()
    st["received"] += 1
    return pickle.dumps(msg, protocol=pickle.HIGHEST_PROTOCOL)


_LOCAL = _Store()
_REMOTE = None              # (host, port) when a TCP broker is used
on_get = []                 # callbacks(queue_name, body) fired on every successful basic_get


def _send(sock, obj):
    b = pickle.dumps(obj, protocol=pickle.HIGHEST_PROTOCOL)
    sock.sendall(struct.pack("<Q", len(b)) + b)


def _recv(sock):
    def exact(n):
        buf = bytearray()
        while len(buf) < n:
            chunk = sock.recv(min(1 << 20, n - len(buf)))
            if not chunk:
                raise ConnectionError("closed")
            buf += chunk
        return bytes(buf)
    (n,) = struct.unpack("<Q", exact(8))
    return pickle.loads(exact(n))


def serve(host="127.0.0.1", port=29655):
    """Start the TCP broker (rank 0)."""
    srv = socket.socket()
    srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
    srv.bind((host, port))
    srv.listen(64)

    def client(conn):
        conn.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)
        try:
            while True:
                op, key, arg = _recv(conn)
                if op == "pub":
                    _LOCAL.publish(key, arg)
                elif op == "get":
                    _send(conn, _LOCAL.get(key))
                elif op == "del":
                    _LOCAL.delete(key)
        except (ConnectionError, OSError, EOFError):
            pass

    def loop():
        while True:
            try:
                c, _ = srv.accept()
            except OSError:
                return
            threading.Thread(target=client, args=(c,), daemon=True).start()
    threading.Thread(target=loop, daemon=True).start()
    return srv


def use_remote(host="127.0.0.1", port=29655):
    global _REMOTE
    _REMOTE = (host, port)


class PlainCredentials:
    def __init__(self, *a, **k): pass


class ConnectionParameters:
    def __init__(self, *a, **k): pass


class BasicProperties:
    def __init__(self, reply_to=None, **k):
        self.reply_to = reply_to


class _Method:
    def __init__(self, tag):
        self.delivery_tag = tag


class _Channel:
    def __init__(self, conn):
        self._conn = conn
        self._consumers = []
        self._tag = 0

    # -- transport ---------------------------------------------------------
    def _pub(self, key, body):
        if self._conn.sock is None:
            _LOCAL.publish(key, body)
        else:
            with self._conn.lock:
                _send(self._conn.sock, ("pub", key, body))

    def _get(self, key):
        if self._conn.sock is None:
            return _LOCAL.get(key)
        with self._conn.lock:
            _send(self._conn.sock, ("get", key, None))
            return _recv(self._conn.sock)

    # -- pika surface ------------------------------------------------------
    def queue_declare(self, queue=None, durable=False, **k): return None
    def basic_qos(self, prefetch_count=0, **k): return None
    def queue_purge(self, queue=None): return None

    def queue_delete(self, queue=None):
        if self._conn.sock is None:
            _LOCAL.delete(queue)

    def basic_publish(self, exchange="", routing_key="", body=b"", properties=None, **k):
        if _NCCL is not None and routing_key.startswith(("intermediate_queue_", "gradient_queue_")):
            return _nccl_publish(self, routing_key, body)
        self._pub(routing_key, body)

    def basic_get(self, queue=None, auto_ack=False):
        hot = _NCCL is not None and queue.startswith(("intermediate_queue_", "gradient_queue_"))
        key = f"{queue}@{_NCCL['rank']}" if (hot and queue.startswith("intermediate_queue_")) else queue
        body = self._get(key)
        if body is None:
            return None, None, None
        if hot:
            body = _nccl_receive(queue, body)
        for cb in on_get:
            cb(queue, body)
        self._tag += 1
        return _Method(self._tag), BasicProperties(), body

    def basic_ack(self, delivery_tag=0, **k): return None

    def basic_consume(self, queue=None, on_message_callback=None, **k):
        self._consumers.append((queue, on_message_callback))

    def start_consuming(self):
        while self._consumers:
            for q, cb in list(self._consumers):
                body = self._get(q)
                if body is not None:
                    self._tag += 1
                    cb(self, _Method(self._tag), BasicProperties(), body)

    def stop_consuming(self):
        self._consumers = []


class BlockingConnection:
    def __init__(self, parameters=None):
        self.lock = threading.Lock()
        self.sock = None
        if _REMOTE is not None:
            deadline = time.time() + 60
            while True:
                try:
                    self.sock = socket.create_connection(_REMOTE, timeout=5)
                    break
                except OSError:
                    if time.time() > deadline:
                        raise
                    time.sleep(0.05)
            self.sock.settimeout(None)
            self.sock.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)

    def channel(self):
        return _Channel(self)

    def process_data_events(self, *a, **k): return None

    def close(self):
        if self.sock is not None:
            self.sock.close()
