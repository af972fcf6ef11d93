"""Coordinator (reference L4, src/Server.py:22-434) — main algorithm.

Same verbs, same bookkeeping, same aggregation maths; differences are deliberate:
  * no RabbitMQ: the server owns an in-box broker (``transport``) and serves ``rpc_queue``;
  * the fixed ``time.sleep(25)`` between START and SYN (src/Server.py:289) is replaced by a
    READY barrier (every trainable client acknowledges START before SYN is sent);
  * a watchdog raises instead of dead-locking when a client disappears;
  * numpy's RNG is seeded as well as ``random`` (reference quirk C4);
  * ``selection-mode`` compares ``profile["speed"]`` (the reference compares the dict and
    would raise, quirk C3);
  * N > 2 stages are supported end to end (middle stages; auto-mode uses ``partition_multi``).
When clients report ``resident=True`` in UPDATE (GPU path: parameters were averaged in place
over NVLink by ``parallel.fedavg``), stage dicts arrive only from the designated uploader of
each (cluster, stage) and are taken as already averaged.
"""
from __future__ import annotations

import os
import random
import time
from typing import Dict, List, Optional

import numpy as np
import torch

from . import messages as M
from .checkpoint import checkpoint_path, load_checkpoint, save_checkpoint, slice_for_stage
from .config import Config
from .data.distribution import label_counts as make_label_counts
from .fedavg import fedavg_state_dicts, has_nan
from .log import Logger, print_with_color
from .plan import ClientInfo, ClusterPlan, Topology
from .planning import auto_threshold, clustering_algorithm, partition, partition_multi
from .transport import Channel


import contextlib
import threading

_NO_LOCK = contextlib.nullcontext()


class Server:
    ALGORITHM = "main"

    def __init__(self, config: Config, channel: Channel, logger: Optional[Logger] = None, workdir: str = "."):
        self.cfg = config
        self.ch = channel
        self.workdir = workdir
        self.total_clients: List[int] = list(config.clients)
        self.num_stages = len(self.total_clients)
        self.global_round = config.global_round
        self.round = self.global_round
        self.learning = dict(config.learning)
        self.model_name, self.data_name = config.model, config.data_name
        self.save_parameters = config.save_parameters
        self.load_parameters = config.load_parameters
        self.validation = config.validation
        self.refresh = config.refresh
        if config.random_seed:
            random.seed(config.random_seed)
            np.random.seed(int(config.random_seed) % (2 ** 32))

        self.ch.queue_declare(M.RPC_QUEUE)
        self.register_clients = [0] * self.num_stages
        self.current_clients = [0] * self.num_stages
        self.clients: List[ClientInfo] = []
        self.topology: Optional[Topology] = None
        self.label_counts = None
        self.size_data = None
        self.round_result = True
        self.reject_sent = False
        self.first_layer_done: List[int] = []
        self.params: List[List[List[dict]]] = []
        self.sizes: List[List[List[int]]] = []
        self.avg_state_dict: List[List[dict]] = []
        self.ready_pending: set = set()
        self.done = False
        self.history: List[dict] = []         # per-round metrics (loss/acc/seconds)
        self._round_t0 = time.monotonic()
        self.watchdog = float(config.b200.get("watchdog-seconds", 120.0))
        # liveness: clients beacon every ``heartbeat-seconds``; one that has beaconed before and stays silent for
        # ``watchdog-seconds`` is declared dead (the round is aborted with STOP instead of dead-locking); the server relays
        # a beacon to every client so that *their* waits (PAUSE, sequential turns, long rounds) never expire on a live run
        self.heartbeat = float(config.b200.get("heartbeat-seconds", min(10.0, self.watchdog / 4)))
        self.last_seen: Dict[str, float] = {}
        self._last_beacon = time.monotonic()
        self.logger = logger or Logger(os.path.join(config.log_path, "app.log"), config.debug_mode)
        self.logger.log_info(f"Application start. Server is waiting for {self.total_clients} clients.")
        for w in config.warnings:
            self.logger.log_warning(w)

    # ------------------------------------------------------------------ loop
    def start(self, idle_timeout: Optional[float] = None) -> None:
        """Serve ``rpc_queue`` until training is finished (blocking)."""
        last = time.monotonic()
        limit = idle_timeout if idle_timeout is not None else max(self.watchdog * 4, 600.0)
        self._start_checkpoint_receiver()
        try:
            self._serve(last, limit)
        finally:
            self._ckpt_stop.set()
            if self._ckpt_rx is not threading.current_thread():
                self._ckpt_rx.join(5.0)

    def _serve(self, last: float, limit: float) -> None:
        while not self.done:
            m = self.ch.get_obj(M.RPC_QUEUE, 0.1)
            now = time.monotonic()
            if now - self._last_beacon >= self.heartbeat:
                self._beacon(now)
            if m is None:
                if now - last > limit:
                    raise TimeoutError(f"server: no client message for {limit}s (registered "
                                       f"{self.register_clients} of {self.total_clients})")
                continue
            last = now
            self.on_request(m)
        self._finish_checkpoints()

    def _start_checkpoint_receiver(self) -> None:
        """CHECKPOINT messages arrive on their own queue and are taken by their own thread (own channel): receiving a
        134 MB body takes tens of milliseconds, during which the control loop must stay free for NOTIFY / UPDATE."""
        import threading
        self._ckpt_lock = threading.Lock()
        self._ckpt_stop = threading.Event()
        ch = self.ch.clone()
        ch.queue_declare(M.CKPT_QUEUE)

        def loop():
            while not self._ckpt_stop.is_set():
                try:
                    m = ch.get_obj(M.CKPT_QUEUE, 0.2)
                except Exception as e:              # noqa — broker gone: the run is over
                    self.logger.log_warning(f"checkpoint receiver stopped: {e}")
                    return
                if m is not None and m.get("action") == M.CHECKPOINT:
                    self.on_checkpoint(m)
        self._ckpt_rx = threading.Thread(target=loop, daemon=True, name="slb200-ckpt-receiver")
        self._ckpt_rx.start()

    def _finish_checkpoints(self, timeout: float = 180.0) -> None:
        """Training is over; stage leaders may still be shipping the last rounds' parameters for the checkpoint."""
        deadline = time.monotonic() + timeout
        while self.__dict__.get("_ckpt_pending") and time.monotonic() < deadline:
            time.sleep(0.01)
        if self.__dict__.get("_ckpt_pending"):
            self.logger.log_warning(f"checkpoint parts of rounds {sorted(self._ckpt_pending)} never arrived")
        if self.__dict__.get("_ckpt_stop") is not None:
            self._ckpt_stop.set()
            self._ckpt_rx.join(5.0)
        self.drain_checkpoints()

    def _beacon(self, now: float) -> None:
        """Relay liveness to every client and check that every beaconing client is still there."""
        self._last_beacon = now
        total = self.__dict__.get("_handled", 0) + sum(int(v) for v in self.__dict__.get("progress_of", {}).values())
        for c in self.clients:
            self.send_to_response(c.client_id, M.heartbeat(progress=total))
        dead = [cid for cid, t in self.last_seen.items() if now - t > max(self.watchdog, 3 * self.heartbeat)]
        if dead and not self.done:
            self.logger.log_error(f"clients silent for {self.watchdog}s: {dead}; stopping the run")
            self.notify_clients(start=False)
            raise TimeoutError(f"server: client(s) {dead} stopped sending heartbeats")

    def on_request(self, message: dict) -> None:
        action = message["action"]
        if action == M.HEARTBEAT:
            cid = str(message.get("client_id"))
            self.last_seen[cid] = time.monotonic()
            if message.get("progress") is not None:
                self.__dict__.setdefault("progress_of", {})[cid] = int(message["progress"])
            return
        self._handled = self.__dict__.get("_handled", 0) + 1          # control traffic is progress too
        handler = {M.REGISTER: self.on_register, M.NOTIFY: self.on_notify, M.UPDATE: self.on_update,
                   M.READY: self.on_ready, M.CHECKPOINT: self.on_checkpoint}.get(action)
        if handler is None:
            self.logger.log_warning(f"unknown action {action}")
            return
        handler(message)

    def send_to_response(self, client_id, message: dict) -> None:
        self.ch.publish_obj(M.reply_queue(client_id), message)

    # ------------------------------------------------------------- REGISTER
    def on_register(self, message: dict) -> None:
        cid, layer_id = str(message["client_id"]), int(message["layer_id"])
        profile, cluster = message.get("profile"), message.get("cluster", -1)
        if self.size_data is None and layer_id == 1 and profile:
            self.size_data = profile.get("size_data")
        if not any(c.client_id == cid for c in self.clients):      # duplicate REGISTER de-dup
            extras = {k: message[k] for k in ("idx", "in_cluster", "out_cluster", "select", "rank") if k in message}
            self.clients.append(ClientInfo(cid, layer_id, profile, cluster if cluster is not None else -1,
                                           rank=message.get("rank"), idx=message.get("idx"), extras=extras))
            self.register_clients[layer_id - 1] += 1
        print_with_color(f"[<<<] REGISTER from {cid} (layer {layer_id}, cluster {cluster})", "blue")
        if self.register_clients == self.total_clients:
            print_with_color("All clients are connected. Sending notifications.", "green")
            self.distribution()
            self.cluster_and_selection()
            print_with_color(f"List cut point: {self.topology.cut_layers()}", "yellow")
            print_with_color(f"Infor clusters: {self.topology.infor_cluster()}", "yellow")
            self.logger.log_info(f"{self.learning}")
            self.begin_round()

    def label_matrix(self):
        """Fixed non-IID matrix, if configured (the FLEX / 2LS servers default to their built-in presets)."""
        return self.cfg.label_matrix

    def distribution(self) -> None:
        n1 = self.total_clients[0]
        self.label_counts = make_label_counts(
            n1, self.cfg.num_label, self.cfg.num_sample, non_iid=self.cfg.non_iid,
            alpha=self.cfg.dirichlet_alpha, seed=self.cfg.random_seed, non_iid_rate=self.cfg.non_iid_rate,
            matrix=self.label_matrix())
        pool = self.label_counts.tolist()
        for c in self.clients:
            c.label_counts = pool.pop() if c.layer_id == 1 else []

    # ------------------------------------------------- topology / selection
    def cluster_and_selection(self) -> None:
        cfg = self.cfg
        if cfg.auto_mode:
            self._auto_topology()
        elif cfg.cluster_mode:
            ncl = cfg.num_cluster
            for c in self.clients:
                c.train = True
                if c.cluster is None or c.cluster < 0:
                    c.cluster = 0
            # clients that registered without --cluster are dealt to clusters by infor-cluster
            self._assign_unclustered(ncl)
            clusters = []
            for k in range(ncl):
                members = [[c.client_id for c in self.clients if c.cluster == k and c.layer_id == s + 1]
                           for s in range(self.num_stages)]
                clusters.append(ClusterPlan(k, list(cfg.cluster_cut_layers[k]), members))
            self.topology = Topology(self.num_stages, clusters)
        else:
            for c in self.clients:
                c.cluster, c.train = 0, True
            # members of a stage in GPU-ordinal order when the clients announced one (REGISTER ``rank``): the device data
            # plane pairs lane i with member i % n of the next stage, so the launcher decides the placement (ring / split)
            order = sorted(self.clients, key=lambda c: (c.rank is None, c.rank if c.rank is not None else 0))
            members = [[c.client_id for c in order if c.layer_id == s + 1] for s in range(self.num_stages)]
            self.topology = Topology(self.num_stages, [ClusterPlan(0, list(cfg.no_cluster_cut_layers), members)])
        self._reset_round_buffers()

    def _assign_unclustered(self, ncl: int) -> None:
        """Main-tree manual cluster mode trusts ``--cluster``; if every client came with the
        default -1→0 and infor-cluster is given, fill clusters in registration order."""
        if not self.cfg.infor_cluster_given:
            return
        want = self.cfg.infor_cluster
        have = [[sum(1 for c in self.clients if c.cluster == k and c.layer_id == s + 1)
                 for s in range(self.num_stages)] for k in range(ncl)]
        if have == [list(w) for w in want]:
            return
        for s in range(self.num_stages):
            stage_clients = [c for c in self.clients if c.layer_id == s + 1]
            it = iter(stage_clients)
            for k in range(ncl):
                for _ in range(want[k][s]):
                    try:
                        next(it).cluster = k
                    except StopIteration:
                        break

    def _auto_topology(self) -> None:
        cfg = self.cfg
        ncl = cfg.sel_num_cluster
        labels, _ = clustering_algorithm(self.label_counts, ncl)
        labels = labels.tolist()
        for c in self.clients:
            c.train = True
            if c.layer_id == 1:
                c.cluster = int(labels.pop())
            elif c.cluster is None or c.cluster < 0:
                c.cluster = 0
        if cfg.selection_mode:
            for k in range(ncl):
                speeds = [c.profile["speed"] for c in self.clients if c.layer_id == 1 and c.cluster == k and c.profile]
                thr = auto_threshold(speeds) if speeds else 0.0
                for c in self.clients:
                    if c.layer_id == 1 and c.cluster == k and c.profile and c.profile["speed"] < thr:
                        c.train = False
                        self.total_clients[0] -= 1
                        print_with_color(f"Remove a device has id: {c.client_id}", "red")
        clusters = []
        for k in range(ncl):
            per_stage = [[c for c in self.clients if c.cluster == k and c.layer_id == s + 1 and c.train]
                         for s in range(self.num_stages)]
            exe = [[c.profile["exe_time"] for c in st] for st in per_stage]
            net = [[c.profile["network"] for c in st] for st in per_stage]
            if self.num_stages == 2:
                cut = partition(exe[0], net[0], exe[1], net[1], self.size_data)
            else:
                cut = partition_multi(exe, net, self.size_data)
            clusters.append(ClusterPlan(k, cut, [[c.client_id for c in st] for st in per_stage]))
        self.topology = Topology(self.num_stages, clusters)

    def _reset_round_buffers(self) -> None:
        ncl = len(self.topology.clusters)
        self.params = [[[] for _ in range(self.num_stages)] for _ in range(ncl)]
        self.sizes = [[[] for _ in range(self.num_stages)] for _ in range(ncl)]
        self.avg_state_dict = [[] for _ in range(ncl)]
        self.first_layer_done = [0] * ncl

    # ------------------------------------------------------------ rounds
    def begin_round(self) -> None:
        self._round_t0 = time.monotonic()
        self._phase = {}
        self.logger.log_info(f"Start training round {self.global_round - self.round + 1}")
        self.notify_clients(start=True)
        self._mark("start_sent")

    def _mark(self, name: str) -> None:
        """Milliseconds since the round began at which a protocol phase completed (round-overhead accounting)."""
        self.__dict__.setdefault("_phase", {})[name] = (time.monotonic() - self._round_t0) * 1e3

    def stage_parameters_for(self, c: ClientInfo, layers: List[int]):
        """Resume path (src/Server.py:230-254): slice the full checkpoint for this stage."""
        if not self.save_parameters:
            return None
        path = checkpoint_path(self.model_name, self.data_name, self.workdir)
        full = load_checkpoint(path)
        if full is None:
            return None
        try:
            sd = slice_for_stage(full, self.model_name, self.data_name, layers)
            print_with_color(f"Load model {path} successfully", "green")
            return sd
        except KeyError as e:
            self.logger.log_warning(f"checkpoint {path} lacks key {e}; starting fresh")
            return None

    def start_payload(self, c: ClientInfo) -> dict:
        layers = self.topology.layers_for(c.cluster, c.layer_id)
        if self.topology.clusters[c.cluster].cut_layers[:1] == [0] and c.layer_id == 1:
            layers = [0, 0]
        # every client averaged in place on the device (all clusters joined one all-reduce): nothing to ship
        resident = bool(getattr(self, "all_resident", False))
        params = None if resident else self.stage_parameters_for(c, layers)
        return M.start(params, layers, self.model_name, self.data_name,
                       self.learning, c.label_counts, self.refresh, c.cluster,
                       num_layers=self.num_stages, round=self.global_round - self.round + 1,
                       peers=self._peer_table(c), num_clusters=len(self.topology.clusters), resident=resident,
                       save_parameters=bool(self.save_parameters),
                       async_checkpoint=bool(self.save_parameters and not self.validation
                                             and self.cfg.b200.get("async-checkpoint", True)))

    def _peer_table(self, c: ClientInfo) -> dict:
        """Who is upstream/downstream of this client (ranks + ids): lets the GPU data plane
        wire peer mailboxes without further round trips."""
        cl = self.topology.clusters[c.cluster]
        table = {}
        for s, ids in enumerate(cl.members):
            table[s + 1] = [(cid, next((x.rank for x in self.clients if x.client_id == cid), None)) for cid in ids]
        everyone = [(x.client_id, int(x.cluster), int(x.layer_id)) for x in self.clients if x.train]
        return {"members": table, "cut_layers": list(cl.cut_layers), "all": everyone}

    def notify_clients(self, start: bool = True) -> None:
        if not start:
            for c in self.clients:
                print_with_color(f"[>>>] Sent stop training request to client {c.client_id}", "red")
                self.send_to_response(c.client_id, M.stop())
            self.done = True
            return
        self.ready_pending = set()
        for c in self.clients:
            if c.train:
                self.ready_pending.add(c.client_id)
                self.send_to_response(c.client_id, self.start_payload(c))
                print_with_color(f"[>>>] Sent start training request to client {c.client_id}", "red")
            elif not self.reject_sent:
                self.send_to_response(c.client_id, M.stop("Reject Device"))
        self.reject_sent = True

    def on_ready(self, message: dict) -> None:
        self.ready_pending.discard(str(message["client_id"]))
        if not self.ready_pending:
            for c in self.clients:
                if c.train:
                    self.send_to_response(c.client_id, M.syn())
            self._mark("syn_sent")

    # -------------------------------------------------------------- NOTIFY
    def on_notify(self, message: dict) -> None:
        cluster = int(message.get("cluster") or 0)
        if int(message["layer_id"]) == 1:
            self.first_layer_done[cluster] += 1
        need = sum(1 for c in self.clients if c.layer_id == 1 and c.cluster == cluster and c.train)
        if self.first_layer_done[cluster] == need:
            self.first_layer_done[cluster] = 0
            print_with_color(f"Received finish training notification cluster {cluster}", "yellow")
            for c in self.clients:
                if c.train and c.cluster == cluster:
                    self.send_to_response(c.client_id, self.pause_payload(c))
            self._mark("pause_sent")

    def pause_payload(self, c: ClientInfo) -> dict:
        return M.pause()

    # -------------------------------------------------------------- UPDATE
    def on_update(self, message: dict) -> None:
        cid, layer_id = str(message["client_id"]), int(message["layer_id"])
        cluster = int(message.get("cluster") or 0)
        print_with_color(f"[<<<] UPDATE from {cid}: {message.get('message')}", "blue")
        self.current_clients[layer_id - 1] += 1
        if not message.get("result", True):
            self.round_result = False
        sd = message.get("parameters")
        self._resident_votes = getattr(self, "_resident_votes", [])
        self._resident_votes.append(bool(message.get("resident", False)))
        if message.get("checkpoint_follows"):
            with self.__dict__.get("_ckpt_lock") or _NO_LOCK:
                rnd = int(message["checkpoint_follows"])
                if rnd not in self.__dict__.setdefault("_ckpt_done", set()):
                    self.__dict__.setdefault("_ckpt_pending", set()).add(rnd)
        if message.get("device_ms") is not None:
            self._device_ms = getattr(self, "_device_ms", []) + [float(message["device_ms"])]
        if layer_id == 1:
            self._first_mb = self.__dict__.get("_first_mb", 0) + int(message.get("size") or 0)
        if message.get("loss") is not None:
            self._losses = getattr(self, "_losses", []) + [float(message["loss"])]
        if message.get("timing"):
            per = {k: ((float(v) - self._round_t0) * 1e3 if k.startswith("at_") else float(v)) for k, v in message["timing"].items()}
            per["layer_id"] = layer_id
            self.__dict__.setdefault("_client_timings", []).append(per)
            acc = self.__dict__.setdefault("_client_timing", {})
            for k, v in message["timing"].items():
                if k.startswith("at_"):                     # absolute stamps -> ms since the round began, latest client
                    v = (float(v) - self._round_t0) * 1e3
                acc[k] = max(acc.get(k, 0.0), float(v))
        if self.save_parameters and self.round_result and sd is not None:
            if has_nan(sd):
                self.round_result = False
            else:
                self.params[cluster][layer_id - 1].append(sd)
                # resident=True: already the NVLink-averaged stage; weight irrelevant
                self.sizes[cluster][layer_id - 1].append(message.get("size", 1))
        if self.current_clients == self.total_clients:
            self.finish_round()

    def finish_round(self) -> None:
        print_with_color("Collected all parameters.", "yellow")
        self.current_clients = [0] * self.num_stages
        votes = getattr(self, "_resident_votes", [])
        # every client averaged in place over peer memory and still holds the result: next START needs no payload
        self.all_resident = bool(votes) and all(votes) and self.round_result
        self._resident_votes = []
        metrics = {"round": self.global_round - self.round + 1, "ok": self.round_result,
                   "seconds": time.monotonic() - self._round_t0}
        if getattr(self, "_device_ms", None):         # device time of the training loops (CUDA events), max over clients
            metrics["device_ms"] = max(self._device_ms)
        if getattr(self, "_losses", None):
            metrics["train_loss"] = sum(self._losses) / len(self._losses)
        self._device_ms, self._losses = [], []
        metrics["first_stage_microbatches"] = self.__dict__.get("_first_mb", 0)       # the round's training volume
        self._first_mb = 0
        self._mark("updates_in")
        metrics["phases_ms"] = dict(self._phase)
        if self.__dict__.get("_client_timing"):
            metrics["client_timing_ms"] = dict(self._client_timing)       # max over clients, per client-side phase
            metrics["client_timings"] = list(self.__dict__.get("_client_timings", []))
            self._client_timing, self._client_timings = {}, []
        if self.save_parameters and self.round_result:
            for k in range(len(self.topology.clusters)):
                self.avg_all_parameters(k)
            full = self.concatenate_and_avg_clusters()
            ok = True
            if self.validation and full:
                from .validation import get_val
                ok, val = get_val(self.model_name, self.data_name, full, self.logger,
                                  native=self.cfg.b200.get("native-validation", False),
                                  speech_features=self.cfg.b200.get("speech-features", "engine"))
                metrics.update(val)
            if ok:
                if full:
                    save_checkpoint(full, checkpoint_path(self.model_name, self.data_name, self.workdir),
                                    meta={"round": metrics["round"]})
                self.round -= 1
            else:
                self.logger.log_warning("Training failed!")
                self.round = 0
        else:
            self.round -= 1          # reference: a NaN round still counts (quirk C5)
        self.history.append(metrics)
        self._reset_round_buffers()
        self.round_result = True
        if self.round > 0:
            self.begin_round()
        else:
            self.logger.log_info("Stop training !!!")
            self.notify_clients(start=False)

    # ---------------------------------------------------------- asynchronous checkpoint (device plane)
    def on_checkpoint(self, message: dict) -> None:
        """Stage state-dicts of an already finished ``resident`` round: collected per round, written by a background thread
        once every stage of the (first) cluster has arrived — the next round is not held up by a 134 MB upload + torch.save."""
        import threading
        rnd = int(message["round"])
        with self.__dict__.get("_ckpt_lock") or _NO_LOCK:
            parts = self.__dict__.setdefault("_ckpt_parts", {}).setdefault(rnd, {})
            parts[int(message["layer_id"])] = message["parameters"]
            if len(parts) < self.num_stages:
                return
            full: Dict[str, torch.Tensor] = {}
            for s in sorted(parts):
                full.update(parts[s])
            del self._ckpt_parts[rnd]
            self.__dict__.setdefault("_ckpt_done", set()).add(rnd)
            self.__dict__.setdefault("_ckpt_pending", set()).discard(rnd)
        path = checkpoint_path(self.model_name, self.data_name, self.workdir)

        def write():
            with self.__dict__.setdefault("_ckpt_write_lock", threading.Lock()):     # one writer at a time, never back in time
                if rnd < self.__dict__.get("_ckpt_written", 0):
                    return
                save_checkpoint(full, path, meta={"round": rnd})
                self._ckpt_written = rnd
            self.logger.log_info(f"checkpoint of round {rnd} written ({len(full)} entries)")
        t = threading.Thread(target=write, daemon=True, name=f"slb200-ckpt-{rnd}")
        self.__dict__.setdefault("_ckpt_threads", []).append(t)
        t.start()

    def drain_checkpoints(self, timeout: float = 60.0) -> None:
        for t in self.__dict__.get("_ckpt_threads", []):
            t.join(timeout)

    # ---------------------------------------------------------- aggregation
    def avg_all_parameters(self, cluster: int) -> None:
        self.avg_state_dict[cluster] = []
        for stage, dicts in enumerate(self.params[cluster]):
            sizes = self.sizes[cluster][stage]
            if not dicts or not sizes:
                self.avg_state_dict[cluster].append({})
                continue
            self.avg_state_dict[cluster].append(fedavg_state_dicts(dicts, weights=sizes))

    def concatenate_and_avg_clusters(self) -> Dict[str, torch.Tensor]:
        cluster_dicts = []
        for k, cl in enumerate(self.topology.clusters):
            layers = self.avg_state_dict[k] or []
            if not layers:
                continue
            full: Dict[str, torch.Tensor] = {}
            if cl.cut_layers and cl.cut_layers[0] == 0:
                full.update(layers[0])
            else:
                for sd in layers:
                    full.update(sd)
            if full:
                cluster_dicts.append(full)
        if not cluster_dicts:
            return {}
        return fedavg_state_dicts(cluster_dicts)
