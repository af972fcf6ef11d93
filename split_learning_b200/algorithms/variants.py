"""The five ``other/*`` algorithm forks of the reference as policies over the main skeleton.

=============  =====================================================================================
vanilla_sl     classic sequential split learning: first-stage clients train one after another, the
               server hands client i's weights to client i+1; later stages keep training throughout;
               only the last edge + later-stage devices are averaged; ``limited-time`` budget;
               ``clip-grad-norm``; NaN-gated validation   (other/Vanilla_SL/src/Server.py:95-268)
cluster_fsl    clusters run sequentially, first-stage clients inside a cluster in parallel and
               FedAvg'd, the average seeds the next cluster   (other/Cluster_FSL/src/Server.py:97-200)
dcsl           cluster_fsl + ``local-round`` epochs, strict 1-in-flight first stage, per-device
               round-robin queues and SDA batch concatenation on the last stage
               (other/DCSL/src/Scheduler.py:23-26,99-133,152-221; Server.py:138,237,285-298)
flex           per-cluster cut layers, device selection flag, multi-rate aggregation: clients upload
               every ``t-c`` rounds, edges every ``t-g`` rounds (PAUSE carries ``send``); global =
               unweighted mean over clusters of (client average ∪ edge)  (other/FLEX/src/Server.py:105-309)
2ls            two-level clusters: out-clusters sequential in shuffled order, in-clusters concurrent
               with a dedicated last-stage device each (queue per ``idx``), per-in-cluster FedAvg
               then FedAsync merge (alpha = 1/(1+k)) into the running global model, checkpoint after
               every merge   (other/2LS/src/Server.py:117-233)
=============  =====================================================================================
"""
from __future__ import annotations

import random
import time
from typing import List, Optional

from .. import messages as M
from ..checkpoint import checkpoint_path, save_checkpoint
from ..client import RpcClient
from ..fedavg import fedasync_merge, fedavg_state_dicts, has_nan
from ..log import print_with_color
from ..plan import ClientInfo, ClusterPlan, Topology
from ..server import Server
from ..train import HostDataPlane, QueueGrammar


# =============================================================================== sequential family
class SequentialServer(Server):
    """Groups of first-stage clients run one after another (group = one client for vanilla_sl,
    one cluster for cluster_fsl / dcsl); stages >= 2 are shared by every group."""

    ALGORITHM = "vanilla_sl"
    STRICT_VALIDATION = True
    STOP_ON_VALIDATION_FAILURE = False        # Vanilla_SL / Cluster_FSL retry the round; DCSL stops (see DCSLServer)
    MAX_ROUND_RETRIES = 5                     # a persistently diverging run must not loop forever (the reference would)

    def cluster_and_selection(self) -> None:
        cfg = self.cfg
        for c in self.clients:
            c.train = True
        firsts = [c for c in self.clients if c.layer_id == 1]
        if self.ALGORITHM == "vanilla_sl":
            self.groups: List[List[ClientInfo]] = [[c] for c in firsts]
        else:
            ids = sorted({max(c.cluster, 0) for c in firsts})
            self.groups = [[c for c in firsts if max(c.cluster, 0) == k] for k in ids]
        for c in self.clients:
            c.cluster = 0
        members = [[c.client_id for c in self.clients if c.layer_id == s + 1] for s in range(self.num_stages)]
        cut = cfg.cluster_cut_layers[0] if (cfg.cluster_mode and cfg.cluster_cut_layers) else cfg.no_cluster_cut_layers
        self.topology = Topology(self.num_stages, [ClusterPlan(0, list(cut), members)])
        self._reset_round_buffers()
        self.gidx = 0
        self.handoff = None                       # averaged first-stage weights of the previous group
        self.group_updates: List[dict] = []
        self.group_sizes: List[int] = []

    def extra_start(self, c: ClientInfo) -> dict:
        return {"config_time": self.cfg.limited_time, "local_round": self.cfg.local_round}

    def start_payload(self, c: ClientInfo) -> dict:
        p = super().start_payload(c)
        p.update(self.extra_start(c))
        if c.layer_id == 1 and self.handoff is not None:
            p["parameters"] = self.handoff
        return p

    def _start_wave(self, clients: List[ClientInfo]) -> None:
        self.ready_pending = {c.client_id for c in clients}
        self.wave = list(clients)
        for c in clients:
            self.send_to_response(c.client_id, self.start_payload(c))

    def begin_round(self) -> None:
        self._round_t0 = time.monotonic()
        self.logger.log_info(f"Start training round {self.global_round - self.round + 1}")
        self.gidx, self.handoff = 0, None
        self.group_updates, self.group_sizes = [], []
        later = [c for c in self.clients if c.layer_id > 1]
        self._start_wave(later + self.groups[0])

    def on_ready(self, message: dict) -> None:
        self.ready_pending.discard(str(message["client_id"]))
        if not self.ready_pending:
            for c in self.wave:
                self.send_to_response(c.client_id, M.syn())
            self.wave = []

    def on_notify(self, message: dict) -> None:
        self.first_layer_done[0] += 1
        group = self.groups[self.gidx]
        if self.first_layer_done[0] < len(group):
            return
        self.first_layer_done[0] = 0
        last_group = self.gidx == len(self.groups) - 1
        targets = list(group) + ([c for c in self.clients if c.layer_id > 1] if last_group else [])
        for c in targets:
            self.send_to_response(c.client_id, self.pause_payload(c))

    def on_update(self, message: dict) -> None:
        layer_id = int(message["layer_id"])
        if not message.get("result", True):
            self.round_result = False
        sd = message.get("parameters")
        last_group = self.gidx == len(self.groups) - 1
        if layer_id == 1 and not last_group:
            self.group_updates.append(sd)
            self.group_sizes.append(message.get("size", 1))
            if len(self.group_updates) == len(self.groups[self.gidx]):
                self.handoff = fedavg_state_dicts(self.group_updates)      # unweighted hand-off (reference)
                self.group_updates, self.group_sizes = [], []
                self.gidx += 1
                self._start_wave(self.groups[self.gidx])
            return
        if sd is not None and self.round_result and not has_nan(sd):
            self.params[0][layer_id - 1].append(sd)
            self.sizes[0][layer_id - 1].append(message.get("size", 1))
        elif sd is not None:
            self.round_result = False
        self.current_clients[layer_id - 1] += 1
        expect = [len(self.groups[-1])] + self.total_clients[1:]
        if self.current_clients == expect:
            self.finish_round()

    def finish_round(self) -> None:
        self.current_clients = [0] * self.num_stages
        metrics = {"round": self.global_round - self.round + 1, "ok": self.round_result,
                   "seconds": time.monotonic() - self._round_t0}
        if self.round_result:
            self.avg_all_parameters(0)
            full = self.concatenate_and_avg_clusters()
            ok = True
            if self.validation and full:
                from ..validation import get_val
                ok, val = get_val(self.model_name, self.data_name, full, self.logger, strict=self.STRICT_VALIDATION,
                                  native=self.cfg.b200.get("native-validation", False),
                                  speech_features=self.cfg.b200.get("speech-features", "engine"))
                metrics.update(val)
            if ok:
                if full and self.save_parameters:
                    save_checkpoint(full, checkpoint_path(self.model_name, self.data_name, self.workdir))
                self.round -= 1
            else:
                self.logger.log_warning("Training failed!")
                self._retries = getattr(self, "_retries", 0) + 1
                if self.STOP_ON_VALIDATION_FAILURE or self._retries > self.MAX_ROUND_RETRIES:
                    self.round = 0                    # other/DCSL/src/Server.py:213 — stop instead of retrying
        else:
            self.round -= 1
        self.history.append(metrics)
        self._reset_round_buffers()
        self.round_result = True
        if self.round > 0:
            self.begin_round()
        else:
            self.notify_clients(start=False)


class VanillaSLServer(SequentialServer):
    ALGORITHM = "vanilla_sl"


class ClusterFSLServer(SequentialServer):
    ALGORITHM = "cluster_fsl"


class DCSLServer(SequentialServer):
    ALGORITHM = "dcsl"
    STOP_ON_VALIDATION_FAILURE = True         # reference DCSL sets round = 0 when validation fails (other/DCSL/src/Server.py:213)

    def extra_start(self, c: ClientInfo) -> dict:
        last = [x.client_id for x in self.clients if x.layer_id == self.num_stages]
        sda = max(len(g) for g in self.groups)
        return {"local_round": self.cfg.local_round, "sda_size": sda, "layer2_devices": last,
                "config_time": self.cfg.limited_time}


class SequentialClient(RpcClient):
    """First stage honours ``limited-time`` / ``local-round`` from START."""

    VARIANT = "vanilla_sl"
    STRICT = False

    def algorithm(self) -> str:
        return self.VARIANT

    def run_stage(self):
        msg = self.start_msg
        t = self.trainer
        if self.is_first and not self.is_last:
            return t.train_on_first_layer(self.learning, self.train_loader, self.cluster,
                                          local_round=int(msg.get("local_round", 1)),
                                          limited_time=msg.get("config_time"), strict=self.STRICT,
                                          targets=self.targets(msg))
        if self.is_last and not self.is_first:
            return t.train_on_last_layer(self.learning, self.cluster, sda_size=self.sda(msg), source=self.source())
        return super().run_stage()

    def targets(self, msg):
        return None

    def sda(self, msg) -> int:
        return 1

    def source(self):
        return None


class VanillaSLClient(SequentialClient):
    VARIANT = "vanilla_sl"


class ClusterFSLClient(SequentialClient):
    VARIANT = "cluster_fsl"


class DCSLClient(SequentialClient):
    VARIANT, STRICT = "dcsl", True

    def targets(self, msg):
        return list(msg.get("layer2_devices") or []) or None

    def sda(self, msg) -> int:
        return max(1, int(msg.get("sda_size", 1)))

    def source(self):
        return self.client_id                   # own queue: intermediate_queue_{device_id}


# =============================================================================== FLEX
class FlexServer(Server):
    ALGORITHM = "flex"

    def label_matrix(self):
        return self.cfg.label_matrix if self.cfg.label_matrix is not None else "flex"

    def cluster_and_selection(self) -> None:
        cfg = self.cfg
        ncl = cfg.num_cluster
        pool = self.label_counts.tolist()
        kept: List[ClientInfo] = []
        for c in self.clients:
            c.cluster = max(c.cluster, 0)
            if c.layer_id == 1:
                lab = pool.pop(0)
                if c.extras.get("select", 1):
                    c.label_counts, c.train = lab, True
                    kept.append(c)
                else:                              # un-selected devices are dropped at registration
                    c.train = False
                    self.total_clients[0] -= 1
            else:
                c.label_counts, c.train = [], True
                kept.append(c)
        clusters = []
        for k in range(ncl):
            members = [[c.client_id for c in kept if c.cluster == k and c.layer_id == s + 1] for s in range(self.num_stages)]
            clusters.append(ClusterPlan(k, list(cfg.cluster_cut_layers[k]), members))
        self.topology = Topology(self.num_stages, clusters)
        self._reset_round_buffers()
        self.flex_round = 1
        self.clients_avg: List[dict] = [{} for _ in range(ncl)]
        self.edge_params: List[dict] = [{} for _ in range(ncl)]
        self.notified = 0

    def distribution(self) -> None:
        super().distribution()
        # FLEX hands labels out in registration order (pop(0)) — redone in cluster_and_selection
        for c in self.clients:
            c.label_counts = []

    def _sends(self):
        return self.flex_round % self.cfg.t_c == 0, self.flex_round % self.cfg.t_g == 0

    def on_notify(self, message: dict) -> None:
        self.notified += 1
        if self.notified < self.total_clients[0]:
            return
        self.notified = 0
        client_send, edge_send = self._sends()
        for c in self.clients:
            if c.train:
                self.send_to_response(c.client_id, M.pause(send=client_send if c.layer_id == 1 else edge_send))

    def start_payload(self, c: ClientInfo) -> dict:
        p = super().start_payload(c)
        p["cut_layer"] = self.topology.clusters[c.cluster].cut_layers[0]
        mode = getattr(self, "_start_mode", "full")
        if mode == "sub_update":
            p["parameters"] = self.clients_avg[c.cluster] if c.layer_id == 1 and self.clients_avg[c.cluster] else None
            p["resident"] = p["parameters"] is None
        elif mode == "sub":
            p["parameters"], p["resident"] = None, True
        return p

    def on_update(self, message: dict) -> None:
        layer_id, cluster = int(message["layer_id"]), int(message.get("cluster") or 0)
        self.current_clients[layer_id - 1] += 1
        if not message.get("result", True):
            self.round_result = False
        sd = message.get("parameters")
        if sd is not None and self.round_result:
            if layer_id == 1:
                self.params[cluster][0].append(sd)
                self.sizes[cluster][0].append(message.get("size", 1))
            else:
                self.edge_params[cluster] = sd
        if self.current_clients != self.total_clients:
            return
        self.current_clients = [0] * self.num_stages
        client_send, edge_send = self._sends()
        metrics = {"round": self.flex_round, "ok": self.round_result, "seconds": time.monotonic() - self._round_t0}
        if self.round_result:
            if client_send:
                for k in range(len(self.topology.clusters)):
                    if self.params[k][0]:
                        self.clients_avg[k] = fedavg_state_dicts(self.params[k][0], self.sizes[k][0])
            if edge_send:
                fulls = []
                for k in range(len(self.topology.clusters)):
                    d = dict(self.clients_avg[k])
                    d.update(self.edge_params[k])
                    if d:
                        fulls.append(d)
                full = fedavg_state_dicts(fulls)
                ok = True
                if self.validation and full:
                    from ..validation import get_val
                    ok, val = get_val(self.model_name, self.data_name, full, self.logger,
                                      native=self.cfg.b200.get("native-validation", False),
                                      speech_features=self.cfg.b200.get("speech-features", "engine"))
                    metrics.update(val)
                if ok and full:
                    save_checkpoint(full, checkpoint_path(self.model_name, self.data_name, self.workdir))
                elif not ok:
                    self.flex_round = self.global_round + 1
            self.flex_round += 1
        else:
            self.flex_round = self.global_round + 1
        self.history.append(metrics)
        self._reset_round_buffers()
        self.round_result = True
        if self.flex_round <= self.global_round:
            cs, es = self.flex_round % self.cfg.t_c == 0, self.flex_round % self.cfg.t_g == 0
            prev_cs, prev_es = client_send, edge_send
            self._start_mode = "full" if prev_es else ("sub_update" if prev_cs else "sub")
            self.begin_round()
        else:
            self.logger.log_info("Stop training !!!")
            self.notify_clients(start=False)


class FlexClient(RpcClient):
    def algorithm(self) -> str:
        return "flex"

    def on_syn(self, msg: dict) -> None:
        if hasattr(self.executor, "reset_epoch"):
            self.executor.reset_epoch()
        if self.is_first and not self.is_last:
            result, size = self.trainer.train_on_first_layer(self.learning, self.train_loader, self.cluster, strict=True)
        else:
            result, size = self.run_stage()
        send = bool((self.trainer.pause_msg or {}).get("send", True))
        self.upload(result, size, send=send)
        self.rounds_done += 1


# =============================================================================== 2LS
class TwoLSServer(Server):
    ALGORITHM = "2ls"

    def label_matrix(self):
        return self.cfg.label_matrix if self.cfg.label_matrix is not None else "2ls"

    def cluster_and_selection(self) -> None:
        cfg = self.cfg
        for c in self.clients:
            c.train = True
            c.extras.setdefault("in_cluster", 0)
            c.extras.setdefault("out_cluster", 0)
        self.out_ids = sorted({c.extras["out_cluster"] for c in self.clients if c.layer_id == 1})
        self.in_ids = sorted({c.extras["in_cluster"] for c in self.clients})
        cut = cfg.cluster_cut_layers[0] if cfg.cluster_cut_layers else cfg.no_cluster_cut_layers
        clusters = []
        for k, in_id in enumerate(self.in_ids):
            members = [[c.client_id for c in self.clients if c.extras["in_cluster"] == in_id and c.layer_id == s + 1]
                       for s in range(self.num_stages)]
            clusters.append(ClusterPlan(k, list(cut), members))
        self.topology = Topology(self.num_stages, clusters)
        for c in self.clients:
            c.cluster = self.in_ids.index(c.extras["in_cluster"])
        self._reset_round_buffers()
        self.global_model: Optional[dict] = None

    # -- out-cluster sequencing ---------------------------------------------------
    def begin_round(self) -> None:
        self._round_t0 = time.monotonic()
        self.logger.log_info(f"Start training round {self.global_round - self.round + 1}")
        self.pending_out = list(self.out_ids)
        random.shuffle(self.pending_out)
        self.global_model = None
        self._start_out_cluster()

    def _active(self) -> List[ClientInfo]:
        return [c for c in self.clients if c.layer_id > 1 or c.extras["out_cluster"] == self.cur_out]

    def _start_out_cluster(self) -> None:
        self.cur_out = self.pending_out.pop(0)
        print_with_color(f"Start out-cluster {self.cur_out}", "yellow")
        act = self._active()
        self.notify_left = {k: sum(1 for c in act if c.layer_id == 1 and c.cluster == k) for k in range(len(self.in_ids))}
        self.update_left = {k: sum(1 for c in act if c.cluster == k) for k in range(len(self.in_ids))}
        self.finished_in: List[int] = []
        self._reset_round_buffers()
        self.ready_pending = {c.client_id for c in act}
        self.wave = act
        for c in act:
            self.send_to_response(c.client_id, self.start_payload(c))

    def start_payload(self, c: ClientInfo) -> dict:
        p = super().start_payload(c)
        p.update({"idx": c.idx if c.idx is not None else c.cluster, "in_cluster_id": c.extras["in_cluster"],
                  "out_cluster_id": c.extras["out_cluster"]})
        if self.global_model is not None:      # continue from the running FedAsync model
            from ..checkpoint import slice_for_stage
            p["parameters"] = slice_for_stage(self.global_model, self.model_name, self.data_name, p["layers"])
        return p

    def on_ready(self, message: dict) -> None:
        self.ready_pending.discard(str(message["client_id"]))
        if not self.ready_pending:
            for c in self.wave:
                self.send_to_response(c.client_id, M.syn())

    def on_notify(self, message: dict) -> None:
        k = int(message.get("cluster") or 0)
        self.notify_left[k] -= 1
        if self.notify_left[k] == 0:
            for c in self._active():
                if c.cluster == k:
                    self.send_to_response(c.client_id, M.pause())

    def on_update(self, message: dict) -> None:
        layer_id, k = int(message["layer_id"]), int(message.get("cluster") or 0)
        if not message.get("result", True):
            self.round_result = False
        sd = message.get("parameters")
        if sd is not None:
            self.params[k][layer_id - 1].append(sd)
            self.sizes[k][layer_id - 1].append(message.get("size", 1))
        self.update_left[k] -= 1
        if self.update_left[k] == 0:
            self.finished_in.append(k)
        active_in = [k2 for k2, n in self.notify_left.items() if k2 in self.finished_in or n == 0]
        if len(self.finished_in) < sum(1 for k2 in range(len(self.in_ids)) if any(c.cluster == k2 for c in self._active())):
            return
        # every in-cluster of this out-cluster reported: FedAvg per in-cluster, FedAsync in completion order
        for num, k2 in enumerate(self.finished_in):
            self.avg_all_parameters(k2)
            full = {}
            for sdict in self.avg_state_dict[k2]:
                full.update(sdict)
            if not full:
                continue
            self.global_model = fedasync_merge(self.global_model, full, 1.0 / (1 + num))
            save_checkpoint(self.global_model, checkpoint_path(self.model_name, self.data_name, self.workdir))
        if self.pending_out:
            self._start_out_cluster()
            return
        metrics = {"round": self.global_round - self.round + 1, "ok": self.round_result,
                   "seconds": time.monotonic() - self._round_t0}
        if self.round_result and self.global_model:
            ok = True
            if self.validation:
                from ..validation import get_val
                ok, val = get_val(self.model_name, self.data_name, self.global_model, self.logger,
                                  native=self.cfg.b200.get("native-validation", False),
                                  speech_features=self.cfg.b200.get("speech-features", "engine"))
                metrics.update(val)
            self.round = self.round - 1 if ok else 0
        else:
            self.round = 0
        self.history.append(metrics)
        self.round_result = True
        if self.round > 0:
            self.begin_round()
        else:
            self.logger.log_info("Stop training !!!")
            self.notify_clients(start=False)


class TwoLSClient(RpcClient):
    def algorithm(self) -> str:
        return "2ls"

    def make_dataplane(self, msg: dict):
        self.idx = msg.get("idx", 0)
        return HostDataPlane(self.channel, self.client_id, self.layer_id, self.cluster, QueueGrammar("2ls"), device=self.device,
                             wire=str(self.opts.get("wire", "host")))

    def run_stage(self):
        t = self.trainer
        if self.is_first and not self.is_last:
            return t.train_on_first_layer(self.learning, self.train_loader, self.cluster, strict=True, targets=[self.idx])
        if self.is_last and not self.is_first:
            return t.train_on_last_layer(self.learning, self.cluster, source=self.idx)
        return super().run_stage()


SERVERS = {"vanilla_sl": VanillaSLServer, "cluster_fsl": ClusterFSLServer, "dcsl": DCSLServer, "flex": FlexServer,
           "2ls": TwoLSServer}
CLIENTS = {"vanilla_sl": VanillaSLClient, "cluster_fsl": ClusterFSLClient, "dcsl": DCSLClient, "flex": FlexClient,
           "2ls": TwoLSClient}
