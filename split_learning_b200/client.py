"""Client FSM (reference L4, src/RpcClient.py:16-146).

START → build the stage (``build_stage``), load weights if given, wrap BERT with LoRA, move
to the device, build the loader (first stage), acknowledge with READY.  SYN → run the stage
loop for this ``layer_id`` then UPDATE with the stage state-dict and the microbatch count.
STOP → leave.  Differences from the reference: middle stages are dispatched to
``train_on_middle_layer`` (the reference sends every ``layer_id != 1`` to the last-layer
loop, SURVEY §3.5); no 0.5 s polling — the reply queue is a blocking get; LoRA comes from
``models.lora`` (``peft`` is not required to import the client).
"""
from __future__ import annotations

import threading
import time
from typing import Optional

import torch

from . import messages as M
from .data import data_loader
from .log import print_with_color
from .models import build_stage
from .models.lora import LoraConfig, apply_lora, merge_lora
from .train import HostDataPlane, QueueGrammar, StageTrainer, make_executor
from .transport import Channel


class RpcClient:
    def __init__(self, client_id, layer_id: int, channel: Channel, device="cpu", b200_opts: Optional[dict] = None,
                 rank: Optional[int] = None, verbose: bool = False):
        self.client_id, self.layer_id, self.channel, self.device = client_id, layer_id, channel, device
        self.opts = dict(b200_opts or {})
        self.rank = rank
        self.verbose = verbose
        self.response = None
        self.model = None
        self.executor = None
        self.trainer: Optional[StageTrainer] = None
        self.train_loader = None
        self.label_count = None
        self.cluster = None
        self.learning = None
        self.model_name = self.data_name = None
        self.num_layers = 2
        self.lora = False
        self.rounds_done = 0
        self.watchdog = float(self.opts.get("watchdog-seconds", 120.0))
        self.heartbeat = float(self.opts.get("heartbeat-seconds", min(10.0, self.watchdog / 4)))
        self._hb_stop = threading.Event()
        self._hb_thread: Optional[threading.Thread] = None
        self._stopped = False
        self.channel.queue_declare(M.reply_queue(client_id))

    # ------------------------------------------------------------------ liveness
    def start_heartbeat(self) -> None:
        """Beacon to the server from a daemon thread (own channel) for as long as this client lives: the server's and the
        peers' idle timers measure silence, not the length of a healthy round (sequential variants wait N epochs)."""
        if self._hb_thread is not None or self.heartbeat <= 0:
            return
        ch = self.channel.clone()

        def beat():
            while not self._hb_stop.wait(self.heartbeat):
                try:
                    ch.publish_obj(M.RPC_QUEUE, M.heartbeat(self.client_id, progress=self.progress()))
                except Exception:
                    return
        self._hb_thread = threading.Thread(target=beat, daemon=True, name=f"slb200-heartbeat-{self.client_id}")
        self._hb_thread.start()

    def progress(self) -> int:
        """Monotonic count of work done by this client: control messages handled + microbatches trained."""
        t = self.trainer
        return int(self.__dict__.get("_handled", 0)) + (int(getattr(t, "data_count", 0)) if t is not None else 0)

    def stop_heartbeat(self) -> None:
        """Also joins the beacon thread: a daemon thread that is still alive when the interpreter finalises is killed with
        ``pthread_exit`` inside whatever native frame it sits in (observed: ``terminate called without an active
        exception`` + SIGABRT at client exit)."""
        self._hb_stop.set()
        t = self._hb_thread
        if t is not None and t is not threading.current_thread():
            t.join(5.0)

    # ------------------------------------------------------------------
    def send_to_server(self, message) -> None:
        self.channel.publish_obj(M.RPC_QUEUE, message)

    def register(self, profile: Optional[dict], cluster: int = -1, **extra) -> None:
        self.send_to_server(M.register(self.client_id, self.layer_id, profile, cluster, rank=self.rank, **extra))
        self.start_heartbeat()

    def wait_response(self, idle_timeout: Optional[float] = None) -> None:
        try:
            self._serve(idle_timeout)
        finally:
            self.stop_heartbeat()

    def _serve(self, idle_timeout: Optional[float]) -> None:
        last = time.monotonic()
        # the server relays a heartbeat every few seconds: its silence for a watchdog period means it is gone
        limit = idle_timeout if idle_timeout is not None else (max(self.watchdog, 3 * self.heartbeat) if self.heartbeat > 0
                                                               else max(4 * self.watchdog, 600.0))
        while True:
            m = self.channel.get_obj(M.reply_queue(self.client_id), 0.25)
            if m is None:
                if time.monotonic() - last > limit:
                    raise TimeoutError(f"client {self.client_id}: server silent for {limit}s")
                continue
            last = time.monotonic()
            if m.get("action") == M.HEARTBEAT:          # the server (and through it every peer) is alive
                continue
            if not self.response_message(m):
                return

    # ------------------------------------------------------------------
    def response_message(self, msg: dict) -> bool:
        self.response = msg
        self._handled = self.__dict__.get("_handled", 0) + 1
        action = msg["action"]
        print_with_color(f"[<<<] Client received: {msg.get('message')}", "blue")
        if action == M.START:
            self.on_start(msg)
            return True
        if action == M.SYN:
            self.on_syn(msg)
            return not self._stopped          # a STOP consumed inside the training loop ends the client too
        if action == M.PAUSE:          # stray PAUSE outside a training loop: ignore
            return True
        if action == M.STOP:
            return False
        return True

    def algorithm(self) -> str:
        return str(self.opts.get("algorithm", "main"))

    def on_start(self, msg: dict) -> None:
        self.model_name, self.data_name = msg["model_name"], msg["data_name"]
        self.learning = msg["learning"]
        self.num_layers = int(msg.get("num_layers", max(self.layer_id, 2)))
        layers = msg["layers"]
        if self.label_count is None or msg.get("label_count"):
            self.label_count = msg.get("label_count")
        if msg.get("cluster") is not None:
            self.cluster = msg["cluster"]
        is_first = self.layer_id == 1
        is_last = self.layer_id == self.num_layers or (layers[1] == 0)
        state_dict = msg.get("parameters")

        keep = self.executor is not None and msg.get("resident") and state_dict is None
        if not keep:
            self.model = build_stage(self.model_name, self.data_name, layers)
            if state_dict:
                self.model.load_state_dict(state_dict)
            self.lora = self.model_name.upper() == "BERT" and self.opts.get("lora", True)
            if self.lora:
                keep_trainable = ("layer15.classifier", "layer27.classifier") if is_last else ()
                apply_lora(self.model, LoraConfig(), keep_trainable)
            self.executor = make_executor(self.model, self.model_name, self.learning, self.device,
                                          is_first, is_last, self.opts)
        dp = self.make_dataplane(msg)
        self.trainer = StageTrainer(self.client_id, self.layer_id, self.channel, self.executor, dp,
                                    watchdog=self.watchdog, verbose=self.verbose)
        self.trainer.data_count = 0
        if is_first and (self.train_loader is None or msg.get("refresh", True)):
            import zlib
            self.train_loader = data_loader(self.data_name, int(self.learning["batch-size"]), self.label_count,
                                            train=True, synthetic=True if self.opts.get("synthetic-data") else None,
                                            seed=zlib.crc32(str(self.client_id).encode()) & 0x7FFFFFFF,   # every client its own samples
                                            device=self.device, gpu_loader=bool(self.opts.get("gpu-loader", False)),
                                            speech_features=self.opts.get("speech-features", "engine"))
        self.is_first, self.is_last = is_first, is_last
        self.start_msg = msg
        self.send_to_server(M.ready(self.client_id, self.layer_id))

    def make_dataplane(self, msg: dict):
        grammar = QueueGrammar(self.algorithm())
        return HostDataPlane(self.channel, self.client_id, self.layer_id, self.cluster, grammar, device=self.device,
                             wire=str(self.opts.get("wire", "host")))

    def run_stage(self):
        t = self.trainer
        if self.is_first and self.is_last:       # cut == 0: whole model on one client
            return self._train_whole_model()
        if self.is_first:
            return t.train_on_first_layer(self.learning, self.train_loader, self.cluster)
        if self.is_last:
            return t.train_on_last_layer(self.learning, self.cluster)
        return t.train_on_middle_layer(self.learning, self.cluster)

    def _train_whole_model(self):
        n = 0
        for batch in self.train_loader:
            x, y = (batch, batch["labels"]) if isinstance(batch, dict) else batch
            self.executor.forward_backward_last(x, torch.as_tensor(y))
            n += 1
        self.send_to_server(M.notify(self.client_id, self.layer_id, self.cluster))
        self.trainer._wait_pause()
        return (not self.executor.nan_detected()), n

    def on_syn(self, msg: dict) -> None:
        if hasattr(self.executor, "reset_epoch"):
            self.executor.reset_epoch()
        result, size = self.run_stage()
        self.upload(result, size)
        self.rounds_done += 1
        pm = getattr(self.trainer, "pause_msg", None)
        if pm is not None and pm.get("action") == M.STOP:
            self._stopped = True

    def upload(self, result: bool, size: int, send: bool = True) -> None:
        sd = None
        if send:
            if self.lora:
                merge_lora(self.model)
            sd = {k: v.detach().to("cpu") for k, v in self.executor.state_dict().items()}
        self.send_to_server(M.update(self.client_id, self.layer_id, result, size, self.cluster, sd))
        print_with_color("[>>>] Client sent parameters to server", "red")
