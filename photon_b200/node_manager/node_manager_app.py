"""Node manager: the per-box scheduler between the federation control plane and the workers
(ref: photon/node_manager/node_manager_app.py:163-725).

* owns the ``task_queue`` / ``result_queue`` pair and one :class:`Worker` process per device
  (``spawn`` start method);
* publishes the round's parameters once in ``{nm_uuid}_nm_par_shm`` — workers map it zero-copy;
* ``fit`` / ``eval``: clients of the node run SEQUENTIALLY, every worker collaborating (DDP) on the
  current client; the per-client config travels pickled in ``{nm_uuid}_nm_cnf_shm`` together with
  the MASTER_PORT of the node-local process group;
* supervision: dead workers are restarted before each client; a failed task (``n_samples == -1`` or a
  worker dying while we poll) re-queues the client and rebuilds the pool — bounded by ``max_retries``
  (the reference retries forever, SURVEY §5.3);
* ``refresh_workers`` recycles the pool every ``photon.refresh_period`` rounds.

This is the host (shm) topology kept for parity and CPU runs; on a H100 box the SPMD
:class:`photon_b200.federation.FederationRuntime` is the primary path.
"""
from __future__ import annotations

import multiprocessing as mp
import queue
import time
import uuid
from typing import Any, Sequence

import numpy as np

from photon_b200.config.composer import to_container
from photon_b200.messages import Code, EvaluateRes, FitRes, ParamHandle, Status
from photon_b200.shm import constants as C
from photon_b200.shm.utils import (ModelParametersMetadata, close_all_shms, get_dict_shm, get_eval_loss_shm, get_n_samples_shm,
                                   get_parameters_shm, set_dict_shm, set_parameters_shm, unlink_quietly)
from photon_b200.strategy.aggregation import weighted_average, weighted_loss_avg
from photon_b200.utils.core import get_n_cuda_devices
from photon_b200.worker.utils import get_free_tcp_port
from photon_b200.worker.worker import Worker


class NodeManagerApp:
    def __init__(self, cfg: Any, n_workers: int | None = None, nm_uuid: str | None = None, max_retries: int = 2,
                 poll_s: float = 0.1, devices: list[int] | None = None) -> None:
        """``devices``: the GPUs this node owns (default: every visible one — the reference gives each node process its
        own ``CUDA_VISIBLE_DEVICES``); one worker per device."""
        self.cfg_dict = to_container(cfg)
        self.nm_uuid = nm_uuid or f"nm-{uuid.uuid4().hex[:10]}"
        n_gpu = get_n_cuda_devices()
        self.devices = list(devices) if devices else (list(range(n_gpu)) if n_gpu else None)
        n_gpu = len(self.devices) if self.devices else 0
        self.n_workers = int(n_workers or max(1, n_gpu))
        self.max_retries, self.poll_s = int(max_retries), float(poll_s)
        # a worker that neither answers nor dies (a wedged collective, a stuck filesystem) is treated like a dead one after
        # ``photon.task_timeout_s``: the pool is torn down, respawned and the client retried. null = wait forever (reference).
        tmo = (self.cfg_dict.get("photon") or {}).get("task_timeout_s")
        self.task_timeout_s = float(tmo) if tmo else None
        ctx = mp.get_context("spawn")
        self.task_queue: Any = ctx.Queue()
        self.result_queue: Any = ctx.Queue()
        self.workers: list[Worker] = []
        self._param_shm: Any = None
        self._meta: ModelParametersMetadata | None = None
        self.node_training_time_s = 0.0

    # ------------------------------------------------------------------- worker pool
    def create_and_start_workers(self) -> None:
        for r in range(self.n_workers):
            w = Worker(self.cfg_dict, self.nm_uuid, r, self.n_workers, self.task_queue, self.result_queue, self.devices)
            w.start()
            self.workers.append(w)

    def check_workers_health(self) -> None:
        if len(self.workers) != self.n_workers or any(not w.is_alive() for w in self.workers):
            self.close_workers()
            self.create_and_start_workers()

    def close_workers(self) -> None:
        for _ in self.workers:
            self.task_queue.put(None)
        t0 = time.time()
        for w in self.workers:
            w.join(timeout=max(0.1, 5 - (time.time() - t0)))
        for w in self.workers:
            if w.is_alive():
                w.terminate()
                w.join(timeout=2)
            close_all_shms(w.worker_uuid)
            unlink_quietly(w.worker_uuid + C.W_PARAMS_SHM + "_meta")
        self.workers = []
        for q in (self.task_queue, self.result_queue):   # drop stale items of a torn-down pool
            try:
                while True:
                    q.get_nowait()
            except queue.Empty:
                pass

    def refresh_workers(self) -> None:
        self.close_workers()
        self.create_and_start_workers()

    # ---------------------------------------------------------------------- parameters
    def set_parameters(self, arrays: Sequence[np.ndarray]) -> None:
        """Broadcast sink: publish the global model for this node's workers (ref: client_app.py:78-118)."""
        name = self.nm_uuid + C.NM_PARAMS_SHM
        self._param_shm, self._meta = set_parameters_shm(name, arrays, self._meta if self._meta and self._meta.same_layout(
            ModelParametersMetadata.from_ndarrays(arrays)) else None)
        set_dict_shm(name + "_meta", self._meta.to_literal())

    # ----------------------------------------------------------------------------- tasks
    def _run_client(self, cid: int, kind: str, task_cfg: dict[str, Any]) -> tuple[Any, str | None]:
        """One client on the whole pool; returns (rank-0 result message | None, error)."""
        self.check_workers_health()
        task_cfg = dict(task_cfg, MASTER_PORT=get_free_tcp_port(), run_uuid=self.cfg_dict.get("run_uuid"))
        set_dict_shm(self.nm_uuid + C.NM_CONFIG_SHM, {str(cid): task_cfg})
        for _ in self.workers:
            self.task_queue.put((cid, kind))
        got: list[Any] = []
        t0 = time.time()
        while len(got) < self.n_workers:
            try:
                msg = self.result_queue.get(timeout=self.poll_s)
            except queue.Empty:
                if any(not w.is_alive() for w in self.workers):
                    return None, "a worker died while running the task"
                if self.task_timeout_s is not None and time.time() - t0 > self.task_timeout_s:
                    return None, f"no result after {self.task_timeout_s:.0f}s (photon.task_timeout_s): workers presumed hung"
                continue
            if msg.n_samples < 0:
                return None, msg.error or "worker reported failure"
            got.append(msg)
        rank0 = next(m for m in got if m.worker_uuid == self.workers[0].worker_uuid)
        return rank0, None

    def _with_retries(self, cid: int, kind: str, task_cfg: dict[str, Any]) -> tuple[Any, str | None]:
        err: str | None = None
        for attempt in range(self.max_retries + 1):
            msg, err = self._run_client(cid, kind, task_cfg if attempt == 0 else {k: v for k, v in task_cfg.items() if k not in ("inject_failure", "inject_hang")})
            if msg is not None:
                return msg, None
            self.close_workers()   # soft close then terminate; next attempt respawns (ref: node_manager_app.py:553-579)
        return None, err

    def collaborative_fit(self, cid: int, task_cfg: dict[str, Any]) -> tuple[Any, str | None]:
        """ALL workers of the node train ONE client together (one DDP / ZeRO group); on failure the client is
        re-queued after the pool is torn down and respawned (ref: node_manager_app.py:405-592)."""
        return self._with_retries(int(cid), "fit", task_cfg)

    def fit(self, configs: dict[int, dict[str, Any]]) -> list[FitRes]:
        """``configs``: cid → {"fit_config": wire dict, ...}. Clients run sequentially."""
        t0 = time.time()
        out: list[FitRes] = []
        for cid, task_cfg in configs.items():
            msg, err = self.collaborative_fit(int(cid), task_cfg)
            if msg is None:
                out.append(FitRes(Status(Code.FAILED, err or "failed"), None, 0, {}, int(cid)))
                continue
            wu = msg.worker_uuid
            meta = ModelParametersMetadata.from_literal(get_dict_shm(wu + C.W_PARAMS_SHM + "_meta"))
            shm, views = get_parameters_shm(wu + C.W_PARAMS_SHM, meta, copy=True)   # own the data before the worker reuses it
            shm.close()
            metrics = dict(get_dict_shm(wu + C.W_METRICS_SHM))
            metrics["node_training_time_s"] = msg.delta
            out.append(FitRes(Status(Code.OK, ""), ParamHandle("inline", views), get_n_samples_shm(wu), metrics, int(cid)))
        self.node_training_time_s = time.time() - t0
        return out

    def eval(self, configs: dict[int, dict[str, Any]]) -> EvaluateRes:
        """Evaluate the listed clients and fold them into ONE node-level result (ref: :594-725)."""
        t0 = time.time()
        per: list[tuple[int, float, dict[str, Any]]] = []
        for cid, task_cfg in configs.items():
            msg, err = self._with_retries(int(cid), "evaluate", task_cfg)
            if msg is None:
                return EvaluateRes(Status(Code.FAILED, err or "failed"), 0.0, 0, {}, int(cid))
            wu = msg.worker_uuid
            per.append((get_n_samples_shm(wu), get_eval_loss_shm(wu), dict(get_dict_shm(wu + C.W_METRICS_SHM))))
        n = sum(p[0] for p in per)
        metrics = weighted_average([(p[0], p[2]) for p in per])
        metrics["node_eval_time_s"] = time.time() - t0
        return EvaluateRes(Status(Code.OK, ""), weighted_loss_avg([(p[0], p[1]) for p in per]), n, metrics)

    def close(self) -> None:
        self.close_workers()
        if self._param_shm is not None:
            self._param_shm.close()
        for suffix in (C.NM_PARAMS_SHM, C.NM_PARAMS_SHM + "_meta", C.NM_CONFIG_SHM):
            unlink_quietly(self.nm_uuid + suffix)
