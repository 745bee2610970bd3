"""Round transports: how client results reach the server optimizer and how the new global
model reaches the clients — the four ``photon.comm_stack`` options.

=========  ================================================================================
``nvl``    PRODUCT PATH. One fused sm_90a kernel per GPU over the symmetric NVLink arena
           (:class:`photon_b200.parallel.fed_round.NvlFedRound`): weighted reduce + server
           optimizer on the GPU's shard + broadcast with bf16 cast. No NCCL, no host.
``ray``    Collective baseline: weighted local sums → ``torch.distributed.all_reduce`` (NCCL on
           GPUs, gloo on CPU) → every rank applies the server optimizer redundantly.  Stands
           in for the reference's Ray-plasma stack (Ray is not installable offline).
``shm``    Reference-equivalent HOST path (ref: photon/server/s3_utils.py:865-903,
           photon/strategy/aggregation.py:57-75): D2H → per-tensor ndarrays → POSIX shm →
           rank-0 streaming mean + server optimizer on the CPU → shm → H2D.
``s3``     Same as ``shm`` but through ``.npz`` objects, layout
           ``{bucket}/{run_uuid}/server/comm_stack/{endpoint}/parameters.npz`` (ref: s3_utils.py:812-864): in an S3
           bucket when an endpoint is configured (own SigV4 REST client, utils/objstore.py — works across hosts),
           in a directory otherwise.
=========  ================================================================================

All share one interface: ``begin_round`` → ``add_client`` × k → ``finish_round`` →
``global_params`` / ``global_shadow`` and produce the same model within fp32 tolerance
(``tests/test_federation_cpu.py::test_transports_agree``; nvl vs ray on GPUs: ``tests/test_multiproc_gpu.py``).
"""
from __future__ import annotations

import os
import time
import uuid
from pathlib import Path
from typing import Any

import numpy as np
import torch
import torch.distributed as dist

from photon_b200.shm.utils import ModelParametersMetadata, get_parameters_shm, set_parameters_shm, unlink_quietly
from photon_b200.strategy.strategies import ServerStrategy
from photon_b200.utils.core import dump_model_parameters_to_file, load_model_parameters_from_file
from photon_b200.utils.flat import FlatLayout


def _dist_on(group: Any = None) -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1


class RoundBackend:
    name = "base"

    def __init__(self, layout: FlatLayout, strategy: ServerStrategy, device: torch.device, *, rank: int = 0,
                 world_size: int = 1, group: Any = None) -> None:
        self.layout, self.strategy, self.device = layout, strategy, device
        self.rank, self.world_size, self.group = rank, world_size, group
        self.last_metrics: dict[str, Any] = {}
        self.timings: dict[str, float] = {}
        # host control plane (photon_b200.server.control): when set, the tiny metadata exchanges of a round go through it instead
        # of torch.distributed collectives, so they keep working (over the survivors) after a rank died
        self.ctl: Any = None

    # -- metadata exchange: control plane when present, torch.distributed otherwise ---------------------------------------
    def _gather_objects(self, tag: str, obj: Any) -> list[Any]:
        """One object per LIVING rank, in rank order."""
        if self.ctl is not None:
            parts = self.ctl.gather(f"rb/{tag}", obj)
            return [parts[r] for r in sorted(parts)]
        if _dist_on(self.group):
            box: list[Any] = [None] * self.world_size
            dist.all_gather_object(box, obj, group=self.group)
            return box
        return [obj]

    def _bcast_object(self, tag: str, obj: Any) -> Any:
        if self.ctl is not None:
            return self.ctl.broadcast(f"rb/{tag}", obj, src=0)
        if _dist_on(self.group):
            box = [obj]
            dist.broadcast_object_list(box, src=0, group=self.group)
            return box[0]
        return obj

    def _barrier(self, tag: str) -> None:
        if self.ctl is not None:
            self.ctl.barrier(f"rb/{tag}")
        elif _dist_on(self.group):
            dist.barrier(group=self.group)

    def _sum_small(self, tag: str, t: torch.Tensor) -> torch.Tensor:
        if self.ctl is not None:
            return self.ctl.sum_tensor(f"rb/{tag}", t)
        if self.world_size > 1 and _dist_on(self.group):
            if dist.get_backend(self.group) != "nccl":
                t = t.cpu()
            dist.all_reduce(t, group=self.group)
        return t

    def status(self) -> int:
        """Non-zero when the last ``finish_round`` could not include every participant (bit mask; nvl only)."""
        return 0

    def set_global(self, params: torch.Tensor, momentum: torch.Tensor | None = None, second: torch.Tensor | None = None) -> None:
        raise NotImplementedError

    def begin_round(self) -> None:
        raise NotImplementedError

    def add_client(self, params: torch.Tensor, weight: float) -> None:
        raise NotImplementedError

    def finish_round(self, server_round: int, alive: list[int] | None = None) -> None:
        """``alive``: the ranks taking part when some died (None = all)."""
        raise NotImplementedError

    def global_params(self) -> torch.Tensor:
        raise NotImplementedError

    def global_shadow(self) -> torch.Tensor | None:
        return None

    def moments(self) -> tuple[torch.Tensor | None, torch.Tensor | None]:
        return self.strategy.momentum_vector, self.strategy.second_momentum_vector

    # -- server metric callback (noise scale): additive per-client statistics, reduced over ranks at collection time
    def _cb_begin(self) -> None:
        self._cb_sq: torch.Tensor | None = None
        self._cb_n = 0

    def _cb_add(self, params: torch.Tensor) -> None:
        if self.strategy.metrics_callback is None:
            return
        d = (self.global_params().to(params.device)[: params.numel()] - params.reshape(-1)).float()
        sq = torch.dot(d, d).double()       # stays on the device: no host sync inside the round
        self._cb_sq = sq if self._cb_sq is None else self._cb_sq + sq
        self._cb_n += 1

    def _pg_sq(self) -> float | None:
        return self.strategy.last_pg_sq

    def collect_metrics(self) -> dict[str, Any]:
        """Server-side metrics of the round that just finished (collective: every rank calls it)."""
        cb = self.strategy.metrics_callback
        if cb is None:
            return self.last_metrics
        stats = torch.zeros(2, dtype=torch.float64, device=self.device)
        if getattr(self, "_cb_sq", None) is not None:
            stats[0], stats[1] = self._cb_sq.to(self.device), float(self._cb_n)
        stats = self._sum_small("cbstats", stats)
        g_big = self._pg_sq()
        if g_big is not None:
            sum_sq, n = stats.tolist()
            cb.round_end_from_stats(float(sum_sq), int(round(n)), float(g_big), self.last_metrics)
        return self.last_metrics

    def close(self) -> None:
        pass


class _HostAccumulating(RoundBackend):
    """Shared piece of the non-NVL backends: keep x on ``device``, accumulate Σ n_k·x_k locally."""

    def set_global(self, params: torch.Tensor, momentum: torch.Tensor | None = None, second: torch.Tensor | None = None) -> None:
        self.strategy.initialize(params.to(self.server_device, torch.float32).clone(),
                                 None if momentum is None else momentum.to(self.server_device).clone(),
                                 None if second is None else second.to(self.server_device).clone(), layout=self.layout)
        self._x_dev = params.to(self.device, torch.float32).clone()

    @property
    def server_device(self) -> torch.device:
        return self.device

    def begin_round(self) -> None:
        self._acc: torch.Tensor | None = None
        self._w = 0.0
        self._kept: list[tuple[torch.Tensor, float]] = []
        self._cb_begin()

    def add_client(self, params: torch.Tensor, weight: float) -> None:
        if weight <= 0:
            raise ValueError("client weight must be positive")
        self._cb_add(params)
        if self.strategy.track_inplace:   # debug self-check: keep every client to form the textbook mean later
            self._kept.append((params.detach().to("cpu", torch.float64), float(weight)))
        if self._acc is None:
            self._acc = params.detach().to(self.device, torch.float32) * float(weight)
        else:
            self._acc.add_(params.to(self.device, torch.float32), alpha=float(weight))
        self._w += float(weight)

    def global_params(self) -> torch.Tensor:
        return self._x_dev

    def _fedavg_gap(self, avg: torch.Tensor | None, scale: float) -> dict[str, float]:
        """``server/l2_norm_fedavg_gap``: distance between the transport's aggregate and the textbook float64
        Σ n_k x_k / Σ n_k over ALL clients of the round (ref: fedavg_eff.py:366-391). Collective — every rank calls
        it at the same point of ``finish_round``; ranks that do not hold ``avg`` pass None."""
        if not self.strategy.track_inplace:
            return {}
        num = torch.zeros(self.layout.total, dtype=torch.float64)
        den = torch.zeros(1, dtype=torch.float64)
        for x, w in self._kept:
            num += x * w
            den += w
        if self.world_size > 1 and _dist_on(self.group):
            nccl = dist.get_backend(self.group) == "nccl"
            num, den = (num.to(self.device), den.to(self.device)) if nccl else (num, den)
            dist.all_reduce(num, group=self.group)
            dist.all_reduce(den, group=self.group)
        self._kept = []
        if avg is None or float(den) <= 0:
            return {}
        naive = (num / den).to("cpu") * scale
        return {"server/l2_norm_fedavg_gap": float((naive - avg.detach().to("cpu", torch.float64)).norm())}


class CollectiveRoundBackend(_HostAccumulating):
    """``comm_stack.ray`` slot: all-reduce of the weighted sums, redundant server update."""

    name = "ray"

    def finish_round(self, server_round: int, alive: list[int] | None = None) -> None:
        if alive is not None and len(alive) < self.world_size:
            raise RuntimeError("comm_stack.ray all-reduces over the job's process group and cannot leave a dead rank out; "
                               "use comm_stack.nvl (GPU) or comm_stack.shm (host) for fault-tolerant rounds")
        t0 = time.perf_counter()
        acc = self._acc if self._acc is not None else torch.zeros(self.layout.total, device=self.device)
        w = torch.tensor([self._w], dtype=torch.float64, device=acc.device if _dist_on(self.group) and dist.get_backend(self.group) == "nccl" else "cpu")
        if _dist_on(self.group):
            dist.all_reduce(acc, group=self.group)
            dist.all_reduce(w, group=self.group)
        total = float(w.item())
        if total <= 0:
            self.last_metrics = {}
            return
        avg = acc / total
        s = self.strategy.scaling_factor()
        if s != 1.0:
            avg.mul_(s)
        gap = self._fedavg_gap(avg, s)
        self.last_metrics = {**self.strategy.apply_server_update(avg, server_round), **gap}
        self._x_dev = self.strategy.parameters
        self.timings["aggregate_broadcast_s"] = time.perf_counter() - t0


class ShmRoundBackend(_HostAccumulating):
    """``comm_stack.shm``: the reference's host path, faithfully (D2H per tensor, shm, NumPy-era
    streaming mean on rank 0's CPU, shm back, H2D per tensor)."""

    name = "shm"

    def __init__(self, *a: Any, run_uuid: str = "run", **kw: Any) -> None:
        super().__init__(*a, **kw)
        self.uid = f"{run_uuid}-{uuid.uuid4().hex[:8]}" if self.rank == 0 else ""
        if _dist_on(self.group):
            box = [self.uid]
            dist.broadcast_object_list(box, src=0, group=self.group)
            self.uid = box[0]
        self._handles: list[Any] = []
        self._n = 0

    @property
    def server_device(self) -> torch.device:
        return torch.device("cpu")  # the reference's server never touches a GPU

    def _put(self, name: str, flat: torch.Tensor) -> ModelParametersMetadata:
        arrays = self.layout.to_ndarrays(flat)  # D2H + per-tensor split (ref: photon/utils.py:243-244)
        shm, meta = set_parameters_shm(name, arrays)
        self._handles.append(shm)
        return meta

    def _get(self, name: str, meta: ModelParametersMetadata) -> list[np.ndarray]:
        shm, views = get_parameters_shm(name, meta, copy=True)
        shm.close()
        return views

    def finish_round(self, server_round: int, alive: list[int] | None = None) -> None:
        t0 = time.perf_counter()
        self._n += 1
        up = f"{self.uid}_r{self.rank}_up"
        have = self._acc is not None and self._w > 0
        meta = self._put(up, self._acc / self._w) if have else None
        mine = (up, meta.to_literal() if meta else None, self._w)
        infos = self._gather_objects(f"shm_up/{self._n}", mine)     # only the living ranks answer (parameters travel through POSIX shm)
        down = f"{self.uid}_down"
        down_meta: list[Any] = [None]
        agg: torch.Tensor | None = None
        agg_scale = 1.0
        if self.rank == 0:
            from photon_b200.strategy.aggregation import StreamingMean

            sm = StreamingMean()
            for name, lit, w in infos:
                if lit is None or w <= 0:
                    continue
                arrays = self._get(name, ModelParametersMetadata.from_literal(lit))
                host = torch.zeros(self.layout.total)
                self.layout.from_ndarrays(host, arrays)
                sm.add(host, w)
            if sm.result() is not None:
                avg = sm.result()
                s = self.strategy.scaling_factor()
                if s != 1.0:
                    avg.mul_(s)
                agg, agg_scale = avg.clone() if self.strategy.track_inplace else None, s
                self.last_metrics = self.strategy.apply_server_update(avg, server_round)
            down_meta[0] = self._put(down, self.strategy.parameters).to_literal()
        gap = self._fedavg_gap(agg, agg_scale)
        if gap:
            self.last_metrics = {**self.last_metrics, **gap}
        down_meta[0] = self._bcast_object(f"shm_down/{self._n}", down_meta[0])
        arrays = self._get(down, ModelParametersMetadata.from_literal(down_meta[0]))
        host = torch.zeros(self.layout.total)
        self.layout.from_ndarrays(host, arrays)
        self._x_dev = host.to(self.device)  # H2D
        self._barrier(f"shm_done/{self._n}")
        for h in self._handles:
            h.close()
        self._handles = []
        unlink_quietly(up)
        if self.rank == 0:
            unlink_quietly(down)
        self.timings["aggregate_broadcast_s"] = time.perf_counter() - t0


class FileRoundBackend(_HostAccumulating):
    """``comm_stack.s3``: npz objects under ``{bucket}/{run_uuid}/server/comm_stack/…`` (ref: photon/server/s3_utils.py:812-864).
    With ``remote`` (an :class:`photon_b200.utils.objstore.ObjectStore`, i.e. a configured S3 endpoint) every object travels
    through the store — ranks on different hosts need no shared file system; without it the bucket is a directory."""

    name = "s3"

    def __init__(self, *a: Any, root: str | os.PathLike = "./checkpoints", run_uuid: str = "run", num_attempts: int = 3,
                 remote: Any = None, **kw: Any) -> None:
        super().__init__(*a, **kw)
        self.bucket_dir = Path(root)
        self.dir = self.bucket_dir / run_uuid / "server" / "comm_stack"
        self.dir.mkdir(parents=True, exist_ok=True)
        self.num_attempts = int(num_attempts)
        self.remote = remote

    def _publish(self, path: Path) -> None:
        if self.remote is not None:
            self.remote.upload(path.relative_to(self.bucket_dir).as_posix(), path)

    def _fetch(self, path: Path, mine: bool = False) -> Path:
        """Make ``path`` local: objects written by OTHER ranks always come from the store (a stale local copy must not win)."""
        if self.remote is not None and not mine:
            self.remote.download(path.relative_to(self.bucket_dir).as_posix(), path)
        return path

    @property
    def server_device(self) -> torch.device:
        return torch.device("cpu")

    def _load(self, path: Path) -> list[np.ndarray]:
        for attempt in range(self.num_attempts):
            try:
                return load_model_parameters_from_file(path)
            except (OSError, ValueError):
                time.sleep(0.05 * (attempt + 1))
        return load_model_parameters_from_file(path)

    def finish_round(self, server_round: int, alive: list[int] | None = None) -> None:
        t0 = time.perf_counter()
        have = self._acc is not None and self._w > 0
        mine = self.dir / f"client-rank{self.rank}" / "parameters.npz"
        if have:
            dump_model_parameters_to_file(mine, self.layout.to_ndarrays(self._acc / self._w))
            self._publish(mine)
        self._n = getattr(self, "_n", 0) + 1
        rec = (str(mine) if have else None, self._w)
        infos = self._gather_objects(f"s3_up/{self._n}", rec)
        down = self.dir / "server" / "parameters.npz"
        agg: torch.Tensor | None = None
        agg_scale = 1.0
        if self.rank == 0:
            from photon_b200.strategy.aggregation import StreamingMean

            sm = StreamingMean()
            for path, w in infos:
                if path is None or w <= 0:
                    continue
                host = torch.zeros(self.layout.total)
                self.layout.from_ndarrays(host, self._load(self._fetch(Path(path), mine=(Path(path) == mine))))
                sm.add(host, w)
            if sm.result() is not None:
                avg = sm.result()
                s = self.strategy.scaling_factor()
                if s != 1.0:
                    avg.mul_(s)
                agg, agg_scale = avg.clone() if self.strategy.track_inplace else None, s
                self.last_metrics = self.strategy.apply_server_update(avg, server_round)
            dump_model_parameters_to_file(down, self.layout.to_ndarrays(self.strategy.parameters))
            self._publish(down)
        gap = self._fedavg_gap(agg, agg_scale)
        if gap:
            self.last_metrics = {**self.last_metrics, **gap}
        self._barrier(f"s3_written/{self._n}")
        host = torch.zeros(self.layout.total)
        self.layout.from_ndarrays(host, self._load(self._fetch(down, mine=(self.rank == 0))))
        self._x_dev = host.to(self.device)
        self._barrier(f"s3_read/{self._n}")
        self.timings["aggregate_broadcast_s"] = time.perf_counter() - t0


class NvlRoundBackend(RoundBackend):
    """``comm_stack.nvl``: the fused NVLink kernel (see :mod:`photon_b200.parallel.fed_round`)."""

    name = "nvl"

    def __init__(self, layout: FlatLayout, strategy: ServerStrategy, device: torch.device, *, rank: int = 0,
                 world_size: int = 1, group: Any = None, track_norms: bool = True) -> None:
        super().__init__(layout, strategy, device, rank=rank, world_size=world_size, group=group)
        from photon_b200.parallel.fed_round import NvlFedRound

        self.fed = NvlFedRound(layout.total, strategy, rank=rank, world_size=world_size, device=device, group=group, layout=layout)
        self.track_norms = track_norms
        if strategy.track_inplace and rank == 0:
            print("[round/nvl] track_inplace_aggregation is a host-transport self-check; the fused kernel never materialises "
                  "the aggregate, so server/l2_norm_fedavg_gap is not reported on comm_stack.nvl")

    def set_global(self, params: torch.Tensor, momentum: torch.Tensor | None = None, second: torch.Tensor | None = None) -> None:
        self.fed.set_global(params)
        self.fed.set_moments(momentum, second)
        # keep the strategy object's state pointing at the device planes (checkpointing reads them)
        self.strategy.parameters = self.fed.global_params()
        self.strategy.layout = self.layout
        # the strategy object only keeps this rank's slices; `moments()` below stitches the full state for checkpoints
        m, v = self.fed.moments()
        self.strategy.momentum_vector, self.strategy.second_momentum_vector = m, v

    def begin_round(self) -> None:
        self.fed.begin_round()
        self._cb_begin()

    def add_client(self, params: torch.Tensor, weight: float) -> None:
        self._cb_add(params)
        self.fed.add_client(params, weight)

    def finish_round(self, server_round: int, alive: list[int] | None = None) -> None:
        self.fed.finish_round(server_round, alive=alive)
        self.last_metrics = {}

    def status(self) -> int:
        """Sticky status of the round kernel (synchronises): 0 = every participant took part; bit t = participant t (index into the
        ``alive`` list of the launch) missed the start barrier -> the kernel ABORTED and nothing was modified; bit 8+t = left mid-kernel."""
        st = self.fed.check_status()
        if st:
            self.fed.clear_status()
        return st

    def _pg_sq(self) -> float | None:
        n = self.last_metrics.get("server/l2_norm_pseudo_gradient")
        return None if n is None else float(n) ** 2

    def collect_metrics(self) -> dict[str, Any]:
        """Norm by-products of the last round's kernel (+ the noise-scale estimate): a tiny host read, done after
        the round's device work instead of inside it."""
        if self.track_norms or self.strategy.metrics_callback is not None:
            self.last_metrics = self.fed.round_norms(self.group, ctl=self.ctl)
        return super().collect_metrics()

    def global_params(self) -> torch.Tensor:
        return self.fed.global_params()

    def global_shadow(self) -> torch.Tensor | None:
        return self.fed.global_shadow()

    def moments(self) -> tuple[torch.Tensor | None, torch.Tensor | None]:
        """Full-length server moments. Each rank only maintains its shard, so the shards are
        stitched with one all-reduce of zero-padded copies (checkpoint path, not the hot path)."""
        out = []
        degraded = self.ctl is not None and bool(self.ctl.dead)
        for j, full in enumerate(self.fed.full_moments()):
            if full is not None and degraded:      # survivors only, through the host control plane (adopted shards included)
                full = self.fed.add_orphans(full, j)
                parts = self.ctl.gather(f"rb/moments/{j}", full.cpu())
                full = sum(parts[r] for r in sorted(parts)).to(self.device)
            elif full is not None and self.world_size > 1 and _dist_on(self.group):
                dist.all_reduce(full, group=self.group)
            out.append(full)
        return out[0], out[1]

    def close(self) -> None:
        self.fed.close()


def build_round_backend(cfg: Any, layout: FlatLayout, strategy: ServerStrategy, device: torch.device, *, rank: int = 0,
                        world_size: int = 1, group: Any = None) -> RoundBackend:
    cs = dict(cfg["photon"]["comm_stack"])
    active = next((k for k in ("nvl", "shm", "ray", "s3") if cs.get(k)), "shm")
    common = dict(rank=rank, world_size=world_size, group=group)
    if active == "nvl":
        if device.type != "cuda":
            raise RuntimeError("photon.comm_stack.nvl needs CUDA devices; use shm/ray on CPU")
        return NvlRoundBackend(layout, strategy, device, **common)
    if active == "ray":
        return CollectiveRoundBackend(layout, strategy, device, **common)
    if active == "s3":
        root = cfg["photon"].get("saving_path") or os.environ.get("PHOTON_SAVE_PATH", ".")
        from photon_b200.utils.objstore import remote_store_from_cfg

        return FileRoundBackend(layout, strategy, device, root=Path(root) / str(cfg["s3_comm_config"]["bucket_name"]),
                                run_uuid=str(cfg["run_uuid"]), num_attempts=int(cfg["s3_comm_config"].get("num_attempts", 3)),
                                remote=remote_store_from_cfg(cfg), **common)
    return ShmRoundBackend(layout, strategy, device, run_uuid=str(cfg["run_uuid"]), **common)
