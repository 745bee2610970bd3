"""N1 — DDP gradient all-reduce as one fused NVLink kernel on the flat gradient bucket.

The reference's Composer ``FORCED_SYNC`` issues one NCCL all-reduce per parameter
(148 for MPT-125M) after the last microbatch, un-overlapped (ref:
photon/clients/trainer_utils.py:1714; SURVEY §2.5 (b) N1).  Here every rank's flat
gradient buffer is a plane of a :class:`SymmArena`; ``all_reduce_mean_`` launches
``ddp_allreduce_kernel`` (reduce-scatter + all-gather in one pass over peer
pointers, mean folded in, squared-norm partials for clipping as a by-product).
``NvlZeroComm`` goes one step further (ZeRO-style): reduce-scatter, clipping, the local optimizer on the rank's
shard and the all-gather of the new parameters in one kernel.  ``NcclGradComm`` is the stock-collective baseline
with the same interface.
"""
from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist

from photon_b200 import ops
from photon_b200.parallel.symm import SymmArena


class NvlGradComm:
    def __init__(self, total: int, *, rank: int, world_size: int, device: torch.device | int | None = None, group: Any = None) -> None:
        self.total = int(total)
        self.arena = SymmArena({"grads": (total, torch.float32)}, rank=rank, world_size=world_size, device=device, group=group)
        self.norm = torch.zeros(1, dtype=torch.float32, device=torch.device("cuda", self.arena.devices[0]))

    @property
    def grads(self) -> torch.Tensor:
        """The local gradient plane — pass as ``grads_storage`` to :class:`FlatParams`."""
        return self.arena.plane("grads")

    def all_reduce_mean_(self, g: torch.Tensor) -> torch.Tensor:
        ar = self.arena
        if g.data_ptr() != ar.ptrs("grads")[ar.rank]:
            raise ValueError("NvlGradComm reduces its own arena plane; build FlatParams with grads_storage=comm.grads")
        lo, hi = ar.shard(self.total)
        ops.ext().ddp_allreduce(ar.ctl_ptrs(), ar.rank, ar.devices[0], ar.next_epoch(), ar.ptrs("grads"), lo, hi, self.norm,
                                ar.mc_ptr("grads"))
        return g

    def last_grad_norm(self) -> torch.Tensor:
        """‖mean gradient‖₂ of the last all-reduce (device scalar)."""
        return self.norm[0]

    def close(self) -> None:
        self.arena.close()


class NvlZeroComm:
    """N1 + K11 + K12 in ONE NVLink kernel (the in-client replacement for FSDP's reduce-scatter → sharded optimizer →
    all-gather, ref: photon/conf/llm_config/mpt-125m.yaml:85-91): every rank reduces its shard of all gradient planes,
    the shard norms meet in the control pages, the clip coefficient is formed on device, the local optimizer runs on the
    rank's shard of (p, m, v) and the new fp32 masters + bf16 compute copies are stored into every rank's planes.
    Gradient, master and bf16 planes live in a :class:`SymmArena`; pass them to the backend as storages."""

    fused_step = True

    def __init__(self, total: int, *, rank: int, world_size: int, device: torch.device | int | None = None, group: Any = None) -> None:
        self.total = int(total)
        self.arena = SymmArena({"grads": (total, torch.float32), "params": (total, torch.float32), "shadow": (total, torch.bfloat16)},
                               rank=rank, world_size=world_size, device=device, group=group)
        self.norm = torch.zeros(1, dtype=torch.float32, device=torch.device("cuda", self.arena.devices[0]))

    @property
    def grads(self) -> torch.Tensor:
        return self.arena.plane("grads")

    @property
    def params(self) -> torch.Tensor:
        return self.arena.plane("params")

    @property
    def shadow(self) -> torch.Tensor:
        return self.arena.plane("shadow")

    def shard(self) -> tuple[int, int]:
        return self.arena.shard(self.total)

    def shard_bounds(self) -> list[tuple[int, int]]:
        return [self.arena.shard(self.total, r) for r in range(self.arena.world_size)]

    def step(self, opt: Any, lr: float, max_norm: float | None, inv_scale: float = 1.0) -> torch.Tensor:
        """One fused training step tail; returns ‖mean gradient‖₂ (device scalar, before clipping)."""
        ar = self.arena
        lo, hi = self.shard()
        if opt.shard != (lo, hi):
            raise ValueError(f"optimizer shard {opt.shard} != arena shard {(lo, hi)}: build it with shard=comm.shard()")
        if opt.flat.params.data_ptr() != ar.ptrs("params")[ar.rank] or opt.flat.grads.data_ptr() != ar.ptrs("grads")[ar.rank]:
            raise ValueError("NvlZeroComm steps its own arena planes; build the backend with its params/grads/shadow storages")
        h = ops.optimizer_hyper(opt, lr)
        shadow = ar.ptrs("shadow") if opt.bf16_shadow is not None else []
        ops.ext().ddp_zero_step(ar.ctl_ptrs(), ar.rank, ar.devices[0], ar.next_epoch(), ar.ptrs("grads"), ar.ptrs("params"), shadow,
                                opt.exp_avg, opt.exp_avg_sq, lo, hi, h["kind"], h["first"], h["lr"], h["beta1"], h["beta2"], h["eps"],
                                h["decay"], h["clip"], h["step_size"], h["inv_sqrt_bc2"],
                                float(max_norm) if max_norm is not None else -1.0, float(inv_scale), self.norm,
                                ar.mc_ptr("grads"), ar.mc_ptr("params"), ar.mc_ptr("shadow"), wd=h["wd"])
        opt.lr = float(lr)
        opt.step_count += 1
        return self.norm[0]

    def all_reduce_mean_(self, g: torch.Tensor) -> torch.Tensor:   # not used on the fused path
        raise RuntimeError("NvlZeroComm fuses the reduction into step(); use NvlGradComm for a bare all-reduce")

    def close(self) -> None:
        self.arena.close()


class NcclGradComm:
    """Baseline: ONE NCCL all-reduce on the flat bucket (already better than the reference's 148)."""

    def __init__(self, group: Any = None) -> None:
        self.group = group

    def all_reduce_mean_(self, g: torch.Tensor) -> torch.Tensor:
        dist.all_reduce(g, group=self.group)
        return g.div_(dist.get_world_size(self.group))

    def close(self) -> None:
        pass


class NcclPerTensorGradComm:
    """The reference's pattern, for baselines: Composer ``DDPSyncStrategy.FORCED_SYNC`` issues one NCCL all-reduce per
    parameter tensor after the last microbatch, un-overlapped, then divides by the world size
    (ref: photon/clients/trainer_utils.py:1714; 148 messages for MPT-125M, the largest 154.7 MB)."""

    def __init__(self, group: Any = None) -> None:
        self.group, self.layout = group, None

    def bind_layout(self, layout: Any) -> None:
        self.layout = layout

    def all_reduce_mean_(self, g: torch.Tensor) -> torch.Tensor:
        if self.layout is None:
            raise RuntimeError("NcclPerTensorGradComm needs bind_layout(flat layout) before the first all-reduce")
        w = dist.get_world_size(self.group)
        for i in range(len(self.layout.names)):
            t = self.layout.view(g, i)
            dist.all_reduce(t, group=self.group)
            t.div_(w)
        return g

    def close(self) -> None:
        pass


def wants_sharded_step(llm_cfg: Any) -> bool:
    """``fsdp_config`` present with a sharding strategy other than NO_SHARD (the reference's YAML default)."""
    fsdp = (llm_cfg or {}).get("fsdp_config") or None
    return bool(fsdp) and str(dict(fsdp).get("sharding_strategy", "FULL_SHARD")).upper() != "NO_SHARD"


def wants_full_sharding(cfg: Any, n_params: int, device: Any = None) -> bool:
    """``kernels.param_sharding``: ``zero3`` / ``zero1`` force a scheme; ``auto`` (default) shards parameters and gradients too
    (ZeRO-3, :mod:`photon_b200.parallel.zero3`) when ``fsdp_config.sharding_strategy`` is FULL_SHARD AND the replicated training
    state (18 B/param) would take more than 40 % of the GPU — on an 80 GB H100 that is MPT-3B and MPT-7B, not MPT-125M / 1B, for
    which the fused ZeRO-1 step (one kernel, CUDA-graphed microbatches) is faster and memory is not a concern. Without a CUDA
    device the capacity of an 80 GB H100 is assumed."""
    llm = cfg["llm_config"]
    mode = str((cfg.get("kernels") or {}).get("param_sharding", "auto") or "auto").lower()
    if mode in ("zero3", "full", "full_shard"):
        return True
    fsdp = (llm or {}).get("fsdp_config") or None
    if mode != "auto" or not fsdp or str(dict(fsdp).get("sharding_strategy", "FULL_SHARD")).upper() != "FULL_SHARD":
        return False
    cap = 80 * 2**30
    try:
        import torch as _t

        if device is not None and _t.device(device).type == "cuda" and _t.cuda.is_available():
            cap = _t.cuda.get_device_properties(device).total_memory
    except Exception:  # noqa: BLE001
        pass
    return 18 * int(n_params) > 0.4 * cap


def build_nvl_comm(total: int, *, sharded: bool, rank: int, world_size: int, device: torch.device | int | None = None,
                   group: Any = None) -> Any:
    """Intra-client gradient communicator on NVLink: the fused ZeRO step when the config asks for sharding
    (``fsdp_config``), the fused all-reduce (replicated optimizer) otherwise."""
    cls = NvlZeroComm if sharded else NvlGradComm
    return cls(total, rank=rank, world_size=world_size, device=device, group=group)

