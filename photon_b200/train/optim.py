"""Local optimizers on flat fp32 buffers: ADOPT and DecoupledAdamW.

The reference reaches these through llm-foundry/Composer per-parameter Python
loops (ref: photon/conf/llm_config/mpt-125m.yaml:58-63 ``adopt``;
mpt-1b.yaml:59-62 ``decoupled_adamw``; state layout ``step, exp_avg,
exp_avg_sq`` confirmed by photon/clients/utils.py:299-370).  Here the whole
model is ONE flat buffer, so a step is one fused multi-tensor kernel on the
GPU (``csrc/optim.cu``: update + bf16 shadow emit + clip-coefficient read from
device memory, no host sync) and a handful of vectorised torch ops on CPU.
The torch path below is also the numerics oracle for the kernel tests.

**Sharded state** (``shard=(lo, hi)`` + ``group``): the in-client replacement for the
reference's FSDP ``FULL_SHARD`` / ``SHARD_GRAD_OP`` (ref: photon/conf/llm_config/
mpt-125m.yaml:85-91; SURVEY §2.5 (b) N2).  Every rank of the client keeps the two
moment planes for its contiguous slice of the flat index space only (8 of the 16
optimizer bytes/param divided by the group size), steps that slice, and the
updated fp32 master + bf16 compute copy are all-gathered slice by slice over
NCCL/NVLink.  Parameters themselves stay replicated (models whose replicated state does not fit use
full parameter sharding instead, :func:`photon_b200.parallel.ddp.wants_full_sharding`).
"""
from __future__ import annotations

import math
from typing import Any

import torch

from photon_b200.utils.flat import FlatParams


class FlatOptimizer:
    """Base: owns ``exp_avg`` / ``exp_avg_sq`` planes shaped like the flat params."""

    name = "base"

    def __init__(self, flat: FlatParams, lr: float, betas: tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 0.0, use_kernel: bool | None = None,
                 bf16_shadow: torch.Tensor | None = None, shard: tuple[int, int] | None = None,
                 group: Any = None, shard_bounds: list[tuple[int, int]] | None = None) -> None:
        self.flat = flat
        total = flat.params.numel()
        self.shard = (int(shard[0]), int(shard[1])) if shard is not None else (0, total)
        self.sharded = self.shard != (0, total)
        self.group, self.shard_bounds = group, shard_bounds
        self.lr = float(lr)
        self.initial_lr = float(lr)
        self.beta1, self.beta2 = float(betas[0]), float(betas[1])
        self.eps = float(eps)
        self.weight_decay = float(weight_decay)
        self.step_count = 0
        n_local = self.shard[1] - self.shard[0]
        self.exp_avg = torch.zeros(n_local, dtype=flat.params.dtype, device=flat.params.device)
        self.exp_avg_sq = torch.zeros_like(self.exp_avg)
        self.bf16_shadow = bf16_shadow
        if use_kernel is None:
            use_kernel = flat.params.is_cuda
        self.use_kernel = bool(use_kernel)

    # -- API ------------------------------------------------------------------------
    def step(self, lr_factor: float = 1.0, grad_mult: torch.Tensor | float | None = None) -> None:
        """One update. ``grad_mult`` (clip coefficient × 1/loss-scale) may be a 0-dim
        device tensor so clipping never synchronises the host."""
        lr = self.initial_lr * float(lr_factor)
        self.lr = lr
        if self.use_kernel:
            from photon_b200 import ops

            ops.fused_optimizer_step(self, lr, grad_mult)
        else:
            lo, hi = self.shard
            g = self.flat.grads[lo:hi]
            if grad_mult is not None:
                g = g * grad_mult
            p = self.flat.params[lo:hi]
            self._torch_step(p, g, lr)
            if self.bf16_shadow is not None:
                self.bf16_shadow[lo:hi].copy_(p)
        self.step_count += 1
        if self.sharded:
            self.all_gather_params()

    # -- sharded state ---------------------------------------------------------------
    def local_views(self) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor | None]:
        """(params, grads, bf16 shadow) restricted to this rank's slice."""
        lo, hi = self.shard
        sh = self.bf16_shadow[lo:hi] if self.bf16_shadow is not None else None
        return self.flat.params[lo:hi], self.flat.grads[lo:hi], sh

    def all_gather_params(self) -> None:
        """Every rank publishes its freshly stepped slice of the fp32 master (and bf16 copy)."""
        import torch.distributed as dist

        if not self.shard_bounds:
            raise RuntimeError("sharded optimizer needs shard_bounds (one (lo, hi) per group rank)")
        for r, (lo, hi) in enumerate(self.shard_bounds):
            if hi <= lo:
                continue
            src = dist.get_global_rank(self.group, r) if self.group is not None else r
            dist.broadcast(self.flat.params[lo:hi], src=src, group=self.group)
            if self.bf16_shadow is not None:
                dist.broadcast(self.bf16_shadow[lo:hi], src=src, group=self.group)

    def full_moments(self) -> tuple[torch.Tensor, torch.Tensor]:
        """(exp_avg, exp_avg_sq) over the whole flat index space (gathered when sharded)."""
        if not self.sharded:
            return self.exp_avg, self.exp_avg_sq
        import torch.distributed as dist

        out = []
        for plane in (self.exp_avg, self.exp_avg_sq):
            full = torch.zeros_like(self.flat.params)
            full[self.shard[0]:self.shard[1]].copy_(plane)
            for r, (lo, hi) in enumerate(self.shard_bounds or []):
                if hi > lo:
                    dist.broadcast(full[lo:hi], src=dist.get_global_rank(self.group, r) if self.group is not None else r,
                                   group=self.group)
            out.append(full)
        return out[0], out[1]

    def set_full_moments(self, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor) -> None:
        lo, hi = self.shard
        self.exp_avg.copy_(exp_avg[lo:hi])
        self.exp_avg_sq.copy_(exp_avg_sq[lo:hi])

    def _torch_step(self, p: torch.Tensor, g: torch.Tensor, lr: float) -> None:
        raise NotImplementedError

    def reset_state(self) -> None:
        self.step_count = 0
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()

    def state_dict(self) -> dict[str, Any]:
        return {"name": self.name, "step": self.step_count, "lr": self.lr, "initial_lr": self.initial_lr,
                "betas": (self.beta1, self.beta2), "eps": self.eps, "weight_decay": self.weight_decay,
                "shard": self.shard,
                "exp_avg": self.exp_avg.detach().cpu(), "exp_avg_sq": self.exp_avg_sq.detach().cpu()}

    def load_state_dict(self, sd: dict[str, Any]) -> None:
        self.step_count = int(sd["step"])
        saved = tuple(sd.get("shard", self.shard))
        if saved != self.shard:
            if saved == (0, self.flat.params.numel()):  # full-state checkpoint into a sharded optimizer
                self.set_full_moments(sd["exp_avg"].to(self.exp_avg.device), sd["exp_avg_sq"].to(self.exp_avg.device))
                return
            raise ValueError(f"optimizer checkpoint holds shard {saved}, this rank owns {self.shard}")
        self.exp_avg.copy_(sd["exp_avg"].to(self.exp_avg.device))
        self.exp_avg_sq.copy_(sd["exp_avg_sq"].to(self.exp_avg_sq.device))


class ADOPT(FlatOptimizer):
    """ADOPT (Taniguchi et al. 2024) with time-dependent clipping ``step**0.25``.
    Step 0 only seeds ``v = g²``; later ``ĝ = clamp(g / max(√v, eps)); m = β1 m +
    (1-β1) ĝ; θ -= lr m; v = β2 v + (1-β2) g²`` — no bias correction."""

    name = "adopt"

    def __init__(self, *a: Any, clip_exp: float | None = 0.25, decouple: bool = True, **kw: Any) -> None:
        super().__init__(*a, **kw)
        self.clip_exp = clip_exp
        self.decouple = decouple

    def _torch_step(self, p: torch.Tensor, g: torch.Tensor, lr: float) -> None:
        if self.weight_decay and not self.decouple:
            g = g + self.weight_decay * p
        if self.step_count == 0:
            self.exp_avg_sq.copy_(g * g)
            return
        if self.weight_decay and self.decouple:
            p.mul_(1.0 - lr * self.weight_decay)
        denom = self.exp_avg_sq.sqrt().clamp_(min=self.eps)
        ng = g / denom
        if self.clip_exp is not None:
            c = float(self.step_count) ** self.clip_exp
            ng.clamp_(-c, c)
        self.exp_avg.lerp_(ng, 1.0 - self.beta1)
        p.add_(self.exp_avg, alpha=-lr)
        self.exp_avg_sq.mul_(self.beta2).addcmul_(g, g, value=1.0 - self.beta2)


class DecoupledAdamW(FlatOptimizer):
    """Composer's DecoupledAdamW: Adam with bias correction; weight decay is
    ``θ *= 1 - (lr/lr₀)·wd`` (decoupled from the LR magnitude)."""

    name = "decoupled_adamw"

    def _torch_step(self, p: torch.Tensor, g: torch.Tensor, lr: float) -> None:
        t = self.step_count + 1
        if self.weight_decay:
            p.mul_(1.0 - (lr / self.initial_lr) * self.weight_decay)
        self.exp_avg.lerp_(g, 1.0 - self.beta1)
        self.exp_avg_sq.mul_(self.beta2).addcmul_(g, g, value=1.0 - self.beta2)
        bc1 = 1.0 - self.beta1 ** t
        bc2 = 1.0 - self.beta2 ** t
        denom = (self.exp_avg_sq.sqrt() / math.sqrt(bc2)).add_(self.eps)
        p.addcdiv_(self.exp_avg, denom, value=-lr / bc1)


class SGD(FlatOptimizer):
    """Plain SGD (no state) — handy for tests and as a LocalSGD inner optimizer."""

    name = "sgd"

    def _torch_step(self, p: torch.Tensor, g: torch.Tensor, lr: float) -> None:
        if self.weight_decay:
            p.mul_(1.0 - lr * self.weight_decay)
        p.add_(g, alpha=-lr)


_REGISTRY = {"adopt": ADOPT, "decoupled_adamw": DecoupledAdamW, "adamw": DecoupledAdamW, "sgd": SGD}


def build_optimizer(cfg: dict[str, Any], flat: FlatParams, **kw: Any) -> FlatOptimizer:
    cfg = dict(cfg)
    name = cfg.pop("name")
    if name not in _REGISTRY:
        raise ValueError(f"unknown optimizer '{name}' (have {sorted(_REGISTRY)})")
    betas = tuple(cfg.pop("betas", (0.9, 0.999)))
    known = {k: cfg.pop(k) for k in ("lr", "eps", "weight_decay") if k in cfg}
    extra = {k: cfg[k] for k in ("clip_exp", "decouple") if k in cfg and name == "adopt"}
    return _REGISTRY[name](flat, betas=betas, **known, **extra, **kw)


def clip_coefficient(total_norm: torch.Tensor, max_norm: float) -> torch.Tensor:
    """``min(1, max_norm / (‖g‖ + 1e-6))`` as a device scalar (``clip_grad_norm_`` rule)."""
    return torch.clamp(max_norm / (total_norm + 1e-6), max=1.0)
