"""fp64 reference of one training step's tail: learning rate, clip coefficient and optimizer update, from the optimizer and
scheduler configs and the step index alone.

It is written from the optimizers' definitions, not from the code that maps them to kernel scalars: nothing here calls
``ops.optimizer_hyper``, the scheduler object or ``FlatOptimizer``, so a wrong learning-rate index, a decay scaled by the
wrong rate, a bias correction one step off or a dropped coupled decay do not cancel out.

* ``lr_factor``: ``cosine_with_warmup`` in closed form: ``t / t_warmup`` during the warmup, then
  ``alpha_f + (1 - alpha_f) * (1 + cos(pi * (t - t_warmup) / (t_max - t_warmup))) / 2``.
* ``clip``: ``‖g‖`` in fp64 and ``min(1, max_norm / (‖g‖ + 1e-6))``.
* ``step`` (``t`` = the step index, 0 for the first step; ``G`` = the clipped gradient):

  - ADOPT: with ``decouple: false`` the gradient is ``G + wd * p`` everywhere below. Step 0 only seeds ``v = G²``. Later
    steps: ``p *= 1 - lr * wd`` (decoupled decay), ``m += (1 - β1) (clamp(G / max(√v, eps), ±t**clip_exp) - m)``,
    ``p -= lr * m``, ``v = β2 v + (1 - β2) G²``.
  - DecoupledAdamW: ``p *= 1 - (lr / lr_0) * wd``, ``m = β1 m + (1 - β1) G``, ``v = β2 v + (1 - β2) G²``,
    ``p -= lr / (1 - β1^(t+1)) * m / (√v / √(1 - β2^(t+1)) + eps)``.
  - SGD: ``p = p * (1 - lr * wd) - lr * G``.

The bounds are ``fused_oracle.optim_step``'s (fp32 ulps per update line of the optimizer kernel, fed with the scalars
derived here), widened by what an fp32 clip coefficient may differ from the fp64 one: ``COEF_REL`` relative, the norm's
relative error (``NORM_REL``) plus the fp32 roundings of ``max_norm``, ``+ 1e-6`` and the division. The widening is the
reference's own change when the coefficient moves by ``COEF_REL`` either way.
"""
from __future__ import annotations

import math
from typing import Any

import torch

import fused_oracle as fo

F64 = torch.float64
NORM_REL = 1e-6 + 2.0 ** -22      # fp32 flat norm (flat_l2_norm is held to 1e-6 of fp64) and a square / sqrt round trip
COEF_REL = NORM_REL + 4 * 2.0 ** -24
KIND = {"adopt": 0, "decoupled_adamw": 1, "adamw": 1, "sgd": 2}

# betas and lr_0 exact in fp32, so the kernel's 1 - beta and the reference's agree before any arithmetic happens. The rates
# keep four steps of the GPU test's model within a few percent of its starting weights (ADOPT and Adam move every weight
# by about lr per step), where the engine's gradients are held to the bf16 bound of the whole-engine test
SETUPS: dict[str, dict[str, Any]] = {
    "adopt": dict(name="adopt", lr=2.0 ** -9, betas=[0.875, 0.9921875], eps=1e-6, weight_decay=0.1, clip_exp=0.25),
    "adopt_coupled": dict(name="adopt", lr=2.0 ** -9, betas=[0.875, 0.9921875], eps=1e-6, weight_decay=0.1, clip_exp=0.25,
                          decouple=False),
    "decoupled_adamw": dict(name="decoupled_adamw", lr=2.0 ** -12, betas=[0.875, 0.9921875], eps=1e-6, weight_decay=0.1),
    "sgd": dict(name="sgd", lr=0.25, weight_decay=0.1),
}
# consecutive learning rates 0, lr/2, lr, 3 lr/4, ... differ by at least 25 %
SCHEDULE = dict(name="cosine_with_warmup", t_warmup="2ba", t_max="5ba", alpha_f=0.0)


def lr_factor(sched: dict[str, Any], t: int) -> float:
    """``cosine_with_warmup`` at batch ``t`` (``t_warmup`` / ``t_max`` given as ``"<n>ba"``)."""
    assert sched["name"] == "cosine_with_warmup"
    tw, tm = int(str(sched["t_warmup"]).removesuffix("ba")), int(str(sched["t_max"]).removesuffix("ba"))
    alpha = float(sched.get("alpha_f", 0.0))
    if t < tw:
        return t / tw
    frac = min(1.0, (t - tw) / (tm - tw))
    return alpha + (1.0 - alpha) * 0.5 * (1.0 + math.cos(math.pi * frac))


def clip(g: torch.Tensor, max_norm: float | None) -> tuple[float, float]:
    """(‖g‖ in fp64, the clip coefficient ``min(1, max_norm / (‖g‖ + 1e-6))``; 1 without a clip)."""
    norm = float(g.to(F64).norm())
    return norm, (1.0 if max_norm is None else min(1.0, max_norm / (norm + 1e-6)))


def plants_for(cfg: dict[str, Any]) -> list[str]:
    """The optimizer-specific mistakes :func:`step` can plant for ``cfg``."""
    kind = KIND[cfg["name"]]
    if kind == 1:
        return ["bias correction at t", "decay scaled by lr"]
    if kind == 0 and not cfg.get("decouple", True) and cfg.get("weight_decay"):
        return ["coupled decay dropped"]
    return []


def _scalars(cfg: dict[str, Any], t: int, lr: float, plant: str | None) -> dict[str, Any]:
    """Per-step scalars of the optimizer in ``fused_oracle.optim_step``'s terms, derived from the config alone."""
    kind = KIND[cfg["name"]]
    lr0, wd = float(cfg["lr"]), float(cfg.get("weight_decay", 0.0))
    b1, b2 = (float(b) for b in cfg.get("betas", (0.9, 0.999)))
    h = dict(first=False, lr=lr, beta1=b1, beta2=b2, eps=float(cfg.get("eps", 1e-8)), decay=1.0, wd=0.0, clip=math.inf,
             step_size=0.0, inv_sqrt_bc2=1.0)
    if kind == 0:
        h["first"] = t == 0
        if cfg.get("decouple", True):
            h["decay"] = 1.0 - lr * wd
        elif plant != "coupled decay dropped":
            h["wd"] = wd
        if t > 0 and cfg.get("clip_exp", 0.25) is not None:
            h["clip"] = float(t) ** cfg.get("clip_exp", 0.25)
    elif kind == 1:
        k = t if plant == "bias correction at t" else t + 1
        h["decay"] = 1.0 - (lr if plant == "decay scaled by lr" else lr / lr0) * wd
        h["step_size"] = lr / (1.0 - b1 ** k) if k > 0 else math.inf
        h["inv_sqrt_bc2"] = 1.0 / math.sqrt(1.0 - b2 ** k) if k > 0 else math.inf
    else:
        h["decay"] = 1.0 - lr * wd
    return h


def _update(kind: int, h: dict[str, Any], p: torch.Tensor, G: torch.Tensor, m: torch.Tensor, v: torch.Tensor):
    """The update in fp64 from the definitions in the module docstring."""
    if kind == 2:
        return p * h["decay"] - h["lr"] * G, m, v
    if kind == 1:
        m1 = h["beta1"] * m + (1.0 - h["beta1"]) * G
        v1 = h["beta2"] * v + (1.0 - h["beta2"]) * G * G
        return p * h["decay"] - h["step_size"] * m1 / (v1.sqrt() * h["inv_sqrt_bc2"] + h["eps"]), m1, v1
    if h["wd"]:
        G = G + h["wd"] * p
    if h["first"]:
        return p, m, G * G
    ng = (G / v.sqrt().clamp(min=h["eps"])).clamp(-h["clip"], h["clip"])
    m1 = m + (1.0 - h["beta1"]) * (ng - m)
    return p * h["decay"] - h["lr"] * m1, m1, h["beta2"] * v + (1.0 - h["beta2"]) * G * G


def step(cfg: dict[str, Any], t: int, lr: float, p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor,
         coef: float = 1.0, coef_rel: float = COEF_REL, plant: str | None = None):
    """Step ``t`` at learning rate ``lr`` from (p, m, v) with gradient ``g`` times the clip coefficient ``coef`` (all fp64).
    Returns (p, m, v, tol). ``plant``: "coupled decay dropped", "bias correction at t" or "decay scaled by lr" computes that
    mistake instead (the plants the tests must flag)."""
    kind = KIND[cfg["name"]]
    h = _scalars(cfg, t, lr, plant)
    p, g, m, v = (x.to(F64) for x in (p, g, m, v))
    out = _update(kind, h, p, g * coef, m, v)
    # fused_oracle's bounds of the optimizer kernel for this state and these scalars
    _, _, _, tol = fo.optim_step(kind, p, g, m if kind != 2 else p, v if kind != 2 else p, h, grad_mult=coef)
    tol = dict(tol)
    if coef_rel:
        for c in (coef * (1.0 + coef_rel), coef * (1.0 - coef_rel)):
            for key, a, b in zip("pmv", out, _update(kind, h, p, g * c, m, v)):
                tol[key] = tol[key] + (b - a).abs()
    return out[0], out[1], out[2], tol
