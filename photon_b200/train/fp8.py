"""FP8 training recipe (``llm_config.precision: amp_fp8``) — the numerics, independent of who multiplies.

The reference reaches fp8 through Composer's ``amp_fp8`` → TransformerEngine (commented out in its launch script,
ref: scripts/centralised_training.sh:91). The recipe is TE's "delayed scaling":

* forward GEMM operands (activations, weights) are cast to **E4M3**, gradients flowing backward to **E5M2**;
* every tensor role of every linear layer keeps an **amax history**; the scale used at step *t* comes from the history up to
  *t−1* (``scale = fp8_max / (amax · 2^margin)``), so no extra pass over the tensor is needed before the cast;
* products are exact, the result is de-scaled by ``1 / (scale_a · scale_b)`` in the epilogue; LayerNorm, softmax,
  residuals, the LM head and the optimizer stay in bf16 / fp32. This emulation accumulates in fp32; fp8 ``wgmma`` on the H100
  does not: it keeps roughly 13 to 14 bits, an error of about ``2^-10 · Σ|a·b|`` per output (up to ``2^-7`` where the
  products cancel), measured in ``tests/fp8_oracle.py``.

This module implements exactly that as a quantise → de-quantise emulation around ``F.linear`` (runs anywhere, CPU included),
which makes ``amp_fp8`` a real reduced-precision mode of the stock-PyTorch backend and is the oracle a wgmma fp8 GEMM
epilogue has to match. The hand-written engine still computes ``amp_fp8`` runs in bf16 (it says so when it starts).
"""
from __future__ import annotations

import types
from dataclasses import dataclass, field
from typing import Any

import torch
import torch.nn as nn
import torch.nn.functional as F

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}


@dataclass
class Fp8Recipe:
    margin: int = 0
    amax_history_len: int = 16
    amax_compute_algo: str = "max"          # "max" over the history | "most_recent"
    fwd_dtype: torch.dtype = E4M3
    bwd_dtype: torch.dtype = E5M2


@dataclass
class Fp8TensorMeta:
    """Scale + amax history of one tensor role (input / weight / grad-output) of one layer."""

    dtype: torch.dtype
    recipe: Fp8Recipe
    history: list[float] = field(default_factory=list)
    scale: float = 1.0

    def observe(self, x: torch.Tensor) -> None:
        """Record this step's amax and derive the scale for the NEXT cast (delayed scaling)."""
        amax = float(x.detach().abs().max()) if x.numel() else 0.0
        self.history.append(amax)
        del self.history[: -self.recipe.amax_history_len]
        ref = max(self.history) if self.recipe.amax_compute_algo == "max" else self.history[-1]
        if ref > 0.0 and ref == ref and ref != float("inf"):
            self.scale = FP8_MAX[self.dtype] / (ref * 2.0 ** self.recipe.margin)

    def quantize(self, x: torch.Tensor) -> torch.Tensor:
        """``x`` as the fp8 tensor core sees it, returned de-scaled in ``x``'s dtype (saturating cast, like TE)."""
        if not self.history:          # first use: no history yet → scale from the tensor itself
            self.observe(x)
        lim = FP8_MAX[self.dtype]
        q = (x.float() * self.scale).clamp_(-lim, lim).to(self.dtype)
        out = (q.float() / self.scale).to(x.dtype)
        self.observe(x)
        return out


class _Fp8LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, metas: dict[str, Fp8TensorMeta]) -> torch.Tensor:
        xq, wq = metas["input"].quantize(x), metas["weight"].quantize(w)
        ctx.save_for_backward(xq, wq)
        ctx.metas, ctx.has_bias = metas, b is not None
        return F.linear(xq, wq.to(xq.dtype), None if b is None else b.to(xq.dtype))

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor) -> tuple[torch.Tensor | None, ...]:
        xq, wq = ctx.saved_tensors
        dyq = ctx.metas["grad_output"].quantize(dy)
        d2, x2 = dyq.reshape(-1, dyq.shape[-1]).float(), xq.reshape(-1, xq.shape[-1]).float()   # fp8 values, fp32 accumulate
        dx = (d2 @ wq.float()).reshape(xq.shape).to(xq.dtype)                    # dgrad: E5M2 × E4M3
        dw = (d2.t() @ x2).to(wq.dtype)                                          # wgrad: E5M2 × E4M3
        db = dy.reshape(-1, dy.shape[-1]).float().sum(0).to(wq.dtype) if ctx.has_bias else None   # from the unquantised dy
        return dx, dw, db, None


def _fp8_forward(self: nn.Linear, x: torch.Tensor) -> torch.Tensor:
    return _Fp8LinearFn.apply(x, self.weight, self.bias, self._fp8_metas)


def enable_fp8(model: nn.Module, recipe: Fp8Recipe | None = None, skip: tuple[str, ...] = ("lm_head",)) -> list[str]:
    """Route every ``nn.Linear`` of ``model`` (the four GEMMs of each MPT block) through the fp8 recipe. Parameters, their
    names and their fp32 masters are untouched, so flat layouts / checkpoints / the federation payload do not change.
    Returns the names of the converted layers."""
    recipe = recipe or Fp8Recipe()
    done = []
    for name, mod in model.named_modules():
        if isinstance(mod, nn.Linear) and not any(s in name for s in skip) and not hasattr(mod, "_fp8_metas"):
            mod._fp8_metas = {"input": Fp8TensorMeta(recipe.fwd_dtype, recipe), "weight": Fp8TensorMeta(recipe.fwd_dtype, recipe),  # noqa: SLF001
                              "grad_output": Fp8TensorMeta(recipe.bwd_dtype, recipe)}
            mod.forward = types.MethodType(_fp8_forward, mod)
            done.append(name)
    return done


def fp8_state_dict(model: nn.Module) -> dict[str, Any]:
    """Scales and amax histories (checkpointed next to the optimizer so a resumed run casts with the same scales)."""
    return {name: {role: {"scale": m.scale, "history": list(m.history)} for role, m in mod._fp8_metas.items()}  # noqa: SLF001
            for name, mod in model.named_modules() if hasattr(mod, "_fp8_metas")}


def load_fp8_state_dict(model: nn.Module, sd: dict[str, Any]) -> None:
    for name, mod in model.named_modules():
        if hasattr(mod, "_fp8_metas") and name in sd:
            for role, m in mod._fp8_metas.items():  # noqa: SLF001
                if role in sd[name]:
                    m.scale, m.history = float(sd[name][role]["scale"]), list(sd[name][role]["history"])
