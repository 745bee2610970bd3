"""Compute backends behind the Trainer.

``TorchBackend`` = MPT in stock PyTorch ops with autograd (CPU path, numerics
oracle, and the "reference-equivalent" GPU baseline: cuBLAS GEMMs, SDPA/FA2
attention, ATen LN/GELU/CE under ``torch.autocast`` — what the reference gets
from Composer + llm-foundry, ref: photon/clients/trainer_utils.py:1615-1719).

``photon_b200.models.engine.B200Engine`` implements the same protocol with the
hand-written sm_90a kernels and an explicit (autograd-free) backward; the
Trainer does not care which one it drives.

Protocol
--------
``flat``                      :class:`FlatParams` (fp32 master params + grads)
``fwd_bwd(ids, denom, scale[, sequence_id])``  accumulate d(Σ token-loss · scale / denom) into ``flat.grads``;
                              returns device scalars ``(loss_sum, n_tokens)``
``eval_stats(ids[, sequence_id])``  ``{"loss_sum","n_tokens","n_correct"[, "unigram_loss_sum"]}``
                              (``sequence_id``: the collator's per-token document ids, applied when the model's
                              ``attn_uses_sequence_id`` is on)
``params_updated()``          hook after optimizer / parameter load (refresh shadows)
"""
from __future__ import annotations

import contextlib
from typing import Any

import torch
import torch.nn.functional as F

from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, check_sequence_id, ffn_desc, nondefault_ffn, shift_labels
from photon_b200.utils.flat import FlatParams


def autocast_ctx(device: torch.device, precision: str) -> Any:
    if precision == "fp32":
        return contextlib.nullcontext()
    dt = torch.float16 if precision == "amp_fp16" else torch.bfloat16
    return torch.autocast(device_type=device.type, dtype=dt)


def apply_freeze(model: torch.nn.Module, frozen: list[str] | None, unfrozen: list[str] | None) -> list[str]:
    """Exact-name freeze lists (ref: photon/utils.py:322-387). Frozen tensors drop out of
    the exchanged parameter list because only ``requires_grad`` tensors are flat-packed."""
    if frozen and unfrozen:
        raise ValueError("frozen_layers and unfrozen_layers are mutually exclusive")
    names = [n for n, _ in model.named_parameters()]
    touched = []
    if frozen:
        missing = [n for n in frozen if n not in names]
        if missing:
            raise KeyError(f"frozen_layers not in model: {missing[:4]}")
        for n, p in model.named_parameters():
            if n in frozen:
                p.requires_grad_(False)
                touched.append(n)
    elif unfrozen:
        missing = [n for n in unfrozen if n not in names]
        if missing:
            raise KeyError(f"unfrozen_layers not in model: {missing[:4]}")
        for n, p in model.named_parameters():
            if n not in unfrozen:
                p.requires_grad_(False)
                touched.append(n)
    return touched


class TorchBackend:
    kind = "torch"

    def __init__(self, cfg: MPTConfig, device: torch.device | str = "cpu", precision: str = "amp_bf16",
                 seed: int | None = 17, frozen_layers: list[str] | None = None,
                 unfrozen_layers: list[str] | None = None, unigram_log_probs: torch.Tensor | None = None,
                 grads_storage: torch.Tensor | None = None, activation_checkpointing: bool = False,
                 params_storage: torch.Tensor | None = None, shadow_storage: torch.Tensor | None = None) -> None:
        self.cfg = cfg
        self.device = torch.device(device)
        self.precision = precision
        self.model = MPTForCausalLM(cfg, device=self.device, seed=seed)
        self.model.activation_checkpointing = bool(activation_checkpointing)
        self.frozen = apply_freeze(self.model, frozen_layers, unfrozen_layers)
        self.flat = FlatParams(self.model, device=self.device, params_storage=params_storage, grads_storage=grads_storage)
        self.bf16_params = shadow_storage   # only kept so a fused NVLink step has a plane to write (autocast casts on the fly)
        self.fp8_layers: list[str] = []
        if precision == "amp_fp8":          # E4M3 forward / E5M2 backward GEMM operands with delayed scaling, bf16 elsewhere
            from photon_b200.train.fp8 import enable_fp8

            self.fp8_layers = enable_fp8(self.model)
        self.unigram_log_probs = unigram_log_probs.to(self.device) if unigram_log_probs is not None else None
        self.collect_activation_stats = False
        self.activation_stats: dict[str, float] = {}
        self.launches_per_microbatch = 0  # stock torch ops are not "our" kernels

    # -- training ---------------------------------------------------------------------
    def fwd_bwd(self, ids: torch.Tensor, denom: float, scale: float = 1.0,
                sequence_id: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        sequence_id = check_sequence_id(self.cfg, sequence_id, train=True)
        with autocast_ctx(self.device, self.precision):
            loss_sum, n = self.model.loss(ids, reduction="sum", sequence_id=sequence_id)
        (loss_sum * (scale / denom)).backward()
        if self.collect_activation_stats:
            self._act_stats(ids)
        return loss_sum.detach(), n

    @torch.no_grad()
    def _act_stats(self, ids: torch.Tensor) -> None:
        t = self.model.transformer
        x = t.wte(ids[:1])
        if self.cfg.learned_pos_emb:
            x = x + t.wpe(torch.arange(ids.shape[1], device=ids.device))[None]
        rope, alibi = self.model._aux(ids.shape[1], ids.device)  # noqa: SLF001
        for i, blk in enumerate(t.blocks):
            x = blk(x, rope, alibi)
            self.activation_stats[f"l2_norm/block_{i}"] = float(x.float().norm(dim=-1).mean())
            self.activation_stats[f"max/block_{i}"] = float(x.abs().max())

    # -- evaluation -------------------------------------------------------------------
    @torch.no_grad()
    def eval_stats(self, ids: torch.Tensor, sequence_id: torch.Tensor | None = None) -> dict[str, torch.Tensor]:
        with autocast_ctx(self.device, self.precision):
            logits = self.model(ids, check_sequence_id(self.cfg, sequence_id, train=False))
        targets = shift_labels(ids)
        lf = logits.float().view(-1, logits.shape[-1])
        tf = targets.view(-1)
        out = {"loss_sum": F.cross_entropy(lf, tf, ignore_index=-100, reduction="sum"),
               "n_tokens": (tf != -100).sum(),
               "n_correct": ((lf.argmax(-1) == tf) & (tf != -100)).sum()}
        if self.unigram_log_probs is not None:
            from photon_b200.metrics.language import unigram_loss_sum

            out["unigram_loss_sum"] = unigram_loss_sum(tf, self.unigram_log_probs)
        return out

    @torch.no_grad()
    def logits(self, ids: torch.Tensor) -> torch.Tensor:
        """``[B,S] → [B,S,V]`` next-token logits (the in-context-learning evaluator's view of the model)."""
        with autocast_ctx(self.device, self.precision):
            return self.model(ids.to(self.device))

    def params_updated(self) -> None:
        pass

    def train_mode(self, on: bool = True) -> None:
        self.model.train(on)

    def close(self) -> None:
        pass


def build_backend(model_cfg: MPTConfig, device: torch.device, precision: str, kernels: dict[str, Any] | None = None,
                  **kw: Any) -> Any:
    """Pick the compute backend. On a CUDA device the sm_90a engine (``B200Engine``) is THE path (and fails
    loudly if its extension is missing); ``kernels.gemm: torch`` etc. selects the stock
    PyTorch baseline explicitly; CPU always uses stock PyTorch."""
    kernels = dict(kernels or {})
    modes = [kernels.get(k, "auto") for k in ("gemm", "attention", "norm", "loss", "optimizer")]
    want_engine = device.type == "cuda" and not all(m == "torch" for m in modes)
    if any(m == "b200" for m in modes) and device.type != "cuda":
        raise RuntimeError("kernels.*=b200 requires a CUDA (sm_90a) device")
    if want_engine:
        unsupported = []
        if precision not in ("amp_bf16", "amp_fp8"):
            unsupported.append(f"precision={precision}")
        if (kw.get("frozen_layers") or kw.get("unfrozen_layers")) and kw.get("zero3") is not None:
            unsupported.append("frozen/unfrozen layers")   # the ZeRO-3 unit plan assumes every block tensor is in the flat
        if nondefault_ffn(model_cfg) and (precision == "amp_fp8" or kw.get("zero3") is not None):
            # the fp8 weight roles, the fp8 GELU epilogue and the ZeRO-3 unit plan know the four mptmlp block matrices only
            unsupported.append(f"{ffn_desc(model_cfg)} with {'amp_fp8' if precision == 'amp_fp8' else 'full parameter sharding'}")
        if unsupported:
            print(f"[backend] {', '.join(unsupported)} not covered by the sm_90a engine -> stock PyTorch backend "
                  "(explicit, logged; set kernels.*=torch to silence)", flush=True)
            kw.pop("zero3", None)
            return TorchBackend(model_cfg, device=device, precision=precision, **kw)
        from photon_b200.models.engine import B200Engine

        return B200Engine(model_cfg, device=device, precision=precision, kernels=kernels, **kw)
    if kw.pop("zero3", None) is not None:
        raise RuntimeError("full parameter sharding (NvlZero3Comm) needs the sm_90a engine on a CUDA device")
    return TorchBackend(model_cfg, device=device, precision=precision, **kw)
