"""Reference model for the whole-engine tests: an fp64 oracle, a bf16 baseline, and a per-tensor acceptance criterion.

* ``oracle``: :class:`MPTForCausalLM` in float64 (explicit attention, ``attn_impl="torch"``) with the engine's weights upcast,
  run with fp64 autograd over one or more microbatches, each with its own ``scale`` / ``denom``. The weights are those the
  engine computes with (the tests make its fp32 masters bf16-exact), so weight rounding is not counted as engine error.
* ``baseline``: the same module and weights in pure bf16 (``.to(torch.bfloat16)``): every activation is stored in bf16, as the
  engine stores them. Its distance from the oracle is the error bf16 arithmetic makes on that exact input. Run it on the GPU
  with ``torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False``.
* ``Checker.tensor(name, got, ref, base)``: with ``o`` the oracle, ``b`` the baseline and ``g`` the engine,

  - whole tensor: ``|g - o| <= A * |b - o| + F * |o|`` (L2 norms);
  - scale: with ``s(x) = <x - o, o> / <o, o>``, ``|s(g)| <= P * (|s(b)| + |b - o| / (|o| * sqrt(n))) + F``. The L2 part cannot
    see a uniform 2 % scaling under 1-2 % of bf16 noise; this part does;
  - row blocks of 128 along the first dimension (output features of a weight, vocabulary rows of ``wte`` / ``lm_head``,
    positions of ``wpe``, token rows of logits): ``max|g - o| <= M * max|b - o| + F * max|o|`` per block. This part finds a
    wrong tail tile;
  - exact zeros: where ``o`` and ``b`` are exactly zero (a frozen tensor, ``wpe`` rows at or past the sequence length, the ``wte`` rows
    of absent tokens under an untied head) ``g`` must be bitwise zero.

* ``Checker.sum``: a sum over tokens (a loss sum, a pair's log p) against the baseline's pooled per-token error.
* ``KNOWN``: (variant, tensor, part) where the H100 engine measurably misses the bound, with the cause. ``Checker`` reports
  those as an expected failure instead of widening the bound for everyone.

Slack constants (``BF16``) are set from the worst ratios measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit over
every variant and engine mode of ``test_engine_oracle_gpu.py``, outside ``KNOWN``, given as ratio to the bound at the slack
in force (<= 1 passes):

  - whole tensor, A = 1.5: worst 0.82 (the v part of the QKV bias under clip_qkv; the engine is within 1.25x the
    baseline's L2 error everywhere);
  - scale, P = 8: worst 0.84 (Wqkv and up_proj weights of the last block under a logit cap: s(g) = 6e-4 against
    s(b) = 6e-5; every other tensor needs P < 4);
  - row blocks, M = 2: worst 0.97 (a norm weight), 0.59 on logits;
  - floor F = 1e-4; loss and log p sums: worst 0.86 of ``Checker.sum``'s bound at A.

A larger M no longer catches the tail-tile and one-head plants on the engine's own gradients (they sit at 1.0-1.1x at
M = 2); hence ``KNOWN`` rather than a wider M. ``FP8`` (amp_fp8 against the ``TorchBackend("amp_fp8")`` emulation): worst
whole 0.74, scale 0.30.
"""
from __future__ import annotations

import dataclasses
import fnmatch
import math
from dataclasses import dataclass, field
from typing import Any

import torch
import torch.nn.functional as F

from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, at_least_fp32, head_transform, shift_labels

ROWS = 128


@dataclass(frozen=True)
class Slack:
    whole: float     # A
    scale: float     # P
    block: float     # M
    floor: float     # F
    parts: tuple[str, ...] = ("whole", "scale", "block", "zeros")


BF16 = Slack(whole=1.5, scale=8.0, block=2.0, floor=1e-4)
# amp_fp8 against the TorchBackend("amp_fp8") emulation: E4M3 / E5M2 scaling decisions differ between the two, element errors
# do not line up, so only the whole-tensor and scale parts apply
FP8 = Slack(whole=1.5, scale=4.0, block=math.inf, floor=1e-3, parts=("whole", "scale", "zeros"))

# (variant, tensor, part) patterns (fnmatch) -> why the H100 engine misses the bound there. The attention backward takes
# delta = rowsum(dO * O) from the bf16-rounded O, so the rows of dS do not sum to zero (attention_oracle.KNOWN); the residual
# multiplies whatever component all keys (for dQ) or all queries (for dK) share.
_RESIDUAL = ("the attention backward's delta comes from the bf16-rounded O, so the rows of dS do not sum to zero "
             "(attention_oracle.KNOWN)")
KNOWN: dict[tuple[str, str, str], str] = {
    # the key part of the QKV bias without RoPE: a bias shared by every key shifts whole score rows, so its exact gradient is
    # zero (or, behind qk_ln, what is left after a per-token normalisation): both engine and baseline are rounding noise there,
    # the engine's up to 3.3x the baseline's by block max
    ("*", "transformer.blocks.*.attn.Wqkv.bias:k", "*"): "key bias gradient, zero in exact arithmetic: " + _RESIDUAL,
    # k_ln's bias is shared by every key: the same, for the whole tensor (whole 2.2x, block 2.4x its bound)
    ("qk_ln_clip", "transformer.blocks.*.attn.k_ln.bias", "*"): "k_ln bias gradient, zero in exact arithmetic: " + _RESIDUAL,
    # k_ln's bias is a component every key shares: the residual lands in dQ and in q_ln's weight gradient (block 1.5x)
    ("gqa", "transformer.blocks.*.attn.q_ln.weight", "block"): "q_ln weight gradient through dQ: " + _RESIDUAL,
    # clip_qkv 0.5 clips most of q, k, v: a value within a bf16 step of the clip passes the gradient in one computation and not
    # in the other, so a whole token's contribution to a row differs (block up to 1.5x)
    ("qk_ln_clip", "transformer.blocks.*.attn.Wqkv.*", "block"): "values within a bf16 step of clip_qkv are clipped in one "
                                                                 "computation and not in the other",
}


def known(variant: str, name: str, part: str) -> str | None:
    for (v, n, p), why in KNOWN.items():
        if fnmatch.fnmatchcase(variant, v) and fnmatch.fnmatchcase(name, n) and fnmatch.fnmatchcase(part, p):
            return why
    return None


# ------------------------------------------------------------------------------------------------ the model
@dataclass
class Batch:
    ids: torch.Tensor                      # [B, S] int64
    scale: float = 1.0
    denom: float = 1.0
    sequence_id: torch.Tensor | None = None


@dataclass
class Result:
    loss_sum: float                        # sum over microbatches of the summed token losses (unscaled)
    n_tokens: int
    token_loss: list[torch.Tensor]         # per microbatch: [B, S] float64 token losses (0 where ignored)
    logits: list[torch.Tensor]             # per microbatch: [B, S, V] float64 raw head logits (before logit_scale / cap)
    grads: dict[str, torch.Tensor] = field(default_factory=dict)   # name -> float64 d(sum_m loss_m * scale_m / denom_m)


def build(cfg: MPTConfig, weights: dict[str, torch.Tensor], dtype: torch.dtype, device: Any = None) -> MPTForCausalLM:
    """The module of ``cfg`` (explicit attention) in ``dtype`` holding ``weights`` (name -> tensor, cast to ``dtype``)."""
    m = MPTForCausalLM(dataclasses.replace(cfg, attn_impl="torch"), device=device, init=False).to(dtype)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.copy_(weights[n].to(p.device, dtype))
    return m


def bf16_exact_weights(named: Any, seed: int) -> dict[str, torch.Tensor]:
    """fp32 weights for a test, every value exactly representable in bf16: the matrices of ``named`` (name -> tensor, e.g. a
    freshly initialised module) rounded, biases drawn from N(0, 0.05^2) and norm weights from 1 + N(0, 0.1^2) instead of the
    init's zeros and ones, so a bias or a norm weight applied wrongly changes the result."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    for n, p in sorted(dict(named).items()):
        x = p.detach().float().cpu().clone()
        if n.endswith(".bias"):
            x = 0.05 * torch.randn(x.shape, generator=gen)
        elif x.dim() == 1:
            x = 1.0 + 0.1 * torch.randn(x.shape, generator=gen)
        out[n] = x.bfloat16().float()
    return out


def transformed(cfg: MPTConfig, raw: torch.Tensor) -> torch.Tensor:
    """The logits the loss reads: ``raw`` through the head's transform (fp32, or float64 for float64 input), as the module."""
    return head_transform(at_least_fp32(raw), cfg.head_scale, cfg.final_logit_softcapping) if cfg.head_transformed else raw


def run(m: MPTForCausalLM, batches: list[Batch], frozen: Any = (), grad: bool = True) -> Result:
    """Forward (and, with ``grad``, autograd) of the microbatches through module ``m`` in its own dtype; ``frozen``: names
    without a gradient (their entries in ``grads`` stay zero)."""
    cfg = m.cfg
    frozen = set(frozen or ())
    trainable = [(n, p) for n, p in m.named_parameters() if n not in frozen]
    for n, p in m.named_parameters():
        p.requires_grad_(grad and n not in frozen)
    res = Result(0.0, 0, [], [])
    if grad:
        res.grads = {n: torch.zeros(p.shape, dtype=torch.float64, device=p.device) for n, p in m.named_parameters()}
    head = m.transformer.wte.weight if cfg.tie_word_embeddings else m.lm_head.weight
    for mb in batches:
        ids = mb.ids.to(head.device)
        sid = None if mb.sequence_id is None else mb.sequence_id.to(head.device)
        with torch.set_grad_enabled(grad):
            h = m.hidden_states(ids, sid)
            raw = F.linear(h, head.to(h.dtype))
            logits = transformed(cfg, raw)
            targets = shift_labels(ids)
            tok = F.cross_entropy(at_least_fp32(logits).view(-1, logits.shape[-1]), targets.view(-1), ignore_index=-100,
                                  reduction="none")
            loss = tok.sum()
        if grad:
            gs = torch.autograd.grad(loss * (mb.scale / mb.denom), [p for _, p in trainable], allow_unused=True)
            for (n, _), g in zip(trainable, gs):
                if g is not None:
                    res.grads[n] += g.double()
        res.loss_sum += float(loss.detach().double())
        res.n_tokens += int((targets != -100).sum())
        res.token_loss.append(tok.detach().double().view(ids.shape))
        res.logits.append(raw.detach().double())
    return res


def oracle(cfg: MPTConfig, weights: dict[str, torch.Tensor], batches: list[Batch], frozen: Any = (), device: Any = None,
           grad: bool = True) -> Result:
    """fp64 forward (and, with ``grad``, fp64 autograd) of the microbatches; ``frozen``: names without a gradient."""
    return run(build(cfg, weights, torch.float64, device), batches, frozen, grad)


def baseline(cfg: MPTConfig, weights: dict[str, torch.Tensor], batches: list[Batch], frozen: Any = (), device: Any = None,
             grad: bool = True) -> Result:
    """The same module and weights in pure bf16 (the loss and the head's transform in fp32, as the module computes them)."""
    return run(build(cfg, weights, torch.bfloat16, device), batches, frozen, grad)


# ------------------------------------------------------------------------------------------------ criterion
def _ratio(err: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    return torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))


def tensor_report(name: str, got: torch.Tensor, ref: torch.Tensor, base: torch.Tensor, slack: Slack = BF16) -> dict:
    """Each part's ratio of error to bound (<= 1 passes) and a message; see the module docstring. Rows: the first dimension."""
    g, o, b = (t.detach().to(ref.device, torch.float64) for t in (got, ref, base))
    assert g.shape == o.shape == b.shape, (name, got.shape, ref.shape, base.shape)
    n = o.numel()
    g2, o2, b2 = (t.reshape(t.shape[0], -1) if t.dim() > 1 else t.reshape(-1, 1) for t in (g, o, b))
    eg, eb = g2 - o2, b2 - o2
    A, P, M, Fl = slack.whole, slack.scale, slack.block, slack.floor
    no, neg, neb = o2.norm(), eg.norm(), eb.norm()
    oo = (o2 * o2).sum()
    s = (lambda e: ((e * o2).sum() / oo).abs()) if oo > 0 else (lambda e: torch.zeros((), dtype=torch.float64, device=o.device))
    whole = _ratio(neg, A * neb + Fl * no).item()
    noise = neb / (no * math.sqrt(n)) if no > 0 else torch.zeros_like(no)
    scale = _ratio(s(eg), P * (s(eb) + noise) + Fl).item() if no > 0 else 0.0
    R = o2.shape[0]
    nb = -(-R // ROWS)
    pad = nb * ROWS - R

    def blockmax(x):
        x = x.abs().amax(-1)
        return F.pad(x, (0, pad)).view(nb, ROWS).amax(-1)

    ebk = _ratio(blockmax(eg), M * blockmax(eb) + Fl * blockmax(o2)) if math.isfinite(M) else torch.zeros(nb, dtype=torch.float64)
    worst_blk = int(ebk.argmax())
    block = ebk[worst_blk].item()
    # structural zeros: exactly zero in fp64 and in bf16 (a gradient that only cancels to zero, like that of a key bias without
    # RoPE, is rounding noise in both and is left to the other parts)
    zeros = int(((o2 == 0) & (b2 == 0) & (g2 != 0)).sum())
    nan = bool(torch.isnan(g2).any())
    msg = (f"{name}: whole {whole:.2f} (err {neg.item():.3e}, baseline {neb.item():.3e}, |o| {no.item():.3e}); scale {scale:.2f} "
           f"(s(g) {s(eg).item():+.2e}, s(b) {s(eb).item():+.2e}); block {block:.2f} (rows {worst_blk * ROWS}..); "
           f"nonzero where the oracle is zero: {zeros}" + ("; NaN" if nan else ""))
    if nan:
        whole = scale = block = math.inf
    return {"whole": whole, "scale": scale, "block": block, "zeros": zeros, "msg": msg}


def failed_parts(rep: dict, slack: Slack = BF16) -> list[str]:
    return [p for p in slack.parts if (rep[p] > 0 if p == "zeros" else not rep[p] <= 1.0)]


class Checker:
    """Collects the criterion's verdicts over one test, so a failing tensor does not hide the ratios of the others.
    ``finish()`` at the end of the test fails it with every miss; a miss listed in ``KNOWN`` for (variant, tensor, part)
    becomes an expected failure instead (NaN never does). ``worst``: part -> (ratio, where), updated with every ratio."""

    def __init__(self, variant: str, slack: Slack = BF16, worst: dict | None = None) -> None:
        self.variant, self.slack, self.worst = variant, slack, worst
        self.failures: list[str] = []
        self.known: list[str] = []

    def _note(self, part: str, ratio: float, name: str) -> None:
        """Track the worst ratio of each part outside ``KNOWN`` (what the slack constants were set from)."""
        if self.worst is None or known(self.variant, name, part):
            return
        if ratio > self.worst.get(part, (-1.0, ""))[0]:
            self.worst[part] = (ratio, f"{self.variant}:{name}")

    def tensor(self, name: str, got: torch.Tensor, ref: torch.Tensor, base: torch.Tensor) -> dict:
        """Every part of the criterion for one tensor (see the module docstring)."""
        rep = tensor_report(name, got, ref, base, self.slack)
        print(f"[{self.variant}] {rep['msg']}")
        for p in ("whole", "scale", "block"):
            if p in self.slack.parts:
                self._note(p, rep[p], name)
        for p in failed_parts(rep, self.slack):
            why = known(self.variant, name, p)
            if why and math.isfinite(rep[p]):
                self.known.append(f"{why}: {rep['msg']}")
            else:
                self.failures.append(f"[{self.variant}] {name} fails {p}: {rep['msg']}")
        return rep

    def sum(self, name: str, got: float, ref: float, token_err_rms: float, n: int) -> float:
        """A sum of ``n`` per-token values (a loss sum, a pair's log p): ``|g - o| <= A * rms(e) * sqrt(n) + F * |o|`` with ``e``
        the baseline's per-token errors, pooled over every token the test has (``token_err_rms``): the size of a sum of ``n``
        independent token errors, where the baseline's own sum can land near zero by chance."""
        bound = self.slack.whole * token_err_rms * math.sqrt(n) + self.slack.floor * abs(ref)
        err = abs(got - ref)
        r = err / bound if bound > 0 else (math.inf if err > 0 else 0.0)
        if not math.isfinite(got):
            r = math.inf
        print(f"[{self.variant}] {name}: got {got:.6f} oracle {ref:.6f} err {err:.3e} bound {bound:.3e} (ratio {r:.2f})")
        self._note("sum", r, name)
        if not r <= 1.0:
            self.failures.append(f"[{self.variant}] {name}: |{got} - {ref}| = {err:.3e} > {bound:.3e}")
        return r

    def expect(self, ok: bool, msg: str) -> None:
        if not ok:
            self.failures.append(f"[{self.variant}] {msg}")

    def finish(self) -> None:
        assert not self.failures, "\n".join(self.failures)
        if self.known:
            import pytest

            pytest.xfail("known deviation from the bf16 bound: " + " | ".join(self.known))


def rms(x: torch.Tensor) -> float:
    return float(x.double().pow(2).mean().sqrt())


def ambiguous_rows(ref_logits: torch.Tensor, base_logits: torch.Tensor) -> torch.Tensor:
    """bool per row of [..., V] logits: the oracle's top-2 margin is below the baseline's largest logit error on that row, so
    bf16 arithmetic may legitimately pick another argmax."""
    o = ref_logits.double()
    top2 = o.topk(2, dim=-1).values
    return (top2[..., 0] - top2[..., 1]) <= (base_logits.double() - o).abs().amax(-1)


def argmax_bounds(ref_logits: torch.Tensor, base_logits: torch.Tensor, targets: torch.Tensor) -> tuple[int, int]:
    """(least, most) correct next-token predictions an engine may count: rows whose oracle argmax is the target, give or take
    the ambiguous rows (see :func:`ambiguous_rows`); ignored targets (-100) never count."""
    valid = targets != -100
    hit = (ref_logits.argmax(-1) == targets) & valid
    amb = ambiguous_rows(ref_logits, base_logits) & valid
    return int((hit & ~amb).sum()), int((hit | amb).sum())


# ------------------------------------------------------------------------------------------------ plants
def plants(cfg: MPTConfig, S: int, grads: dict[str, torch.Tensor], first_only: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """Small errors the criterion must flag, each planted in a copy of one tensor of ``grads`` (name -> gradient of a
    training step over two microbatches of length ``S``): label -> planted tensor, the label starting with the tensor's name.
    ``first_only``: the gradients of the first microbatch alone (the second microbatch's contribution missing)."""
    d, dh = cfg.d_model, cfg.d_head
    out = {}

    def put(key, tensor, fn):
        x = grads[tensor].detach().clone()
        fn(x)
        out[f"{tensor} {key}"] = x

    bias = "transformer.blocks.1.ffn.down_proj.bias" if not cfg.no_bias else None
    if bias in grads:
        put("x1.02", bias, lambda x: x.mul_(1.02))
    put("x0.98", "transformer.blocks.0.norm_2.weight", lambda x: x.mul_(0.98))
    if cfg.learned_pos_emb:
        put("last 8 positions zeroed", "transformer.wpe.weight", lambda x: x[S - 8:S].zero_())
    head = "transformer.wte.weight" if cfg.tie_word_embeddings else "lm_head.weight"
    tail = (cfg.vocab_size - 1) // ROWS * ROWS
    put("vocabulary tail tile x1.05", head, lambda x: x[tail:].mul_(1.05))
    kv = cfg.kv_n_heads - 1   # the K slice of the last kv head
    put(f"K slice of kv head {kv} x0.95", "transformer.blocks.0.attn.Wqkv.weight",
        lambda x: x[d + kv * dh: d + (kv + 1) * dh].mul_(0.95))
    t = "transformer.blocks.1.attn.out_proj.weight"
    out[f"{t} second microbatch missing"] = first_only[t].detach().clone()
    return out
