"""MPT decoder-only LM (``mpt_causal_lm``) in plain PyTorch.

This is the *oracle / CPU / baseline* implementation: parameter names, init
and math follow what the reference trains through llm-foundry
(ref: photon/conf/llm_config/mpt-125m.yaml:18-28; names relied on at
photon/utils.py:572,591,602-637; SURVEY Appendix C). The B200 hot path lives in
:mod:`photon_b200.models.engine`, which runs the same parameters through
hand-written sm_90a kernels and is tested against this module.

Block: ``x = x + attn(norm_1(x)); x = x + ffn(norm_2(x))``; ``ffn = down(act(up(x)))`` (``mptmlp``) or
``down(act(gate(x)) * up(x))`` (``mptglu``), ``act`` exact GELU (default) or SiLU; every norm LayerNorm (default) or RMSNorm
(``norm_type``); LM head tied to ``wte`` (default) or its own ``lm_head`` (``tie_word_embeddings: false``), its logits optionally
scaled (``logit_scale``) and soft-capped (``final_logit_softcapping``, see :func:`head_transform`); loss = CE over
``targets = roll(labels, -1)`` with the last position ignored (-100).
"""
from __future__ import annotations

import math
import numbers
from dataclasses import dataclass, field
from typing import Any

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class MPTConfig:
    d_model: int = 768
    n_heads: int = 12
    n_layers: int = 12
    expansion_ratio: float = 4   # may be fractional, as in llm-foundry: the FFN width is int(d_model * expansion_ratio)
    max_seq_len: int = 2048
    vocab_size: int = 50368
    attn_impl: str = "flash"  # flash | torch | b200
    alibi: bool = False
    alibi_bias_max: int = 8
    rope: bool = False
    rope_theta: float = 10000.0
    qk_ln: bool = False
    clip_qkv: float | None = None
    no_bias: bool = False
    learned_pos_emb: bool = True
    norm_eps: float = 1e-5
    # model.norm_type: "layernorm" (LayerNorm, weight + bias unless no_bias) or "rmsnorm" (RMSNorm, weight only) for norm_1,
    # norm_2, norm_f and, under qk_ln, q_ln / k_ln; any name of NORM_TYPES is accepted and stored as one of the two
    norm_type: str = "layernorm"
    # attn_config.attn_uses_sequence_id: attention stays inside each document of a packed row (the collator's sequence_id)
    attn_uses_sequence_id: bool = False
    # attn_config.attn_type grouped_query_attention / multiquery_attention: K / V have kv_n_heads heads (None: n_heads), query
    # head h attending with kv head h // (n_heads // kv_n_heads)
    kv_n_heads: int | None = None
    # attn_config.sliding_window_size W: query i sees keys i - W .. i only (W + 1 keys, intersected with the document mask;
    # positions stay absolute); -1 is off. Unrelated to the ICL evaluator's context truncation.
    sliding_window_size: int = -1
    # attn_config.softmax_scale: the factor on q·k in every attention path (None: 1 / sqrt(d_head))
    softmax_scale: float | None = None
    # ffn_config (llm-foundry): ffn_type mptmlp (down(act(up(x)))) or mptglu (down(act(gate(x)) * up(x))); ffn_act_fn gelu
    # (exact) or silu; ffn_hidden_size overrides the width int(d_model * expansion_ratio)
    ffn_type: str = "mptmlp"
    ffn_act: str = "gelu"
    ffn_hidden_size: int | None = None
    # LM head (llm-foundry MPTForCausalLM): tie_word_embeddings false gives it its own weight lm_head.weight [V, d] (no bias);
    # logit_scale (None, a number or "inv_sqrt_d_model") and final_logit_softcapping c (None or a number) transform its logits
    # as c · tanh(scale · x / c), see head_transform
    tie_word_embeddings: bool = True
    logit_scale: float | str | None = None
    final_logit_softcapping: float | None = None
    init_std: float | None = None  # None -> kaiming_normal_ (llm-foundry default)
    extra: dict[str, Any] = field(default_factory=dict)

    def __post_init__(self) -> None:
        if self.kv_n_heads is None:
            self.kv_n_heads = self.n_heads
        if self.kv_n_heads < 1 or self.n_heads % self.kv_n_heads:
            raise ValueError(f"kv_n_heads = {self.kv_n_heads} must divide n_heads = {self.n_heads}")
        if self.ffn_type not in FFN_TYPES:
            raise ValueError(f"unsupported ffn_config.ffn_type {self.ffn_type!r} (supported: {', '.join(FFN_TYPES)})")
        if self.ffn_act not in FFN_ACTS:
            raise ValueError(f"unsupported FFN activation {self.ffn_act!r} (supported: {', '.join(FFN_ACTS)})")
        if self.ffn_hidden < 1:
            raise ValueError(f"the FFN width must be positive, got {self.ffn_hidden}")
        norm = str(self.norm_type).lower()
        if norm not in NORM_TYPES:
            raise ValueError(f"unsupported model.norm_type {self.norm_type!r} (supported: {', '.join(NORM_TYPES)})")
        self.norm_type = NORM_TYPES[norm]
        w = self.sliding_window_size
        if isinstance(w, bool) or not isinstance(w, numbers.Integral) or w < -1:
            raise ValueError(f"attn_config.sliding_window_size must be an integer >= 0, or -1 (off); got {w!r}")
        self.sliding_window_size = int(w)
        sc = self.softmax_scale
        if sc is not None:
            if isinstance(sc, bool) or not isinstance(sc, numbers.Real) or not math.isfinite(sc) or sc <= 0:
                raise ValueError(f"attn_config.softmax_scale must be a positive number or None; got {sc!r}")
            self.softmax_scale = float(sc)
        if not isinstance(self.tie_word_embeddings, (bool, np.bool_)):
            raise ValueError(f"tie_word_embeddings must be true or false; got {self.tie_word_embeddings!r}")
        self.tie_word_embeddings = bool(self.tie_word_embeddings)
        ls = self.logit_scale
        if isinstance(ls, str):
            if ls != "inv_sqrt_d_model":
                raise ValueError(f"logit_scale must be a positive number, 'inv_sqrt_d_model' or None; got {ls!r}")
        elif ls is not None:
            self.logit_scale = _positive(ls, "logit_scale")
        if self.final_logit_softcapping is not None:
            self.final_logit_softcapping = _positive(self.final_logit_softcapping, "final_logit_softcapping")

    @property
    def head_scale(self) -> float | None:
        """The factor on the LM head's logits: ``logit_scale`` as a number (``inv_sqrt_d_model`` = ``1 / sqrt(d_model)``), None
        without one."""
        if self.logit_scale == "inv_sqrt_d_model":
            return 1.0 / math.sqrt(self.d_model)
        return self.logit_scale

    @property
    def head_transformed(self) -> bool:
        """Whether the LM head's logits go through :func:`head_transform` (a scale or a cap is set)."""
        return self.head_scale is not None or self.final_logit_softcapping is not None

    @property
    def attn_scale(self) -> float:
        """The attention score scale: ``softmax_scale``, else ``1 / sqrt(d_head)``."""
        return 1.0 / math.sqrt(self.d_head) if self.softmax_scale is None else self.softmax_scale

    @property
    def rmsnorm(self) -> bool:
        return self.norm_type == "rmsnorm"

    @property
    def ffn_hidden(self) -> int:
        """Width ``F`` of the feed-forward block: ``ffn_config.ffn_hidden_size``, else ``int(d_model * expansion_ratio)``."""
        return int(self.ffn_hidden_size) if self.ffn_hidden_size is not None else int(self.d_model * self.expansion_ratio)

    @property
    def ffn_gated(self) -> bool:
        return self.ffn_type == "mptglu"

    @property
    def d_head(self) -> int:
        return self.d_model // self.n_heads

    @property
    def kv_dim(self) -> int:
        """Width of the k (and of the v) part of the fused QKV projection: ``kv_n_heads * d_head``."""
        return self.kv_n_heads * self.d_head

    @property
    def qkv_dim(self) -> int:
        """Output width of ``Wqkv``: q (``d_model``), then k, then v (``kv_dim`` each)."""
        return self.d_model + 2 * self.kv_dim

    @classmethod
    def from_model_cfg(cls, m: dict[str, Any]) -> "MPTConfig":
        """Build from ``llm_config.model`` (unknown llm-foundry keys are kept in ``extra``)."""
        m = dict(m)
        attn = dict(m.pop("attn_config", {}) or {})
        rope_cfg = attn.pop("rope_impl", None)
        n_heads = m["n_heads"]
        attn_type = attn.pop("attn_type", "multihead_attention")
        kv = attn.pop("kv_n_heads", None)
        if attn_type == "multihead_attention":
            kv = None   # ignored, as llm-foundry does
        elif attn_type == "multiquery_attention":
            kv = 1
        elif attn_type == "grouped_query_attention":
            if kv is None:
                raise ValueError("attn_config.attn_type: grouped_query_attention needs attn_config.kv_n_heads")
            if int(kv) < 1 or n_heads % int(kv):
                raise ValueError(f"attn_config.kv_n_heads = {kv} must divide n_heads = {n_heads}")
            kv = int(kv)
        else:
            raise ValueError(f"unknown attn_config.attn_type {attn_type!r} (multihead_attention, grouped_query_attention or "
                             "multiquery_attention)")
        if attn_type != "multihead_attention":
            # both change the names or shapes of the attention parameters, which are built here only for multi-head attention
            if attn.get("qk_gn"):
                raise ValueError(f"attn_config.qk_gn is not supported with {attn_type}")
            if attn.get("fused_qkv", True) is False:
                raise ValueError(f"attn_config.fused_qkv: false is not supported with {attn_type}")
        known = dict(
            d_model=m.pop("d_model"), n_heads=m.pop("n_heads"), n_layers=m.pop("n_layers"),
            expansion_ratio=m.pop("expansion_ratio", 4), max_seq_len=m.pop("max_seq_len", 2048),
            vocab_size=m.pop("vocab_size", 50368), attn_impl=attn.pop("attn_impl", "flash"),
            alibi=bool(attn.pop("alibi", False)), alibi_bias_max=attn.pop("alibi_bias_max", 8),
            rope=bool(attn.pop("rope", False)), rope_theta=float(attn.pop("rope_theta", 10000.0)),
            qk_ln=bool(attn.pop("qk_ln", False)), clip_qkv=attn.pop("clip_qkv", None),
            attn_uses_sequence_id=bool(attn.pop("attn_uses_sequence_id", False)), kv_n_heads=kv,
            sliding_window_size=attn.pop("sliding_window_size", -1), softmax_scale=attn.pop("softmax_scale", None),
            no_bias=bool(m.pop("no_bias", False)), learned_pos_emb=bool(m.pop("learned_pos_emb", True)),
            norm_type=m.pop("norm_type", "low_precision_layernorm"), norm_eps=float(m.pop("norm_eps", 1e-5)),
            tie_word_embeddings=m.pop("tie_word_embeddings", True), logit_scale=m.pop("logit_scale", None),
            final_logit_softcapping=m.pop("final_logit_softcapping", None),
        )
        ffn = dict(m.pop("ffn_config", {}) or {})
        known.update(ffn_type=ffn.pop("ffn_type", "mptmlp"), ffn_act=parse_ffn_act(ffn.pop("ffn_act_fn", None)),
                     ffn_hidden_size=ffn.pop("ffn_hidden_size", None))
        for k in ("name", "init_device"):
            m.pop(k, None)
        cfg = cls(**known, extra={**m, **({"attn_config": attn} if attn else {}), **({"ffn_config": ffn} if ffn else {}),
                                  **({"rope_impl": rope_cfg} if rope_cfg else {})})
        if cfg.d_model % cfg.n_heads:
            raise ValueError("d_model must be divisible by n_heads")
        if cfg.alibi or cfg.rope:
            cfg.learned_pos_emb = False if (cfg.alibi or cfg.rope) and "learned_pos_emb" not in m else cfg.learned_pos_emb
        return cfg

    def num_params(self) -> int:
        d, L, V, S, f = self.d_model, self.n_layers, self.vocab_size, self.max_seq_len, self.ffn_hidden
        b = 0 if self.no_bias else 1
        n = 1 if self.no_bias or self.rmsnorm else 2   # tensors per norm: weight, and a LayerNorm's bias unless no_bias
        w = self.qkv_dim
        per_block = 2 * n * d + (w * d + b * w) + (d * d + b * d) + (f * d + b * f) + (f * d + b * d)
        if self.ffn_gated:
            per_block += f * d + b * f   # gate_proj
        head = 0 if self.tie_word_embeddings else V * d   # lm_head.weight
        return V * d + head + (S * d if self.learned_pos_emb else 0) + L * per_block + n * d

    def flops_per_token(self, seq_len: int | None = None) -> float:
        """fwd+bwd model FLOPs per token as SpeedMonitor counts them: 6·N + 12·L·d·S."""
        s = seq_len or self.max_seq_len
        return 6.0 * self.num_params() + 12.0 * self.n_layers * self.d_model * s


FFN_TYPES = ("mptmlp", "mptglu")
# llm-foundry's norm registry -> the normalisation built for it (the low-precision and Triton variants compute the same
# function with the same parameters)
NORM_TYPES = {"layernorm": "layernorm", "low_precision_layernorm": "layernorm", "rmsnorm": "rmsnorm",
              "low_precision_rmsnorm": "rmsnorm", "triton_rmsnorm": "rmsnorm"}
FFN_ACTS = ("gelu", "silu")


def _positive(v: Any, key: str) -> float:
    # a negative scale would reverse the greedy argmax, which the decoder takes on the raw logits (see head_transform)
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v <= 0:
        raise ValueError(f"{key} must be a positive finite number or None; got {v!r}")
    return float(v)


def head_transform(x: torch.Tensor, scale: float | None, cap: float | None) -> torch.Tensor:
    """The LM head's logit transform: ``y = scale · x`` (``logit_scale``), then ``y = cap · tanh(y / cap)``
    (``final_logit_softcapping``); either may be None. With ``scale > 0`` and ``cap > 0`` (the config refuses anything else)
    it is strictly increasing, so the argmax of ``y`` is the argmax of ``x``. The module applies it to fp32 logits; the scorer
    applies it to the target logits it reads, the fused cross-entropy kernel computes the same function per logit."""
    if scale is not None:
        x = x * scale
    if cap is not None:
        x = cap * torch.tanh(x / cap)
    return x


def parse_ffn_act(spec: dict[str, Any] | None) -> str:
    """``ffn_config.ffn_act_fn`` (``{name: <torch.nn.functional name>, **kwargs}``, default exact GELU) -> "gelu" or "silu".
    Anything else is refused rather than approximated."""
    if spec is None:
        return "gelu"
    given, spec = dict(spec), dict(spec)
    name = spec.pop("name", None)
    if name == "gelu" and spec.pop("approximate", "none") == "none" and not spec:
        return "gelu"
    if name == "silu" and not spec.pop("inplace", False) and not spec:
        return "silu"
    raise ValueError(f"unsupported ffn_config.ffn_act_fn {given!r} (supported: {{name: gelu, approximate: none}}, "
                     "{name: silu})")


def ffn_act(x: torch.Tensor, name: str) -> torch.Tensor:
    return F.silu(x) if name == "silu" else F.gelu(x)


def nondefault_ffn(cfg: MPTConfig) -> bool:
    """A feed-forward block other than llm-foundry's default ``mptmlp`` with exact GELU (the width does not count)."""
    return cfg.ffn_type != "mptmlp" or cfg.ffn_act != "gelu"


def ffn_desc(cfg: MPTConfig) -> str:
    return f"ffn_config ffn_type={cfg.ffn_type} ffn_act_fn={cfg.ffn_act}"


def at_least_fp32(x: torch.Tensor) -> torch.Tensor:
    """``x`` in fp32, or in float64 when it already is: the module's fp32 steps (softmax, cross-entropy, RMSNorm, the head's
    transform) keep a float64 model in float64 throughout."""
    return x if x.dtype == torch.float64 else x.float()


def alibi_slopes(n_heads: int, bias_max: int = 8, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """Per-head ALiBi slopes (power-of-two ladder, interleaved for non-pow2 head counts)."""
    p2 = 2 ** math.ceil(math.log2(n_heads))
    m = torch.arange(1, p2 + 1, dtype=dtype) * (bias_max / p2)
    slopes = 1.0 / torch.pow(2.0, m)
    if p2 != n_heads:
        slopes = torch.cat([slopes[1::2], slopes[::2]])[:n_heads]
    return slopes


def window_keep(S: int, window: int, device: Any = None) -> torch.Tensor | None:
    """The sliding window's part of the attention mask: bool [S, S], True where key ``j >= i - window`` (the causal part is
    separate). None when the window is off or wide enough (``window >= S - 1``) to leave causal attention unchanged."""
    if window < 0 or window >= S - 1:
        return None
    return torch.ones(S, S, dtype=torch.bool, device=device).triu(-window)


def rope_tables(seq_len: int, d_head: int, theta: float, device: Any = None,
                dtype: torch.dtype = torch.float32) -> tuple[torch.Tensor, torch.Tensor]:
    inv = 1.0 / (theta ** (torch.arange(0, d_head, 2, dtype=dtype, device=device) / d_head))
    ang = torch.outer(torch.arange(seq_len, dtype=dtype, device=device), inv)
    return ang.cos(), ang.sin()


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x: [B,H,S,dh]; rotate-half (GPT-NeoX) convention."""
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    c, s = cos[None, None].to(x.dtype), sin[None, None].to(x.dtype)
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)


class RMSNorm(nn.Module):
    """llm-foundry's ``RMSNorm``: ``y = x · rsqrt(mean(x²) + eps) · weight`` in fp32 (float64 for float64 inputs), cast back
    to the input dtype; ``weight`` only, initialised to ones."""

    def __init__(self, d: int, eps: float) -> None:
        super().__init__()
        self.eps = float(eps)
        self.weight = nn.Parameter(torch.ones(d))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xf = at_least_fp32(x)
        return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + self.eps) * at_least_fp32(self.weight)).to(x.dtype)


def build_norm(cfg: MPTConfig, d: int, bias: bool) -> nn.Module:
    """The normalisation of ``cfg.norm_type`` over ``d`` features (``bias``: whether a LayerNorm has one)."""
    return RMSNorm(d, cfg.norm_eps) if cfg.rmsnorm else nn.LayerNorm(d, eps=cfg.norm_eps, bias=bias)


class MPTAttention(nn.Module):
    def __init__(self, cfg: MPTConfig) -> None:
        super().__init__()
        self.cfg = cfg
        d = cfg.d_model
        self.Wqkv = nn.Linear(d, cfg.qkv_dim, bias=not cfg.no_bias)
        self.out_proj = nn.Linear(d, d, bias=not cfg.no_bias)
        if cfg.qk_ln:
            self.q_ln = build_norm(cfg, d, bias=True)
            self.k_ln = build_norm(cfg, cfg.kv_dim, bias=True)

    def forward(self, x: torch.Tensor, rope: tuple[torch.Tensor, torch.Tensor] | None,
                alibi: torch.Tensor | None, doc_keep: torch.Tensor | None = None) -> torch.Tensor:
        """``doc_keep``: optional bool [B, 1, S, S], True where query and key belong to the same document."""
        cfg = self.cfg
        B, S, d = x.shape
        qkv = self.Wqkv(x)
        if cfg.clip_qkv:
            qkv = qkv.clamp(-cfg.clip_qkv, cfg.clip_qkv)
        q, k, v = qkv.split([d, cfg.kv_dim, cfg.kv_dim], dim=-1)
        if cfg.qk_ln:
            q, k = self.q_ln(q).to(q.dtype), self.k_ln(k).to(k.dtype)
        H, Hkv, dh = cfg.n_heads, cfg.kv_n_heads, cfg.d_head
        q = q.view(B, S, H, dh).transpose(1, 2)
        k, v = (t.view(B, S, Hkv, dh).transpose(1, 2) for t in (k, v))
        if rope is not None:
            q, k = apply_rope(q, rope[0][:S], rope[1][:S]), apply_rope(k, rope[0][:S], rope[1][:S])
        scale = cfg.attn_scale
        win = window_keep(S, cfg.sliding_window_size, x.device)
        if cfg.attn_impl == "torch" or (alibi is not None and cfg.attn_impl != "flash"):
            if Hkv != H:   # query head h reads kv head h // (H // Hkv)
                k, v = k.repeat_interleave(H // Hkv, dim=1), v.repeat_interleave(H // Hkv, dim=1)
            att = (q @ k.transpose(-1, -2)) * scale
            if alibi is not None:
                att = att + alibi[:, :, :S, :S].to(att.dtype)
            mask = torch.ones(S, S, dtype=torch.bool, device=x.device).tril()
            if doc_keep is not None:
                mask = mask & doc_keep
            if win is not None:
                mask = mask & win
            att = att.masked_fill(~mask, float("-inf"))
            o = torch.softmax(at_least_fp32(att), dim=-1).to(v.dtype) @ v
        else:
            bias = None
            if alibi is not None or doc_keep is not None or win is not None:
                mask = torch.ones(S, S, dtype=torch.bool, device=x.device).tril()
                if doc_keep is not None:
                    mask = mask & doc_keep
                if win is not None:
                    mask = mask & win
                bias = mask if alibi is None else alibi[:, :, :S, :S].to(q.dtype).masked_fill(~mask, float("-inf"))
            gqa = {"enable_gqa": True} if Hkv != H else {}
            o = F.scaled_dot_product_attention(q, k, v, attn_mask=bias, is_causal=bias is None, scale=scale, **gqa)
        return self.out_proj(o.transpose(1, 2).reshape(B, S, d))


class MPTMLP(nn.Module):
    """``down_proj(act(up_proj(x)))`` at width ``cfg.ffn_hidden``."""

    def __init__(self, cfg: MPTConfig) -> None:
        super().__init__()
        d, f = cfg.d_model, cfg.ffn_hidden
        self.act = cfg.ffn_act
        self.up_proj = nn.Linear(d, f, bias=not cfg.no_bias)
        self.down_proj = nn.Linear(f, d, bias=not cfg.no_bias)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.down_proj(ffn_act(self.up_proj(x), self.act))


class MPTGLU(MPTMLP):
    """``down_proj(act(gate_proj(x)) * up_proj(x))`` (llm-foundry ``mptglu``); ``gate_proj`` is registered after
    ``up_proj`` / ``down_proj``, as there."""

    def __init__(self, cfg: MPTConfig) -> None:
        super().__init__(cfg)
        self.gate_proj = nn.Linear(cfg.d_model, cfg.ffn_hidden, bias=not cfg.no_bias)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.down_proj(ffn_act(self.gate_proj(x), self.act) * self.up_proj(x))


class MPTBlock(nn.Module):
    def __init__(self, cfg: MPTConfig) -> None:
        super().__init__()
        self.norm_1 = build_norm(cfg, cfg.d_model, bias=not cfg.no_bias)
        self.attn = MPTAttention(cfg)
        self.norm_2 = build_norm(cfg, cfg.d_model, bias=not cfg.no_bias)
        self.ffn = MPTGLU(cfg) if cfg.ffn_gated else MPTMLP(cfg)

    def forward(self, x: torch.Tensor, rope: Any, alibi: Any, doc_keep: Any = None) -> torch.Tensor:
        x = x + self.attn(self.norm_1(x).to(x.dtype), rope, alibi, doc_keep)
        return x + self.ffn(self.norm_2(x).to(x.dtype))


class MPTTransformer(nn.Module):
    def __init__(self, cfg: MPTConfig) -> None:
        super().__init__()
        self.wte = nn.Embedding(cfg.vocab_size, cfg.d_model)
        if cfg.learned_pos_emb:
            self.wpe = nn.Embedding(cfg.max_seq_len, cfg.d_model)
        self.blocks = nn.ModuleList([MPTBlock(cfg) for _ in range(cfg.n_layers)])
        self.norm_f = build_norm(cfg, cfg.d_model, bias=not cfg.no_bias)


class MPTForCausalLM(nn.Module):
    """``transformer.*`` parameter tree + LM head (tied to ``wte``, or ``lm_head`` when untied) + shifted-target CE loss."""

    def __init__(self, cfg: MPTConfig, device: Any = None, init: bool = True, seed: int | None = None) -> None:
        super().__init__()
        self.cfg = cfg
        self.activation_checkpointing = False   # fsdp_config.activation_checkpointing (ref: conf/llm_config/mpt-1b.yaml:88)
        with torch.device(device or "cpu"):
            self.transformer = MPTTransformer(cfg)
            if not cfg.tie_word_embeddings:   # after the transformer, as in llm-foundry: its seeded init comes last
                self.lm_head = nn.Linear(cfg.d_model, cfg.vocab_size, bias=False)
        if init:
            self.reset_parameters(seed)
        self._rope_cache: tuple[torch.Tensor, torch.Tensor] | None = None
        self._alibi_cache: torch.Tensor | None = None

    # -- init (llm-foundry ``kaiming_normal_`` param_init_fn; SURVEY App. C) ----
    @torch.no_grad()
    def reset_parameters(self, seed: int | None = None) -> None:
        cfg = self.cfg
        gen = None
        if seed is not None:
            gen = torch.Generator(device="cpu").manual_seed(int(seed))
        div = math.sqrt(2 * cfg.n_layers)

        def _fill(w: torch.Tensor, fan_in: int, residual: bool = False) -> None:
            std = cfg.init_std if cfg.init_std is not None else math.sqrt(2.0 / fan_in)
            tmp = torch.empty(w.shape, dtype=torch.float32).normal_(0.0, std, generator=gen)
            if residual:
                tmp /= div
            w.copy_(tmp.to(w.device, w.dtype))

        for name, mod in self.named_modules():
            if isinstance(mod, nn.Linear):
                if name.endswith("Wqkv"):  # fused: initialise q/k/v slices independently
                    d, kvd = cfg.d_model, cfg.kv_dim
                    for lo, hi in ((0, d), (d, d + kvd), (d + kvd, d + 2 * kvd)):
                        _fill(mod.weight[lo:hi], mod.in_features)
                else:
                    _fill(mod.weight, mod.in_features, residual=name.endswith(("out_proj", "down_proj")))
                if mod.bias is not None:
                    mod.bias.zero_()
            elif isinstance(mod, nn.Embedding):
                _fill(mod.weight, mod.embedding_dim)
            elif isinstance(mod, nn.LayerNorm):
                mod.weight.fill_(1.0)
                if mod.bias is not None:
                    mod.bias.zero_()
            elif isinstance(mod, RMSNorm):
                mod.weight.fill_(1.0)

    # -- forward ----------------------------------------------------------------
    def _aux(self, S: int, device: torch.device) -> tuple[Any, Any]:
        cfg = self.cfg
        rope = alibi = None
        # the position tables are fp32, or float64 for a float64 module
        dt = torch.float64 if self.transformer.wte.weight.dtype == torch.float64 else torch.float32
        if cfg.rope:
            if self._rope_cache is None or self._rope_cache[0].device != device or self._rope_cache[0].dtype != dt:
                self._rope_cache = rope_tables(cfg.max_seq_len, cfg.d_head, cfg.rope_theta, device, dt)
            rope = self._rope_cache
        if cfg.alibi:
            if self._alibi_cache is None or self._alibi_cache.device != device or self._alibi_cache.dtype != dt:
                sl = alibi_slopes(cfg.n_heads, cfg.alibi_bias_max, dt).to(device)
                pos = torch.arange(cfg.max_seq_len, device=device)
                rel = (pos[None, :] - pos[:, None]).clamp(max=0).to(dt)  # -(i-j) for j<=i
                self._alibi_cache = (sl[:, None, None] * rel[None])[None]
            alibi = self._alibi_cache
        return rope, alibi

    def doc_keep(self, sequence_id: torch.Tensor | None) -> torch.Tensor | None:
        """llm-foundry's document mask: bool [B, 1, S, S], True where query and key share a ``sequence_id``; None when
        ``attn_uses_sequence_id`` is off (a given ``sequence_id`` is then ignored) or no ids are given (plain causal)."""
        if not self.cfg.attn_uses_sequence_id or sequence_id is None:
            return None
        return (sequence_id[:, :, None] == sequence_id[:, None, :])[:, None]

    def hidden_states(self, input_ids: torch.Tensor, sequence_id: torch.Tensor | None = None) -> torch.Tensor:
        t = self.transformer
        B, S = input_ids.shape
        if S > self.cfg.max_seq_len:
            raise ValueError(f"sequence length {S} > max_seq_len {self.cfg.max_seq_len}")
        x = t.wte(input_ids)
        if self.cfg.learned_pos_emb:
            x = x + t.wpe(torch.arange(S, device=input_ids.device))[None]
        rope, alibi = self._aux(S, input_ids.device)
        keep = self.doc_keep(sequence_id)
        for blk in t.blocks:
            if self.activation_checkpointing and self.training and torch.is_grad_enabled():
                from torch.utils.checkpoint import checkpoint

                x = checkpoint(blk, x, rope, alibi, keep, use_reentrant=False)   # keep only block inputs, recompute in backward
            else:
                x = blk(x, rope, alibi, keep)
        return t.norm_f(x).to(x.dtype)

    def forward(self, input_ids: torch.Tensor, sequence_id: torch.Tensor | None = None) -> torch.Tensor:
        h = self.hidden_states(input_ids, sequence_id)
        w = self.transformer.wte.weight if self.cfg.tie_word_embeddings else self.lm_head.weight
        logits = F.linear(h, w.to(h.dtype))
        if self.cfg.head_transformed:
            logits = head_transform(at_least_fp32(logits), self.cfg.head_scale, self.cfg.final_logit_softcapping)
        return logits

    def loss(self, input_ids: torch.Tensor, labels: torch.Tensor | None = None,
             reduction: str = "mean", sequence_id: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        """Returns (loss, n_valid_tokens). Targets are shifted *inside* (ref semantics); the target that crosses a document
        boundary stays in the loss."""
        logits = self.forward(input_ids, sequence_id)
        targets = shift_labels(input_ids if labels is None else labels)
        flat = F.cross_entropy(at_least_fp32(logits).view(-1, logits.shape[-1]), targets.view(-1),
                               ignore_index=-100, reduction="sum")
        n = (targets != -100).sum()
        return (flat / n.clamp(min=1) if reduction == "mean" else flat), n


def shift_labels(labels: torch.Tensor) -> torch.Tensor:
    """``targets = roll(labels, -1); targets[:, -1] = -100`` (SURVEY App. C)."""
    t = torch.roll(labels, shifts=-1, dims=1).clone()
    t[:, -1] = -100
    return t


def check_sequence_id(cfg: MPTConfig, sequence_id: torch.Tensor | None, train: bool) -> torch.Tensor | None:
    """The ``sequence_id`` a backend should apply: None when ``attn_uses_sequence_id`` is off (ids are ignored). With it on, a
    training batch must carry ids (llm-foundry raises the same in train mode); an eval batch without them is plain causal."""
    if not cfg.attn_uses_sequence_id:
        return None
    if sequence_id is None and train:
        raise ValueError("sequence_id is required to train with attn_config.attn_uses_sequence_id=true "
                         "(set dataset.eos_token_id or dataset.bos_token_id so the collator emits it)")
    return sequence_id


def build_model(model_cfg: dict[str, Any] | MPTConfig, device: Any = None, seed: int | None = None,
                init: bool = True) -> MPTForCausalLM:
    cfg = model_cfg if isinstance(model_cfg, MPTConfig) else MPTConfig.from_model_cfg(model_cfg)
    return MPTForCausalLM(cfg, device=device, init=init, seed=seed)


def trainable_named_parameters(model: nn.Module) -> list[tuple[str, nn.Parameter]]:
    """Trainable parameters in **lexicographic name order** — the order baked into
    every exchanged payload and ``.npz`` (``blocks.10`` < ``blocks.2``; ref:
    photon/utils.py:316-317, photon/clients/utils.py:854-857)."""
    return sorted(((n, p) for n, p in model.named_parameters() if p.requires_grad), key=lambda kv: kv[0])
