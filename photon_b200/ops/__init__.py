"""Python face of the hand-written sm_90a kernels (``photon_b200._C``).

Every function here launches OUR kernels; nothing silently falls back to a
PyTorch op.  If the extension is missing on a machine that has a CUDA device
the import error is raised loudly.  On CPU-only machines the extension still imports
(it is cross-compiled) but these wrappers are never called.
"""
from __future__ import annotations

import math
from typing import Any

import torch

_EXT: Any = None


def ext() -> Any:
    """Load (and cache) the in-tree extension; raise loudly if it is absent."""
    global _EXT
    if _EXT is None:
        try:
            from photon_b200 import _C  # type: ignore[attr-defined]
        except ImportError as e:  # pragma: no cover - depends on the box
            raise ImportError(
                "photon_b200._C (sm_90a kernels) is not built. Run `python -m photon_b200.build` "
                "(or __graft_entry__.build()) — refusing to fall back to PyTorch ops on the GPU path.") from e
        _EXT = _C
    return _EXT


def have_ext() -> bool:
    try:
        ext()
        return True
    except ImportError:
        return False


def launch_count() -> int:
    return int(ext().launch_count())


def reset_launch_count() -> None:
    ext().reset_launch_count()


def add_launch_count(n: int) -> None:
    """Account for kernels replayed from a captured CUDA graph (they never pass through the bindings)."""
    ext().add_launch_count(int(n))


# --------------------------------------------------------------------------------- GEMM
EPI_BF16, EPI_RESIDUAL, EPI_GELU_DUAL, EPI_DGELU, EPI_F32, EPI_GELU_GRAD, EPI_MUL, EPI_GELU_GRAD_Q8 = 0, 1, 2, 3, 4, 5, 6, 7
EPI_SILU_GRAD, EPI_MUL2 = 8, 9
E4M3, E5M2 = 0, 1          # operand formats of the fp8 wgmma GEMMs
FP8_MAX = (448.0, 57344.0)


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         epi: int = EPI_BF16, bias: torch.Tensor | None = None, aux: torch.Tensor | None = None,
         out2: torch.Tensor | None = None, accumulate: bool = False, alpha: float = 1.0, cluster: int = 0,
         aux2: torch.Tensor | None = None) -> torch.Tensor:
    """``out[M,N] = epilogue(alpha * A @ B^T)`` on wgmma tensor cores.

    ``a``: ``[M,K]`` (K-major) or ``[K,M]`` when ``a_mn``; ``b``: ``[N,K]`` or ``[K,N]`` when ``b_mn``."""
    ext().gemm(a, b, out, int(a_mn), int(b_mn), int(epi), bias, aux, out2, bool(accumulate), float(alpha), int(cluster), aux2)
    return out


def linear_fwd(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, out: torch.Tensor,
               residual: torch.Tensor | None = None) -> torch.Tensor:
    """y = x @ w^T + bias (+ residual) — x [T,K], w [N,K] (bf16), bias fp32."""
    return gemm(x, w, out, epi=EPI_RESIDUAL if residual is not None else EPI_BF16, bias=bias, aux=residual)


def linear_gelu_fwd(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, pre: torch.Tensor,
                    act: torch.Tensor) -> torch.Tensor:
    """pre = x @ w^T + bias ; act = gelu(pre) — both written by the same epilogue."""
    return gemm(x, w, act, epi=EPI_GELU_DUAL, bias=bias, out2=pre)


def linear_gelu_grad_fwd(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, dact: torch.Tensor,
                         act: torch.Tensor) -> torch.Tensor:
    """z = x @ w^T + bias ; act = gelu(z) ; dact = gelu'(z) — the derivative is what the backward needs, so it is saved
    INSTEAD of z and the dgrad epilogue becomes a plain multiply (no erf / exp in the backward)."""
    return gemm(x, w, act, epi=EPI_GELU_GRAD, bias=bias, out2=dact)


def linear_silu_grad_fwd(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, dact: torch.Tensor,
                         act: torch.Tensor) -> torch.Tensor:
    """z = x @ w^T + bias ; act = silu(z) = z·σ(z) ; dact = silu'(z) = σ(z)·(1 + z·(1 − σ(z))) — :func:`linear_gelu_grad_fwd`
    with SiLU (one exp per element for both)."""
    return gemm(x, w, act, epi=EPI_SILU_GRAD, bias=bias, out2=dact)


def linear_act_grad_fwd(act_name: str, x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, dact: torch.Tensor,
                        act: torch.Tensor) -> torch.Tensor:
    """:func:`linear_gelu_grad_fwd` (``act_name`` "gelu") or :func:`linear_silu_grad_fwd` ("silu")."""
    f = linear_silu_grad_fwd if act_name == "silu" else linear_gelu_grad_fwd
    return f(x, w, bias, dact, act)


def linear_glu_up_fwd(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, act: torch.Tensor, dact: torch.Tensor,
                      m: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """Up projection of a gated FFN: u = x @ w^T + bias ; m = u * act ; c = u * dact (``act`` / ``dact`` = act(g) / act'(g) of
    the gate projection g). ``m`` is the down projection's input, ``c`` the saved factor of the gate's gradient. The
    outputs must not overlap the multipliers."""
    return gemm(x, w, m, epi=EPI_MUL2, bias=bias, aux=act, aux2=dact, out2=c)


def linear_glu_dgrad(dm: torch.Tensor, w: torch.Tensor, act: torch.Tensor, c: torch.Tensor, du: torch.Tensor,
                     dg: torch.Tensor) -> torch.Tensor:
    """dgrad of a gated FFN's down projection: dm' = dm @ w (w stored [N,K], consumed MN-major) ; du = dm' * act(g) ;
    dg = dm' * c (c = u * act'(g) saved by :func:`linear_glu_up_fwd`): the gradients of the up and gate projections'
    outputs. The outputs must not overlap the multipliers."""
    return gemm(dm, w, du, b_mn=True, epi=EPI_MUL2, aux=act, aux2=c, out2=dg)


def linear_dgrad(dy: torch.Tensor, w: torch.Tensor, dx: torch.Tensor, gelu_pre: torch.Tensor | None = None,
                 mul: torch.Tensor | None = None, residual: torch.Tensor | None = None) -> torch.Tensor:
    """dx = dy @ w  (w stored [N,K] → consumed MN-major, no transpose); optional ``* gelu'(pre)`` (pre-activation given),
    ``* mul`` (saved derivative given) or ``+ residual`` (another input gradient to add; not ``dx`` itself)."""
    if residual is not None:
        return gemm(dy, w, dx, b_mn=True, epi=EPI_RESIDUAL, aux=residual)
    if mul is not None:
        return gemm(dy, w, dx, b_mn=True, epi=EPI_MUL, aux=mul)
    return gemm(dy, w, dx, b_mn=True, epi=EPI_DGELU if gelu_pre is not None else EPI_BF16, aux=gelu_pre)


def linear_wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, accumulate: bool = True, alpha: float = 1.0) -> torch.Tensor:
    """dw[N,K] (+)= dy^T @ x in fp32 (both operands consumed MN-major; red.global.add when accumulating)."""
    return gemm(dy, x, dw, a_mn=True, b_mn=True, epi=EPI_F32, accumulate=accumulate, alpha=alpha)


# ------------------------------------------------------------------------------ fp8 GEMM
def gemm_fp8(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, meta: torch.Tensor, role_a: int, role_b: int, *,
             a_mn: bool = False, b_mn: bool = False, epi: int = EPI_BF16, a_fmt: int = E4M3, b_fmt: int = E4M3,
             bias: torch.Tensor | None = None, aux: torch.Tensor | None = None, out2: torch.Tensor | None = None,
             accumulate: bool = False, alpha: float = 1.0, cluster: int = 0, out8: torch.Tensor | None = None,
             role_out: int = -1) -> torch.Tensor:
    """``out = epilogue(alpha / (scale[role_a] * scale[role_b]) * A8 @ B8^T)`` — 1-byte operands (E4M3 / E5M2 per operand) on
    fp8 ``wgmma`` (MN-major operands are transposed to K-major first), accumulated in fp32 registers at the tensor cores' reduced fp8
    precision (about 2^-10 of Σ|a·b|, see tests/fp8_oracle.py). ``meta`` = float32 ``[3, n_roles]`` (scale, 1/scale, amax) on the device;
    the de-scales are read by the kernel, so nothing here touches the host. ``EPI_GELU_GRAD_Q8`` writes ``out8`` (E4M3,
    scaled by ``scale[role_out]``, amax recorded) and ``out2`` = gelu'; ``out`` is then unused (pass ``out2``)."""
    ext().gemm_fp8(a, b, out, int(a_mn), int(b_mn), int(epi), int(a_fmt), int(b_fmt), meta, int(role_a), int(role_b), bias, aux, out2,
                   bool(accumulate), float(alpha), int(cluster), out8, int(role_out))
    return out


def mx_quantize(x: torch.Tensor, row_blocks: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``[R,K]`` → (E4M3 ``[R,K]`` uint8, E8M0 scale atoms ``[K/128, row_blocks, 512]`` uint8): OCP MXFP8, one power-of-two scale
    per 32 consecutive K elements of a row, stored as 512-byte atoms per 128 rows x 128 K that the GEMM loads with one bulk copy."""
    q, sf = ext().mx_quantize(x, int(row_blocks))
    return q, sf


def gemm_mxfp8(a8: torch.Tensor, b8: torch.Tensor, out: torch.Tensor, sfa: torch.Tensor, sfb: torch.Tensor,
               bias: torch.Tensor | None = None) -> torch.Tensor:
    """``out[M,N] = (A ⊙ SFA) @ (B ⊙ SFB)^T (+ bias)`` with the block scales applied to the fp32 wgmma partial sum
    of every 32-element K group. ``sfb`` needs ``2·ceil(N/256)`` row blocks (``mx_quantize(w, 2 * ceil(N/256))``)."""
    ext().gemm_mxfp8(a8, b8, out, sfa, sfb, bias)
    return out


def layernorm_fwd_q8(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor | None, y8: torch.Tensor, mean: torch.Tensor,
                     rstd: torch.Tensor, eps: float, meta: torch.Tensor, role: int) -> torch.Tensor:
    """LayerNorm whose only output is the E4M3 tensor the next GEMM reads (scaled by ``scale[role]``, ``amax[role]`` updated)."""
    ext().layernorm_fwd_q8(x, gamma, beta, y8, mean, rstd, float(eps), meta, int(role))
    return y8


def rmsnorm_fwd_q8(x: torch.Tensor, gamma: torch.Tensor, y8: torch.Tensor, rstd: torch.Tensor, eps: float, meta: torch.Tensor,
                   role: int) -> torch.Tensor:
    """:func:`layernorm_fwd_q8` for RMSNorm (:func:`rmsnorm_fwd`): E4M3 ``x · rstd · gamma`` and ``rstd``."""
    ext().rmsnorm_fwd_q8(x, gamma, y8, rstd, float(eps), meta, int(role))
    return y8


def colsum_quant(dy: torch.Tensor, out_sum: torch.Tensor | None, y8: torch.Tensor | None, fmt: int = E5M2,
                 meta: torch.Tensor | None = None, role: int = -1) -> None:
    """One read of ``dy`` [T,N]: ``out_sum[j] += Σ_t dy[t,j]`` (bias gradient) and ``y8 = fp8(dy * scale[role])``."""
    ext().colsum_quant(dy, out_sum, y8, int(fmt), meta, int(role))


def fp8_quantize_segments(src_bf16: torch.Tensor, dst8: torch.Tensor, seg: torch.Tensor, meta: torch.Tensor, role0: int) -> None:
    """Per-tensor current scaling of ``seg`` = int64 [n,2] (offset, numel) slices of a flat bf16 plane → E4M3 in ``dst8``."""
    ext().fp8_quantize_segments(src_bf16, dst8, seg, meta, int(role0))


def transpose_u8(src: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """``dst[C,R] = src[R,C]^T`` for 1-byte matrices: a K-major copy of an fp8 operand stored MN-major."""
    ext().transpose_u8(src, dst)
    return dst


def fp8_update_scales(meta: torch.Tensor, hist: torch.Tensor, fmax: torch.Tensor, pos: torch.Tensor, n: int, margin_mult: float = 1.0) -> None:
    """Delayed scaling for roles [0, n): amax → history ring → scale for the next cast; amax reset."""
    ext().fp8_update_scales(meta, hist, fmax, pos, int(n), float(margin_mult))


# ---------------------------------------------------------------------------- fused ops
def embed_fwd(ids: torch.Tensor, wte: torch.Tensor, wpe: torch.Tensor | None, out: torch.Tensor, seq_len: int) -> torch.Tensor:
    ext().embed_fwd(ids, wte, wpe, out, int(seq_len))
    return out


def embed_bwd(ids: torch.Tensor, dh: torch.Tensor, dwte: torch.Tensor | None, dwpe: torch.Tensor | None, seq_len: int) -> None:
    """``dwte[ids[t]] += dh[t]`` and ``dwpe[t % seq_len] += dh[t]`` (fp32); a None gradient (frozen embedding) is skipped."""
    ext().embed_bwd(ids, dh, dwte, dwpe, int(seq_len))


def layernorm_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor | None, y: torch.Tensor, mean: torch.Tensor,
                  rstd: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    ext().layernorm_fwd(x, gamma, beta, y, mean, rstd, float(eps))
    return y


def layernorm_bwd(dy: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor,
                  dres: torch.Tensor | None, dx: torch.Tensor, dgamma: torch.Tensor | None, dbeta: torch.Tensor | None) -> torch.Tensor:
    ext().layernorm_bwd(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta)
    return dx


def rmsnorm_fwd(x: torch.Tensor, gamma: torch.Tensor, y: torch.Tensor, rstd: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """``y = x · rstd · gamma`` per row, ``rstd = rsqrt(mean(x²) + eps)`` in fp32 (llm-foundry's ``rms_norm``); ``rstd`` [T] is
    kept for :func:`rmsnorm_bwd`."""
    ext().rmsnorm_fwd(x, gamma, y, rstd, float(eps))
    return y


def rmsnorm_bwd(dy: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, rstd: torch.Tensor, dres: torch.Tensor | None,
                dx: torch.Tensor, dgamma: torch.Tensor | None) -> torch.Tensor:
    """``dx = rstd · (dy·gamma − x̂ · mean(dy·gamma·x̂)) (+ dres)`` with ``x̂ = x · rstd``; ``dgamma += Σ_t dy·x̂`` unless None."""
    ext().rmsnorm_bwd(dy, x, gamma, rstd, dres, dx, dgamma)
    return dx


def col_sum(dy: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[j] += Σ_t dy[t,j] (bias gradients)."""
    ext().col_sum(dy, out)
    return out


def cross_entropy(logits: torch.Tensor, targets: torch.Tensor, grad_scale: float, write_grad: bool, stats: torch.Tensor,
                  row_lse: torch.Tensor | None = None, unigram_logp: torch.Tensor | None = None, logit_scale: float | None = None,
                  softcap: float | None = None) -> None:
    """In place: logits → dlogits (when ``write_grad``); stats[0..3] += (Σloss, #valid, #correct, Σunigram).

    ``logit_scale`` / ``softcap``: the LM head's transform (:func:`photon_b200.models.mpt.head_transform`) applied to every logit
    before the softmax; the loss and ``row_lse`` are those of the transformed logits, the gradient is w.r.t. the stored ones and
    ``#correct`` counts the argmax of the stored logits (the transform is increasing). None: no scale / no cap."""
    ext().cross_entropy(logits, targets, float(grad_scale), bool(write_grad), stats, row_lse, unigram_logp,
                        1.0 if logit_scale is None else float(logit_scale), 0.0 if softcap is None else float(softcap))


_NORM_SCRATCH: dict[int, tuple[torch.Tensor, torch.Tensor]] = {}


def flat_l2_norm(x: torch.Tensor) -> torch.Tensor:
    """‖x‖₂ of a flat fp32 buffer as a 0-dim device tensor (no host sync).

    Any length: the kernel reads float4s and then the last ``numel % 4`` elements. ``x`` must be contiguous and start on a
    16-byte boundary (a slice of a padded flat buffer at a multiple of 4 elements); anything else raises."""
    key = x.device.index or 0
    if key not in _NORM_SCRATCH:
        _NORM_SCRATCH[key] = (torch.zeros(1, dtype=torch.float64, device=x.device), torch.zeros(1, dtype=torch.float32, device=x.device))
    scratch, out = _NORM_SCRATCH[key]
    ext().flat_l2_norm(x, scratch, out)
    return out[0]


def axpby_(acc: torch.Tensor, x: torch.Tensor, a: float, b: float) -> torch.Tensor:
    ext().axpby(acc, x, float(a), float(b))
    return acc


def cast_bf16(src: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
    """``dst = bf16(src)``, round to nearest even, the same bits as ``src.to(torch.bfloat16)`` (fp32 subnormals are kept, not
    flushed); the length must be a multiple of 4."""
    ext().cast_bf16(src, dst)
    return dst


_KIND = {"adopt": 0, "decoupled_adamw": 1, "sgd": 2}


def optimizer_hyper(opt: Any, lr: float) -> dict[str, Any]:
    """Per-step scalar arguments of the fused optimizer kernels for a :class:`FlatOptimizer` at learning rate ``lr``."""
    kind = _KIND[opt.name]
    first = kind == 0 and opt.step_count == 0
    decay, wd, clip, step_size, inv_sqrt_bc2 = 1.0, 0.0, float("inf"), 0.0, 1.0
    if kind == 0:
        if opt.weight_decay and getattr(opt, "decouple", True):
            decay = 1.0 - lr * opt.weight_decay
        elif opt.weight_decay:      # coupled: the kernel adds wd * p to the gradient (before the step-0 seed of v too)
            wd = opt.weight_decay
        if opt.clip_exp is not None and not first:
            clip = float(opt.step_count) ** opt.clip_exp
    elif kind == 1:
        t = opt.step_count + 1
        decay = 1.0 - (lr / opt.initial_lr) * opt.weight_decay if opt.weight_decay else 1.0
        step_size = lr / (1.0 - opt.beta1 ** t)
        inv_sqrt_bc2 = 1.0 / math.sqrt(1.0 - opt.beta2 ** t)
    else:
        decay = 1.0 - lr * opt.weight_decay if opt.weight_decay else 1.0
    return dict(kind=kind, first=first, lr=float(lr), beta1=opt.beta1, beta2=opt.beta2, eps=opt.eps, decay=float(decay),
                wd=float(wd), clip=float(clip), step_size=float(step_size), inv_sqrt_bc2=float(inv_sqrt_bc2))


def fused_optimizer_step(opt: Any, lr: float, grad_mult: torch.Tensor | float | None) -> None:
    """One fused multi-tensor step for a :class:`photon_b200.train.optim.FlatOptimizer`."""
    flat = opt.flat
    h = optimizer_hyper(opt, lr)
    gm = None
    if grad_mult is not None:
        gm = grad_mult if torch.is_tensor(grad_mult) else torch.tensor(float(grad_mult), device=flat.params.device)
        gm = gm.to(torch.float32).reshape(1)
    params, grads, shadow = opt.local_views()   # the whole flat buffer, or this rank's slice when the state is sharded
    ext().fused_optimizer(params, grads, opt.exp_avg, opt.exp_avg_sq, shadow, h["kind"], h["first"], h["lr"],
                          h["beta1"], h["beta2"], h["eps"], h["decay"], h["clip"], h["step_size"], h["inv_sqrt_bc2"], gm,
                          wd=h["wd"])


# ---------------------------------------------------------------------------- attention
def _kv(n_heads: int, n_kv_heads: int | None) -> int:
    return int(n_heads) if n_kv_heads is None else int(n_kv_heads)


def attention_fwd(qkv: torch.Tensor, out: torch.Tensor, lse: torch.Tensor, n_heads: int, scale: float, causal: bool = True,
                  alibi_slopes: torch.Tensor | None = None, doc_start: torch.Tensor | None = None,
                  n_kv_heads: int | None = None, window: int = -1) -> None:
    """``qkv`` [B, S, (n_heads + 2 * n_kv_heads) * d_head]: the q heads, then the k heads, then the v heads; query head ``h``
    attends with kv head ``h // (n_heads // n_kv_heads)`` (grouped-query attention; None: ``n_heads``, multi-head).
    ``alibi_slopes``: optional fp32 [n_heads]; adds ``slope_h * (key - query)`` to the scores (MPT ``attn_config.alibi``).
    ``doc_start``: optional int32 [B*S] from :func:`doc_bounds` (causal only); query ``q`` then sees key ``k`` iff
    ``doc_start[q] <= k <= q``, and key tiles before a query tile's first document are skipped.
    ``window``: sliding window (causal only; -1: off). Query ``q`` then sees keys ``q - window .. q`` only (intersected with
    the document mask), and key tiles before a query tile's window are skipped."""
    ext().attention_fwd(qkv, out, lse, int(n_heads), float(scale), bool(causal), alibi_slopes, doc_start, _kv(n_heads, n_kv_heads),
                        int(window))


def attention_bwd(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, dqkv: torch.Tensor,
                  delta: torch.Tensor, n_heads: int, scale: float, causal: bool = True,
                  alibi_slopes: torch.Tensor | None = None, doc_start: torch.Tensor | None = None,
                  doc_end: torch.Tensor | None = None, n_kv_heads: int | None = None, window: int = -1) -> None:
    """``doc_start`` / ``doc_end`` (both or neither) and ``window``: the document mask and sliding window of
    :func:`attention_fwd`. ``dqkv`` is shaped like ``qkv``; with grouped-query attention the dK / dV of a kv head are summed
    over its query heads."""
    ext().attention_bwd(qkv, out, dout, lse, dqkv, delta, int(n_heads), float(scale), bool(causal), alibi_slopes, doc_start, doc_end,
                        _kv(n_heads, n_kv_heads), int(window))


def doc_bounds(sequence_id: torch.Tensor, doc_start: torch.Tensor, doc_end: torch.Tensor) -> None:
    """``sequence_id`` int64 [B, S] -> ``doc_start`` / ``doc_end`` int32 [B*S]: the first / last row (within its sequence) of
    each row's document. Documents are maximal runs of equal ids."""
    ext().doc_bounds(sequence_id, doc_start, doc_end)


def rope_(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, inverse: bool = False,
          n_kv_heads: int | None = None) -> torch.Tensor:
    """In-place rotary embedding (rotate-half) of the ``n_heads`` q heads and ``n_kv_heads`` k heads of ``qkv``
    [B, S, (n_heads + 2 * n_kv_heads) * d_head]; ``inverse`` applies the transposed rotation (what the gradients of q and k need)."""
    ext().rope(qkv, cos, sin, int(n_heads), bool(inverse), _kv(n_heads, n_kv_heads))
    return qkv


# ---------------------------------------------------------------------------- decoding
SKINNY_PLAIN, SKINNY_RESIDUAL, SKINNY_GELU, SKINNY_SILU, SKINNY_MUL = 0, 1, 2, 3, 4


def skinny_gemm(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, bias: torch.Tensor | None = None,
                residual: torch.Tensor | None = None, gelu: bool = False, silu: bool = False,
                mul: torch.Tensor | None = None) -> torch.Tensor:
    """``out[M,N] = x[M,K] @ w[N,K]^T (+ bias) (+ residual | then exact GELU | then SiLU | then * mul)`` for 1 <= M <= 64 rows
    (decode steps): the weight rows stream through the GPU once, K is split when the 64-column tiles cannot fill it, and split
    partials are summed in a fixed order, so the result is bitwise reproducible."""
    if mul is not None:
        epi, residual = SKINNY_MUL, mul
    else:
        epi = SKINNY_GELU if gelu else SKINNY_SILU if silu else (SKINNY_RESIDUAL if residual is not None else SKINNY_PLAIN)
    ext().skinny_gemm(x, w, out, bias, residual, epi)
    return out


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, n_heads: int,
                     scale: float, alibi_slopes: torch.Tensor | None = None, n_kv_heads: int | None = None,
                     window: int = -1) -> torch.Tensor:
    """One query row per sequence (``q`` [B, >= H*dh]) against one layer of the cache (``k_cache`` / ``v_cache``
    [B_max, n_kv_heads, S_max, dh]) over keys ``0..pos[b]`` (int32 on the device; ``window`` >= 0: keys
    ``max(0, pos[b] - window)..pos[b]``); ``out`` [B, H*dh]. One CTA serves all query heads of a kv head, so each cached row is
    read once per group."""
    ext().decode_attention(q, k_cache, v_cache, pos, out, int(n_heads), float(scale), alibi_slopes, _kv(n_heads, n_kv_heads),
                           int(window))
    return out


def decode_append(qkv: torch.Tensor, pos: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
                  rope: tuple[torch.Tensor, torch.Tensor] | None, n_heads: int, slot: torch.Tensor | None = None,
                  n_kv_heads: int | None = None) -> None:
    """Rotate q / k of every row of the fused ``qkv`` [B, (n_heads + 2 * n_kv_heads) * d_head] at position ``pos[b]`` (``rope`` =
    the ``rope_`` tables, or None) and write the k / v heads into the cache at ``pos[b]`` of slot ``slot[b]`` (int32 on the
    device; None: row ``b`` writes slot ``b``)."""
    cos, sin = rope if rope is not None else (None, None)
    ext().decode_append(qkv, pos, k_cache, v_cache, cos, sin, int(n_heads), slot, _kv(n_heads, n_kv_heads))


def cache_attention(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, tiles: torch.Tensor, out: torch.Tensor,
                    n_heads: int, scale: float, alibi_slopes: torch.Tensor | None = None, n_kv_heads: int | None = None,
                    window: int = -1) -> torch.Tensor:
    """Several query rows per cache slot on the tensor cores. ``tiles`` int32 [T, 4] on the device, one row per tile
    ``(slot, first_row, n_rows <= 64, first_pos)``: rows ``first_row + i`` of ``qkv`` [N, (n_heads + 2 * n_kv_heads) * d_head]
    (q after RoPE) sit at positions ``first_pos + i`` of that slot and attend to its keys ``0 .. first_pos + i`` (query head
    ``h`` to kv head ``h // (n_heads // n_kv_heads)``; ``window`` >= 0: keys from ``first_pos + i - window`` on). Writes
    those rows of ``out`` [N, d] only."""
    ext().cache_attention(qkv, k_cache, v_cache, tiles, out, int(n_heads), float(scale), alibi_slopes, _kv(n_heads, n_kv_heads),
                          int(window))
    return out


def cache_tiles(runs: list[tuple[int, int, int, int]], device: torch.device | str) -> torch.Tensor:
    """The tile table of :func:`cache_attention` for runs ``(slot, first_row, n_rows, first_pos)`` of any length: each run
    is cut into tiles of at most 64 rows."""
    tiles = [(s, r + o, min(64, n - o), p + o) for s, r, n, p in runs for o in range(0, n, 64)]
    return torch.tensor(tiles, dtype=torch.int32).reshape(-1, 4).to(device)


def embed_pos(ids: torch.Tensor, pos: torch.Tensor, wte: torch.Tensor, wpe: torch.Tensor | None, out: torch.Tensor) -> torch.Tensor:
    """``out[b] = wte[ids[b]] + wpe[pos[b]]`` with int32 ``ids`` / ``pos`` on the device."""
    ext().embed_pos(ids, pos, wte, wpe, out)
    return out


def argmax_advance(logits: torch.Tensor, ids: torch.Tensor, pos: torch.Tensor | None = None) -> torch.Tensor:
    """``ids[b] = argmax(logits[b])`` (lowest index on ties) and ``pos[b] += 1`` when ``pos`` is given."""
    ext().argmax_advance(logits, ids, pos)
    return ids
