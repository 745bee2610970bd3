"""fp64 references for the fused memory-bound kernels (``csrc/fused_ops.cu``, ``csrc/fp8_ops.cu``) and the bounds they are held to.

Every reference takes the kernel's own bf16 / fp32 / int64 inputs, upcasts them to float64 and computes the op as specified.
The bounds come from what the output format can hold and from the fp32 arithmetic the kernel does, never from a per-test guess.
``EPS32`` is the fp32 machine epsilon 2^-23 (twice the unit roundoff, so every "n operations" count below has a factor 2 of slack).

* bf16 outputs, rule ``bf16_tol``: every element within one bf16 ulp of the fp64 value (round to nearest is half an ulp; the
  other half covers an fp32 intermediate that lands across a rounding boundary) plus an absolute floor equal to the fp32
  error bound of the terms that cancel. Used for LayerNorm ``y`` and ``dx`` (whose references use the kernel's own mean / rstd,
  the backward's inputs, checked on their own against fp64), dlogits, and embedding rows (which are bit-exact: the sum of two
  bf16 values is exact in fp32).
* Reductions, rule ``sum_tol``: ``(depth + 3) * EPS32 * sum|terms|`` where ``depth`` is the longest chain of fp32 additions
  a term passes through in the kernel (per-lane row loop, warp / block partials, one atomic per block) and the 3 covers the
  rounding of a term itself. Used for column sums, dgamma / dbeta, embedding gradients and the CE loss sum. Not relative to
  the result, which can cancel to ~0.
* fp32 row statistics: LN mean ``ln_mean_tol`` and rstd ``ln_rstd_rel_tol`` from the length of the per-lane chain; the CE row
  log-sum-exp ``ce_lse_tol`` from the sum-of-exponentials chain, the ``__expf`` argument rounding and ``__logf``.
* fp8 outputs: bit-exact with ``torch``'s saturating cast where kernel and torch round the same fp32 product (``colsum_quant``,
  ``fp8_quantize_segments``); within one E4M3 ulp of the fp64 value elsewhere (``layernorm_fwd_q8``).
* Optimizer: ``optim_step`` is a line-by-line fp64 transcription of ``optim_update4`` (``csrc/optim_dev.cuh``) with the
  hyper-parameters rounded to fp32 as the kernel receives them. One step from the same state must agree within
  ``OPTIM_ULPS`` fp32 ulps of the largest term of each update line (``--use_fast_math``: approximate sqrt and division, ftz),
  plus the error a line inherits from a plane computed on an earlier line of the same step (the new m in the p update).
* Integers (argmax, #valid, #correct) and the fp64 unigram sum: exact.
"""
from __future__ import annotations

import math

import torch

EPS32 = 2.0 ** -23
F64 = torch.float64
OPTIM_ULPS = 8          # fp32 ulps per optimizer update line: sqrt.approx + div.approx (2 ulp each) + 3 roundings, with slack
FP8_FMAX = {"e4m3": 448.0, "e5m2": 57344.0}


# ------------------------------------------------------------------------------------------------ ulps
def _ulp(x: torch.Tensor, mant_bits: int, emin: int) -> torch.Tensor:
    """Spacing of a binary format with ``mant_bits`` stored mantissa bits and minimum normal exponent ``emin`` at ``|x|``."""
    x = x.to(F64).abs()
    _, e = torch.frexp(x)                          # x = m * 2^e, m in [0.5, 1): floor(log2 x) = e - 1
    e = torch.where(x == 0, torch.full_like(x, emin), torch.clamp(e.to(F64) - 1, min=emin))
    return torch.exp2(e - mant_bits)


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    return _ulp(x, 7, -126)


def fp32_ulp(x: torch.Tensor) -> torch.Tensor:
    return _ulp(x, 23, -126)


def e4m3_ulp(x: torch.Tensor) -> torch.Tensor:
    return _ulp(x, 3, -6)


def e5m2_ulp(x: torch.Tensor) -> torch.Tensor:
    return _ulp(x, 2, -14)


def bf16_tol(ref: torch.Tensor, floor: torch.Tensor | float = 0.0) -> torch.Tensor:
    return bf16_ulp(ref) + floor


def sum_tol(abs_sum: torch.Tensor, depth: int | torch.Tensor) -> torch.Tensor:
    return (depth + 3) * EPS32 * abs_sum


def colsum_depth(T: int) -> int:
    """Longest fp32 addition chain of a column sum over T rows in ``col_reduce_kernel`` / ``colsum_quant_kernel`` /
    ``ln_bwd_fused_kernel``: at most 64 rows per lane, 8 warp partials, one atomic per row strip (at most 528 strips),
    and the initial value."""
    return min(T, 64) + 8 + min(T, 528) + 1


def worst(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> tuple[int, str]:
    """(number of elements over tolerance, a description of the worst one relative to its tolerance)."""
    got, ref = got.to(F64), ref.to(F64)
    tol = torch.as_tensor(tol, dtype=F64, device=ref.device).expand_as(ref)
    err = (got - ref).abs()
    err = torch.where(torch.isnan(got) != torch.isnan(ref), torch.full_like(err, math.inf), torch.nan_to_num(err, nan=0.0))
    bad = int((err > tol).sum())
    ratio = err / tol.clamp(min=1e-300)
    i = int(ratio.reshape(-1).argmax())
    idx = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), ref.shape)) if ref.dim() else ()
    return bad, (f"worst at {idx}: got {got.reshape(-1)[i].item():.9g}, want {ref.reshape(-1)[i].item():.9g}, "
                 f"|err| {err.reshape(-1)[i].item():.3g} vs tol {tol.reshape(-1)[i].item():.3g}")


def assert_within(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor | float, what: str) -> None:
    bad, msg = worst(got, ref, torch.as_tensor(tol, dtype=F64, device=ref.device))
    assert bad == 0, f"{what}: {bad} of {ref.numel()} elements out of tolerance; {msg}"


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_chain(d: int) -> int:
    """Per-row fp32 addition chain of the warp-per-row LayerNorm kernels: 8 elements x ceil(d/256) chunks per lane, then a
    5-level shuffle tree."""
    return 8 * ((d + 255) // 256) + 5


def layernorm_fwd(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor | None, eps: float,
                  mean: torch.Tensor | None = None, rstd: torch.Tensor | None = None):
    """y, mean, rstd over the last dim (two-pass variance, biased). Given ``mean`` / ``rstd`` (e.g. the kernel's), y uses them."""
    xd = x.to(F64)
    mu = xd.mean(-1)
    rs = torch.rsqrt(((xd - mu[..., None]) ** 2).mean(-1) + eps)
    m_use = mu if mean is None else mean.to(F64).reshape(mu.shape)
    r_use = rs if rstd is None else rstd.to(F64).reshape(rs.shape)
    y = (xd - m_use[..., None]) * r_use[..., None] * g.to(F64)
    if b is not None:
        y = y + b.to(F64)
    return y, mu, rs


def ln_mean_tol(x: torch.Tensor) -> torch.Tensor:
    d = x.shape[-1]
    return (ln_chain(d) + 2) * EPS32 * x.to(F64).abs().mean(-1)


def ln_rstd_rel_tol(x: torch.Tensor, rstd: torch.Tensor) -> torch.Tensor:
    """Relative bound of the kernel's rstd: the chain of (x - mean)^2 sums, rsqrtf (2 ulp), and the variance a mean that is
    off by ``ln_mean_tol`` adds (its square over the variance)."""
    d = x.shape[-1]
    mt = ln_mean_tol(x)
    return (ln_chain(d) + 10) * EPS32 + (mt * rstd.to(F64)) ** 2


def ln_fwd_floor(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor | None, mean: torch.Tensor, rstd: torch.Tensor) -> torch.Tensor:
    """fp32 error of ``(x - mean) * rstd * g + b`` (four roundings) for a reference that uses the same mean / rstd."""
    lead = (*x.shape[:-1], 1)
    xh = (x.to(F64) - mean.to(F64).reshape(lead)) * rstd.to(F64).reshape(lead)
    t = (xh * g.to(F64)).abs()
    if b is not None:
        t = t + b.to(F64).abs()
    return 4 * EPS32 * t


def layernorm_bwd(dy: torch.Tensor, x: torch.Tensor, g: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor,
                  dres: torch.Tensor | None = None):
    """dx (+ dres), dgamma, dbeta of ``y = (x - mean) * rstd * g + b`` for the given mean / rstd (the op's inputs), plus the
    fp32 floor of dx (see ``bf16_tol``) and the sum of |terms| of each dgamma / dbeta column."""
    d = x.shape[-1]
    xd, dyd, gd = x.to(F64).reshape(-1, d), dy.to(F64).reshape(-1, d), g.to(F64)
    mu, rs = mean.to(F64).reshape(-1, 1), rstd.to(F64).reshape(-1, 1)
    xh = (xd - mu) * rs
    dyg = dyd * gd
    c1 = dyg.mean(-1, keepdim=True)
    c2 = (dyg * xh).mean(-1, keepdim=True)
    dx = rs * (dyg - c1 - xh * c2)
    if dres is not None:
        dx = dx + dres.to(F64).reshape(-1, d)
    ch = ln_chain(d)
    c1_err = (ch + 2) * EPS32 * dyg.abs().mean(-1, keepdim=True)
    c2_err = (ch + 5) * EPS32 * (dyg * xh).abs().mean(-1, keepdim=True)
    floor = rs * (4 * EPS32 * (dyg.abs() + c1.abs() + (xh * c2).abs()) + c1_err + xh.abs() * c2_err) + 2 * EPS32 * dx.abs()
    dgamma, dbeta = (dyd * xh).sum(0), dyd.sum(0)
    abs_dgamma, abs_dbeta = (dyd * xh).abs().sum(0), dyd.abs().sum(0)
    shape = x.shape
    return dx.reshape(shape), dgamma, dbeta, floor.reshape(shape), abs_dgamma, abs_dbeta


# ------------------------------------------------------------------------------------------------ cross-entropy
def cross_entropy(logits: torch.Tensor, tgt: torch.Tensor, scale: float, unigram: torch.Tensor | None = None) -> dict:
    """Per row of ``logits`` [R, V] (bf16 values, fp64 math): loss (0 for ignored rows), lse, argmax (lowest index on ties),
    dlogits = (softmax - onehot) * scale (zero rows where the target is ignored: < 0 or >= V), the four stats
    (sum loss, #valid, #correct, -sum unigram[target]) and the per-element / per-row tolerances of the kernel's fp32 math."""
    R, V = logits.shape
    x = logits.to(F64)
    t = tgt.to(torch.long)
    valid = (t >= 0) & (t < V)
    tc = torch.where(valid, t, torch.zeros_like(t))
    m = x.max(-1, keepdim=True).values
    e = torch.exp(x - m)
    s = e.sum(-1, keepdim=True)
    lse = (m + torch.log(s)).squeeze(-1)
    p = e / s
    am = (x == m).to(torch.int8).argmax(-1)     # first index of the maximum
    lt = x.gather(1, tc[:, None]).squeeze(-1)
    loss = torch.where(valid, lse - lt, torch.zeros_like(lse))
    onehot = torch.zeros_like(x).scatter_(1, tc[:, None], 1.0) * valid[:, None]
    dl = (p - onehot) * scale * valid[:, None]
    # fp32 error of the kernel: the chain of the sum of exponentials (<= V/256 terms per thread, rescales, 5 + 4 tree levels),
    # __expf's argument rounding (relative EPS32 * |x - max| per term), __logf and the final max + log
    chain = V // 256 + 32
    spread = (p * (m - x)).sum(-1)                        # softmax-weighted |x - max|
    lse_tol = chain * EPS32 + EPS32 * spread + 4 * EPS32 * lse.abs()
    p_rel = chain * EPS32 + EPS32 * (m - x)
    dl_tol = bf16_ulp(dl) + abs(scale) * p * p_rel * valid[:, None] + 2.0 ** -125 * max(1.0, abs(scale))
    correct = valid & (am == t)
    stats = torch.stack([loss.sum(), valid.sum().to(F64), correct.sum().to(F64),
                         (-unigram.to(F64)[tc] * valid).sum() if unigram is not None else torch.zeros((), dtype=F64, device=x.device)])
    loss_tol = ((lse_tol + EPS32 * loss.abs()) * valid).sum()
    return dict(loss=loss, lse=lse, argmax=am, dlogits=dl, stats=stats, valid=valid, lse_tol=lse_tol, dl_tol=dl_tol,
                loss_tol=loss_tol)


# ------------------------------------------------------------------------------------------------ embedding, column sums
def embed_fwd(ids: torch.Tensor, wte: torch.Tensor, wpe: torch.Tensor | None, S: int) -> torch.Tensor:
    """``wte[clamp(ids, 0, V-1)] + wpe[t % S]``: out-of-range ids read row 0 (negative) or row V-1 (too large)."""
    V = wte.shape[0]
    out = wte.to(F64)[ids.clamp(0, V - 1)]
    if wpe is not None:
        out = out + wpe.to(F64)[torch.arange(ids.numel(), device=ids.device) % S]
    return out


def embed_bwd(ids: torch.Tensor, dh: torch.Tensor, V: int, S: int, dwte0: torch.Tensor | None = None,
              dwpe0: torch.Tensor | None = None):
    """(dwte, dwpe, their sum_tol bounds): ``dwte[ids[t]] += dh[t]`` for in-range ids only (others are skipped), ``dwpe[s] +=
    sum_b dh[b*S + s]``. dwte's chain is the number of tokens hitting the row (atomics); dwpe's is the batch (a loop)."""
    d = dh.shape[1]
    dhd = dh.to(F64)
    ok = (ids >= 0) & (ids < V)
    idx = ids[ok]
    dwte = (dwte0.to(F64).clone() if dwte0 is not None else torch.zeros(V, d, dtype=F64, device=dh.device))
    dwte_abs = dwte.abs()
    dwte.index_add_(0, idx, dhd[ok])
    dwte_abs.index_add_(0, idx, dhd[ok].abs())
    cnt = torch.zeros(V, dtype=F64, device=dh.device).index_add_(0, idx, torch.ones_like(idx, dtype=F64))
    B = ids.numel() // S
    per = dhd.view(B, S, d)
    dwpe = per.sum(0) + (dwpe0.to(F64)[:S] if dwpe0 is not None else 0.0)
    dwpe_abs = per.abs().sum(0) + (dwpe0.to(F64)[:S].abs() if dwpe0 is not None else 0.0)
    return dwte, dwpe, sum_tol(dwte_abs, cnt[:, None] + 1), sum_tol(dwpe_abs, B + 1)


def col_sum(dy: torch.Tensor, out0: torch.Tensor | None = None):
    """(out0 + sum_t dy[t, :], its sum_tol bound)."""
    T = dy.shape[0]
    dyd = dy.to(F64)
    base = out0.to(F64) if out0 is not None else torch.zeros(dy.shape[1], dtype=F64, device=dy.device)
    return base + dyd.sum(0), sum_tol(base.abs() + dyd.abs().sum(0), colsum_depth(T))


# ------------------------------------------------------------------------------------------------ fp8
def fp8_round(x: torch.Tensor, fmt: str) -> torch.Tensor:
    """Round-to-nearest-even to E4M3 / E5M2 with saturation to the largest finite value, in fp64 (exact)."""
    mant, emin = (3, -6) if fmt == "e4m3" else (2, -14)
    xd = x.to(F64)
    q = _ulp(xd, mant, emin)
    r = torch.round(xd / q) * q                      # torch.round: half to even
    f = FP8_FMAX[fmt]
    return r.clamp(-f, f)


# ------------------------------------------------------------------------------------------------ optimizer
def _f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


def optim_step(kind: int, p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, hyper: dict,
               grad_mult: float | None = None):
    """One step of ``optim_update4`` in fp64. ``hyper``: first, lr, beta1, beta2, eps, decay, wd (optional, 0 if absent),
    clip, step_size, inv_sqrt_bc2 (rounded to fp32 here, as the binding does). kind 0 = ADOPT, 1 = DecoupledAdamW, 2 = SGD.

    Returns (p, m, v, tol): ``tol[k]`` bounds the kernel's error in plane k after one step from the same state. Each update
    line contributes ``OPTIM_ULPS`` fp32 ulps of its largest term (``_line``), and a line that reads a plane computed on an
    earlier line inherits that plane's error: ADOPT's p reads the new m (``lr * tol_m``), AdamW's p reads the new m and v.
    ADOPT's coupled weight decay (``wd``) is a line of its own, ``G + wd * p``, whose error every later line reads: through
    the normalised gradient (divided by ``max(sqrt v, eps)``) into m, and as ``2 |G|`` times it into v."""
    h = {k: (_f32(val) if isinstance(val, float) and math.isfinite(val) else val) for k, val in hyper.items()}
    P, M, Vv = p.to(F64).clone(), m.to(F64).clone(), v.to(F64).clone()
    gm = _f32(grad_mult) if grad_mult is not None else 1.0
    G = g.to(F64) * gm
    tp, tm, tv = _line(P), _line(M), _line(Vv)
    if kind == 2:
        step = h["lr"] * G
        P1 = P * h["decay"] - step
        tp = _line(P, step, P1)
        P = P1
    elif kind == 0:
        t_g = torch.zeros_like(G)
        if h.get("wd", 0.0):
            G1 = G + h["wd"] * P
            t_g = _line(G, h["wd"] * P, G1)
            G = G1
        if h["first"]:
            Vv = G * G
            tv = _line(Vv) + 2 * G.abs() * t_g
        else:
            ng = G / torch.clamp(torch.sqrt(Vv), min=h["eps"])
            ng = ng.clamp(-h["clip"], h["clip"])
            t_ng = _line(ng) + t_g / torch.clamp(torch.sqrt(Vv), min=h["eps"])   # approximate sqrt and division
            M1 = M + (1.0 - h["beta1"]) * (ng - M)
            tm = _line(M, ng, M1) + (1.0 - h["beta1"]) * t_ng
            P1 = P * h["decay"] - h["lr"] * M1
            tp = _line(P, h["lr"] * M1, P1) + h["lr"] * tm
            V1 = h["beta2"] * Vv + (1.0 - h["beta2"]) * G * G
            tv = _line(Vv, G * G, V1) + (1.0 - h["beta2"]) * 2 * G.abs() * t_g
            P, M, Vv = P1, M1, V1
    else:
        P0 = P * h["decay"]
        M1 = M + (1.0 - h["beta1"]) * (G - M)
        tm = _line(M, G, M1)
        V1 = h["beta2"] * Vv + (1.0 - h["beta2"]) * G * G
        tv = _line(Vv, G * G, V1)
        root = torch.sqrt(V1)
        denom = root * h["inv_sqrt_bc2"] + h["eps"]
        t_denom = _line(denom) + h["inv_sqrt_bc2"] * torch.minimum(tv / (2 * root).clamp(min=1e-300), torch.sqrt(tv))
        upd = h["step_size"] * M1 / denom
        t_upd = _line(upd) + h["step_size"] * (tm / denom + M1.abs() * t_denom / denom ** 2)
        P1 = P0 - upd
        tp = _line(P, P0, upd, P1) + t_upd
        P, M, Vv = P1, M1, V1
    return P, M, Vv, {"p": tp, "m": tm, "v": tv}


def _line(*terms: torch.Tensor) -> torch.Tensor:
    """``OPTIM_ULPS`` fp32 ulps of the largest |term| of one update line, plus as many smallest normals (ftz)."""
    big = terms[0].abs()
    for t in terms[1:]:
        big = torch.maximum(big, t.abs())
    return OPTIM_ULPS * (fp32_ulp(big) + 2.0 ** -126)
