"""fp64 reference of the sm_90a engine's amp_fp8 calls, checked on the engine's own E4M3 / E5M2 operands, and the delayed-scaling
recipe (``photon_b200.train.fp8``) as the oracle of its scale sequence.

Every fp8 GEMM multiplies exact fp8 values, so given the bytes and scales a call actually used, ``A·Bᵀ`` in fp64 is exact up to
fp64 rounding. What is left is the kernel's accumulation, the fp32 epilogue and the output rounding. Each element is held to

    |got − ref| ≤ half-ulp(out dtype, ref) + C_ACC · K · 2^-P_ACC · (|A|·|B|ᵀ) · |alpha / (scale_a · scale_b)| + epilogue terms

and reported by the kernel's 128 x 256 output tile. Quantising producers are the kernels' own fp32 arithmetic (``bf16 · scale``
cast with saturation), so their bytes must match bitwise; the norms' bytes may move one step where the fp64 value sits within
the norm's error bound of a rounding boundary.

Accumulation: fp8 ``wgmma`` on the H100 does not accumulate in fp32. Held to ``K · 2^-24 · (|A|·|B|ᵀ)`` (fp32 accumulation),
the engine's GEMMs miss by up to 200x. Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit over every fp8 GEMM of
``tests/test_fp8_engine_oracle_gpu.py`` (K = 384 .. 16384, the split-K weight gradients at B·S = 16384 included), the largest
error beyond output rounding, in units of ``2^-24 · (|A|·|B|ᵀ)``, does not grow with K:

    K            384    640    768    1152   1360   2304   3072   16384
    bf16 out     9150   9200   8140   18900  12600  2340   12400  -
    fp32 wgrad   -      -      127000 -      -      -      -      4200

so the error is about ``2^-10 · (|A|·|B|ᵀ)`` (an accumulation that keeps roughly 13 to 14 bits, applied per group of products
rather than per element of K) and up to ``2^-7`` in a weight gradient whose products cancel (the key projection's, T = 768).
The bound used is therefore ``C_ACC · 2^-P_ACC · (|A|·|B|ᵀ)`` with ``C_ACC = 1``, the effective precision ``P_ACC = 9`` for
GEMMs with bf16 outputs and ``P_ACC = 6`` for the fp32 weight gradients, about twice the worst measured. Keeping fp32
accumulation would take periodic promotion of the wgmma accumulators to fp32 registers, a kernel change with a speed cost.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from photon_b200.train.fp8 import Fp8Recipe, Fp8TensorMeta

E4M3, E5M2 = 0, 1                      # the operand format codes of photon_b200.ops
DTYPE = {E4M3: torch.float8_e4m3fn, E5M2: torch.float8_e5m2}
FMAX = {E4M3: 448.0, E5M2: 57344.0}
MAXCODE = {E4M3: 0x7E, E5M2: 0x7B}     # largest finite magnitude
TILE = (128, 256)                      # the GEMM kernel's output tile
KBLOCK = 128                           # K per pipeline stage of the fp8 GEMM
EPS32 = 2.0 ** -24
P_ACC, C_ACC = {"bf16": 9, "f32": 6}, 1.0   # effective accumulation precision (see above)
# EPI_GELU_GRAD_Q8 evaluates Φ with the Abramowitz-Stegun erfc (|error| ≤ 1.5e-7, so ≤ 7.5e-8 on Φ) and fast exp / divide
CDF_ABS, PDF_REL = 2e-7, 2.0 ** -20
EPI_BF16, EPI_RESIDUAL, EPI_F32, EPI_MUL, EPI_GELU_GRAD_Q8 = 0, 1, 4, 6, 7


# ------------------------------------------------------------------------------------------------ fp8 bytes
def values(u8: torch.Tensor, fmt: int) -> torch.Tensor:
    """The fp8 values of a byte tensor, in float64 (unscaled)."""
    return u8.contiguous().view(DTYPE[fmt]).double()


def cast(x: torch.Tensor, fmt: int) -> torch.Tensor:
    """Round-to-nearest cast with saturation to ±max-finite (``cvt.rn.satfinite``) of the fp32 values of ``x``; bytes."""
    lim = FMAX[fmt]
    return x.float().clamp(-lim, lim).to(DTYPE[fmt]).view(torch.uint8)


def quantize(x: torch.Tensor, scale: float, fmt: int) -> torch.Tensor:
    """What the producers compute: the fp32 product ``x · scale`` (x bf16, scale fp32), cast with saturation."""
    return cast(x.float() * torch.tensor(scale, dtype=torch.float32, device=x.device), fmt)


def steps(u8: torch.Tensor) -> torch.Tensor:
    """Signed position of each byte on the fp8 number line (adjacent values differ by 1, ±0 are both 0)."""
    v = u8.int()
    return torch.where(v >= 128, -(v & 0x7F), v & 0x7F)


def nonfinite(u8: torch.Tensor, fmt: int) -> torch.Tensor:
    return (u8 & 0x7F) == 0x7F if fmt == E4M3 else (u8 & 0x7C) == 0x7C


def saturated(u8: torch.Tensor, fmt: int) -> torch.Tensor:
    return (u8 & 0x7F) == MAXCODE[fmt]


def byte_errors(got: torch.Tensor, y: torch.Tensor, err: torch.Tensor, fmt: int) -> torch.Tensor:
    """Mask of bytes that are not the cast of the fp64 value ``y``: a byte may be another than ``cast(y)`` only where ``y ± err``
    straddles a rounding boundary, and then only a cast of a value in that interval (one step away, unless ``err`` spans
    several steps: near zero, where the accumulation error exceeds the value); a non-finite byte is always wrong."""
    g = steps(got)
    lo, hi = steps(cast(y - err, fmt)), steps(cast(y + err, fmt))
    return (g < lo) | (g > hi) | nonfinite(got, fmt)


def plant_two_steps(u8: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """A copy of ``u8`` with the byte of the largest ``|y|`` moved two steps towards zero."""
    out = u8.clone()
    i = int(y.abs().argmax())
    out.view(-1)[i] -= 2
    return out


def half_ulp(v: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Half a unit in the last place of ``dtype`` at magnitude ``v`` (float64)."""
    bits = {torch.bfloat16: 8, torch.float32: 24}[dtype]
    tiny = torch.finfo(dtype).tiny
    _, e = torch.frexp(v.abs().clamp_min(tiny))
    return torch.ldexp(torch.ones_like(v), e - bits - 1)


# ------------------------------------------------------------------------------------------------ reports
@dataclass
class Report:
    what: str
    worst: float          # largest |error| / bound
    where: tuple          # its tile (row, column)
    bad_tiles: int        # tiles with an element over its bound

    @property
    def ok(self) -> bool:
        return self.bad_tiles == 0


def tile_report(what: str, err: torch.Tensor, bound: torch.Tensor) -> Report:
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    r = torch.where(torch.isnan(err), math.inf, r)
    if r.dim() == 1:
        r = r[None]
    M, N = r.shape
    tm, tn = -(-M // TILE[0]), -(-N // TILE[1])
    p = torch.zeros(tm * TILE[0], tn * TILE[1], dtype=r.dtype, device=r.device)
    p[:M, :N] = r
    t = p.view(tm, TILE[0], tn, TILE[1]).amax(dim=(1, 3))
    i = int(t.argmax())
    return Report(what, float(t.max()), (i // tn, i % tn), int((t > 1).sum()))


# ------------------------------------------------------------------------------------------------ GEMM
@dataclass
class GemmCall:
    """One ``gemm_fp8`` as the kernel saw it: K-major operands ``a`` [M,K] / ``b`` [N,K] (bytes), their formats and the fp32
    scales they were quantised with, the epilogue inputs and the outputs it wrote (``prev``: an accumulated fp32 output before
    the call)."""
    a: torch.Tensor
    b: torch.Tensor
    a_fmt: int
    b_fmt: int
    sa: float
    sb: float
    epi: int
    out: torch.Tensor | None
    alpha: float = 1.0
    bias: torch.Tensor | None = None
    aux: torch.Tensor | None = None
    prev: torch.Tensor | None = None
    out2: torch.Tensor | None = None
    out8: torch.Tensor | None = None
    q8_scale: float = 1.0
    amax_before: float = 0.0
    amax_after: float = 0.0
    name: str = ""


def accumulation_bound(call: GemmCall) -> tuple[torch.Tensor, torch.Tensor]:
    """(exact de-scaled product ``alpha · A·Bᵀ / (sa · sb)`` + bias, its bound before the epilogue), float64."""
    A, B = values(call.a, call.a_fmt), values(call.b, call.b_fmt)
    d = call.alpha / (call.sa * call.sb)
    z = (A @ B.t()) * d
    mag = (A.abs() @ B.abs().t()) * abs(d)
    bias = call.bias.double() if call.bias is not None else torch.zeros((), dtype=torch.float64, device=z.device)
    # accumulation; the fp32 de-scale factor (three roundings) and the bias add
    p = P_ACC["f32" if call.epi == EPI_F32 else "bf16"]
    err = C_ACC * 2.0 ** -p * mag + 4 * EPS32 * (z.abs() + bias.abs())
    return z + bias, err


def gelu_parts(z: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    cdf = 0.5 * torch.special.erfc(-z / math.sqrt(2.0))
    pdf = torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)
    return cdf, pdf


def gemm_check(call: GemmCall) -> list[Report]:
    """Every output of the call against fp64, by tile; the E4M3 output of ``EPI_GELU_GRAD_Q8`` byte by byte and its amax."""
    z, e = accumulation_bound(call)
    reps = []
    if call.epi in (EPI_BF16, EPI_RESIDUAL, EPI_MUL):
        ref, err = z, e
        if call.epi == EPI_RESIDUAL:
            aux = call.aux.double()
            ref, err = z + aux, e + 2 * EPS32 * (z.abs() + aux.abs())
        elif call.epi == EPI_MUL:
            aux = call.aux.double()
            ref = z * aux
            err = e * aux.abs() + 2 * EPS32 * ref.abs()
        bound = err + half_ulp(ref.abs() + err, torch.bfloat16)
        reps.append(tile_report(f"{call.name} out", (call.out.double() - ref).abs(), bound))
    elif call.epi == EPI_F32:
        prev = call.prev.double() if call.prev is not None else torch.zeros_like(z)
        ref = prev + z
        K = call.a.shape[1]
        # split-K partials and the previous value meet by fp32 red.add: one rounding per split, at most K / 1024 splits
        err = e + (K / 1024 + 2) * EPS32 * (prev.abs() + z.abs() + e)
        bound = err + half_ulp(ref.abs() + err, torch.float32)
        reps.append(tile_report(f"{call.name} out", (call.out.double() - ref).abs(), bound))
    elif call.epi == EPI_GELU_GRAD_Q8:
        cdf, pdf = gelu_parts(z)
        gelu, dgelu = z * cdf, cdf + z * pdf
        pdf_err = PDF_REL * pdf * (1 + z * z)
        # |gelu'| <= 1.13, |gelu''| <= 0.8
        g_err = 1.2 * e + z.abs() * (CDF_ABS + z.abs() * pdf_err) + 4 * EPS32 * gelu.abs()
        d_err = 0.8 * e + CDF_ABS + z.abs() * pdf_err + 4 * EPS32 * (cdf.abs() + (z * pdf).abs())
        reps.append(tile_report(f"{call.name} gelu'", (call.out2.double() - dgelu).abs(),
                                d_err + half_ulp(dgelu.abs() + d_err, torch.bfloat16)))
        y, y_err = gelu * call.q8_scale, g_err * call.q8_scale + 2 * EPS32 * (gelu * call.q8_scale).abs()
        bad = byte_errors(call.out8, y, y_err, E4M3)
        reps.append(tile_report(f"{call.name} gelu E4M3", bad.double(), torch.full_like(y, 0.5)))
        am, am_err = gelu.abs().max(), g_err.max()
        # the running amax: max(before, this call's), the call's within the bound of max |gelu(z)|
        if call.amax_after > call.amax_before:
            miss = abs(call.amax_after - float(am)) / float(am_err)
        else:
            miss = max(0.0, float(am) - call.amax_before) / float(am_err)
        reps.append(Report(f"{call.name} gelu amax", miss, (0, 0), int(miss > 1)))
    else:
        raise ValueError(f"no reference for epilogue {call.epi}")
    return reps


def plant_tile_scale(call: GemmCall, factor: float = 1.01, tile: tuple[int, int] = (0, 0)) -> GemmCall:
    """The call with one output tile of its main output scaled by ``factor``."""
    out = call.out.clone()
    i, j = tile
    v = out[i * TILE[0]:(i + 1) * TILE[0], j * TILE[1]:(j + 1) * TILE[1]]
    v.copy_((v.double() * factor).to(out.dtype))
    return GemmCall(**{**call.__dict__, "out": out})


def plant_dropped_kblock(call: GemmCall, kb: int = 0, tile: tuple[int, int] = (0, 0)) -> GemmCall:
    """The call with the products of one 128-wide K block missing from one output tile (of ``out``, or of the E4M3 output)."""
    i, j = tile
    r, c = slice(i * TILE[0], (i + 1) * TILE[0]), slice(j * TILE[1], (j + 1) * TILE[1])
    k = slice(kb * KBLOCK, (kb + 1) * KBLOCK)
    part = (values(call.a[r, k], call.a_fmt) @ values(call.b[c, k], call.b_fmt).t()) * (call.alpha / (call.sa * call.sb))
    if call.epi == EPI_GELU_GRAD_Q8:
        z, _ = accumulation_bound(call)
        zz = z[r, c] - part
        cdf, _ = gelu_parts(zz)
        out8 = call.out8.clone()
        out8[r, c] = cast(zz * cdf * call.q8_scale, E4M3)
        return GemmCall(**{**call.__dict__, "out8": out8})
    out = call.out.clone()
    v = out[r, c]
    if call.epi == EPI_MUL:
        part = part * call.aux[r, c].double()
    v.copy_((v.double() - part).to(out.dtype))
    return GemmCall(**{**call.__dict__, "out": out})


# ------------------------------------------------------------------------------------------------ producers
def norm_reference(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor | None, eps: float, rms: bool
                   ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(y, bound of the kernel's fp32 y, rstd) of LayerNorm / RMSNorm of bf16 rows in fp64."""
    x = x.double()
    d = x.shape[-1]
    mu = torch.zeros_like(x[..., :1]) if rms else x.mean(-1, keepdim=True)
    xc = x - mu
    rstd = torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)
    g = gamma.double()
    xh = xc * rstd * g
    y = xh + (beta.double() if beta is not None else 0.0)
    # fp32 row sums (mean, variance) over d elements, the fast rsqrt (2^-22.9) and the fp32 multiply-adds
    rel = d * EPS32 + 2.0 ** -20
    err = rel * (xh.abs() + rstd * x.abs().mean(-1, keepdim=True) * g.abs()) + 4 * EPS32 * y.abs()
    return y, err, rstd.squeeze(-1)


def colsum_bound(dy: torch.Tensor, prev: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(prev + Σ_t dy[t], bound of the kernel's fp32 column sums added into ``prev``), float64."""
    d = dy.double()
    T = d.shape[0]
    return prev.double() + d.sum(0), T * EPS32 * (d.abs().sum(0) + prev.double().abs()) + 1e-30


# ------------------------------------------------------------------------------------------------ delayed scaling
def role_formats(n_layers: int) -> list[int]:
    """Formats of the engine's delayed-scaling roles: per block four E4M3 activations, then four E5M2 gradients."""
    return [E4M3 if j < 4 else E5M2 for _ in range(n_layers) for j in range(8)]


class Recipe:
    """The recipe's scale sequence: one :class:`Fp8TensorMeta` per role, fed one amax per training prologue (the max over that
    role's producer calls since the previous one). :meth:`observe` returns the [2, n] fp32 (scale, 1/scale) that follow,
    ``fmax / (m · 2^margin)`` in fp32 with ``m`` the history's max, the scale kept while ``m`` is zero."""

    def __init__(self, formats: list[int], history_len: int = 16, margin: int = 0) -> None:
        rec = Fp8Recipe(margin=margin, amax_history_len=history_len)
        self.formats, self.margin = formats, margin
        self.metas = [Fp8TensorMeta(DTYPE[f], rec) for f in formats]
        self.scale = torch.ones(len(formats), dtype=torch.float32)

    def observe(self, amax: torch.Tensor) -> torch.Tensor:
        a = amax.detach().float().cpu()
        for r, m in enumerate(self.metas):
            m.observe(a[r:r + 1])
            top = max(m.history)
            if 0.0 < top < 3.0e38:
                f32 = lambda v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
                self.scale[r] = f32(FMAX[self.formats[r]]) / (f32(top) * f32(2.0 ** self.margin))
        return torch.stack([self.scale, torch.ones_like(self.scale) / self.scale])


def scale_mismatches(engine: torch.Tensor, recipe: torch.Tensor) -> list[int]:
    """Roles whose (scale, 1/scale) differ bitwise."""
    e, r = engine.detach().float().cpu().contiguous(), recipe.float().contiguous()
    return torch.nonzero((e.view(torch.int32) != r.view(torch.int32)).any(0)).flatten().tolist()


# ------------------------------------------------------------------------------------------------ role wiring
class Producers:
    """Which producer last wrote each fp8 buffer (by device address range), with the scale and role it quantised with and the
    bytes it wrote. A GEMM operand must be read whole from one such write and de-scaled by exactly its scale."""

    def __init__(self) -> None:
        self.writes: list[tuple[int, int, str, int, float, torch.Tensor]] = []   # (start, end, producer, role, scale, bytes)

    def wrote(self, t: torch.Tensor, producer: str, role: int, scale: float, data: torch.Tensor | None = None) -> None:
        lo = t.data_ptr()
        hi = lo + t.numel() * t.element_size()
        self.writes = [w for w in self.writes if w[1] <= lo or w[0] >= hi]     # an overwritten range is no longer the source
        self.writes.append((lo, hi, producer, role, scale, t.clone() if data is None else data))

    def source(self, t: torch.Tensor) -> tuple[str, int, float, torch.Tensor] | None:
        lo = t.data_ptr()
        hi = lo + t.numel() * t.element_size()
        for a, b, producer, role, scale, data in reversed(self.writes):
            if a <= lo and hi <= b and data.numel() == t.numel():
                return producer, role, scale, data
            if a < hi and lo < b:
                return None
        return None


def wiring_errors(what: str, role: int, meta_col: torch.Tensor, source: tuple | None) -> list[str]:
    """An operand read with role ``role`` (``meta_col`` = that role's (scale, 1/scale, amax) when the GEMM ran) must come from one
    producer write of that role, and be de-scaled by exactly the inverse of the scale that write used."""
    if source is None:
        return [f"{what}: no producer wrote this operand"]
    producer, src_role, scale, _ = source
    out = []
    if src_role != role:
        out.append(f"{what}: read as role {role}, written by {producer} as role {src_role}")
    s = torch.tensor(scale, dtype=torch.float32)
    got = meta_col[:2].float().cpu()
    if got[0].view(torch.int32) != s.view(torch.int32) or got[1].view(torch.int32) != (1 / s).view(torch.int32):
        out.append(f"{what}: de-scaled with 1/{float(got[0])!r}, quantised with {scale!r} by {producer}")
    return out


def accumulation_excess(call: GemmCall) -> float:
    """The largest error of the call's main output beyond its output rounding, in units of ``2^-24 · (|A|·|B|ᵀ)`` de-scaled
    (plus twice the previous value of an accumulated output, whose fp32 add is not the accumulation): what the accumulation
    measurably lost (``EPI_BF16`` / ``EPI_RESIDUAL`` / ``EPI_F32`` / ``EPI_MUL`` only)."""
    A, B = values(call.a, call.a_fmt), values(call.b, call.b_fmt)
    d = call.alpha / (call.sa * call.sb)
    z = (A @ B.t()) * d + (call.bias.double() if call.bias is not None else 0.0)
    mag = (A.abs() @ B.abs().t()) * abs(d)
    if call.epi == EPI_RESIDUAL:
        z = z + call.aux.double()
    elif call.epi == EPI_MUL:
        z, mag = z * call.aux.double(), mag * call.aux.double().abs()
    elif call.epi == EPI_F32 and call.prev is not None:
        z = z + call.prev.double()
        mag = mag + 2 * call.prev.double().abs()     # the fp32 red.add into the previous value is not the accumulation
    elif call.epi not in (EPI_BF16, EPI_F32):
        return 0.0
    dt = torch.float32 if call.epi == EPI_F32 else torch.bfloat16
    ex = ((call.out.double() - z).abs() - half_ulp(z, dt)).clamp_min(0) / (EPS32 * mag).clamp_min(1e-300)
    return float(ex.max())
