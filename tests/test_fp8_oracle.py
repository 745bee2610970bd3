"""CPU rehearsal of ``fp8_oracle``: the references accept a kernel-like fp32 computation on synthetic fp8 captures, and every
planted error is flagged."""
import math

import pytest
import torch

import fp8_oracle as FO


def _operand(shape, fmt, g, scale=1.0):
    x = torch.randn(*shape, generator=g) * scale
    s = FO.FMAX[fmt] / float(x.abs().max())
    return FO.quantize(x.bfloat16(), s, fmt), s


def _kernel_like(A8, B8, a_fmt, b_fmt, sa, sb, alpha=1.0):
    """fp32 accumulation over 32-wide K steps of exact fp8 products, de-scaled in fp32 (what the wgmma epilogue does)."""
    A, B = FO.values(A8, a_fmt).float(), FO.values(B8, b_fmt).float()
    acc = torch.zeros(A.shape[0], B.shape[0])
    for k in range(0, A.shape[1], 32):
        acc += A[:, k:k + 32] @ B[:, k:k + 32].t()
    d = torch.tensor(alpha, dtype=torch.float32) * (1 / torch.tensor(sa, dtype=torch.float32)) * (1 / torch.tensor(sb, dtype=torch.float32))
    return acc * d


def _call(epi, M=200, N=328, K=384, seed=0):
    g = torch.Generator().manual_seed(seed)
    a_fmt = FO.E5M2 if epi in (FO.EPI_F32, FO.EPI_MUL) else FO.E4M3
    a8, sa = _operand((M, K), a_fmt, g)
    b8, sb = _operand((N, K), FO.E4M3, g)
    acc = _kernel_like(a8, b8, a_fmt, FO.E4M3, sa, sb)
    bias = torch.randn(N, generator=g) if epi != FO.EPI_F32 else None
    v = acc + bias if bias is not None else acc
    kw = {}
    if epi == FO.EPI_BF16:
        out = v.bfloat16()
    elif epi == FO.EPI_RESIDUAL:
        kw["aux"] = torch.randn(M, N, generator=g).bfloat16()
        out = (v + kw["aux"].float()).bfloat16()
    elif epi == FO.EPI_MUL:
        kw["aux"] = torch.rand(M, N, generator=g).bfloat16()
        out = (v * kw["aux"].float()).bfloat16()
    elif epi == FO.EPI_F32:
        kw["prev"] = torch.randn(M, N, generator=g) * 0.1
        out = kw["prev"] + v
    else:
        z = v.double()
        cdf, pdf = FO.gelu_parts(z)
        q8s = 448.0 / float((z * cdf).abs().max()) * 0.7
        kw.update(out2=(cdf + z * pdf).float().bfloat16(), out8=FO.cast((z * cdf).float() * q8s, FO.E4M3), q8_scale=q8s,
                  amax_after=float((z * cdf).float().abs().max()))
        out = None
    return FO.GemmCall(a8, b8, a_fmt, FO.E4M3, sa, sb, epi, out, bias=bias, name=f"epi {epi}", **kw)


EPIS = [FO.EPI_BF16, FO.EPI_RESIDUAL, FO.EPI_MUL, FO.EPI_F32, FO.EPI_GELU_GRAD_Q8]


def _flagged(call):
    return not all(r.ok for r in FO.gemm_check(call))


@pytest.mark.parametrize("epi", EPIS)
def test_reference_accepts_fp32_accumulation(epi):
    reps = FO.gemm_check(_call(epi))
    assert all(r.ok for r in reps), [(r.what, r.worst) for r in reps]
    assert max(r.worst for r in reps) < 1


@pytest.mark.parametrize("epi", [FO.EPI_BF16, FO.EPI_RESIDUAL, FO.EPI_MUL, FO.EPI_F32])
def test_plants_in_the_output_are_flagged(epi):
    c = _call(epi)
    if epi != FO.EPI_F32:   # the weight gradients' bound (2^-6 of Σ|a·b|) is wider than 1 % of their largest elements
        assert _flagged(FO.plant_tile_scale(c, 1.01, (1, 0)))
    assert _flagged(FO.plant_dropped_kblock(c, kb=2, tile=(0, 1)))
    g = torch.Generator().manual_seed(5)
    _, s_other = _operand((c.a.shape[0], 64), c.a_fmt, g, scale=1.7)
    assert _flagged(FO.GemmCall(**{**c.__dict__, "sa": s_other}))   # de-scaled with another role's scale


def test_plants_in_the_e4m3_epilogue_are_flagged():
    c = _call(FO.EPI_GELU_GRAD_Q8)
    assert _flagged(FO.plant_dropped_kblock(c, kb=1, tile=(1, 1)))
    z, _ = FO.accumulation_bound(c)
    assert _flagged(FO.GemmCall(**{**c.__dict__, "out8": FO.plant_two_steps(c.out8, z * FO.gelu_parts(z)[0])}))
    assert _flagged(FO.GemmCall(**{**c.__dict__, "amax_after": c.amax_after * 1.01}))


def test_cast_saturates_and_steps():
    x = torch.tensor([1e9, -1e9, 448.0 * 1.05, 500.0, 0.0, -0.0, 1.0], dtype=torch.float32)
    b = FO.cast(x, FO.E4M3)
    assert b[:4].tolist() == [0x7E, 0xFE, 0x7E, 0x7E] and not bool(FO.nonfinite(b, FO.E4M3).any())
    assert FO.cast(torch.tensor([1e9, -7e4]), FO.E5M2).tolist() == [0x7B, 0xFB]
    assert bool(FO.saturated(b[:4], FO.E4M3).all())
    v = torch.arange(-126, 127, dtype=torch.int32)
    u = torch.where(v < 0, 128 - v, v).to(torch.uint8)
    assert torch.equal(FO.steps(u), v)
    vals = FO.values(u, FO.E4M3)
    assert bool((vals[1:] >= vals[:-1]).all())   # the step order is the value order


def test_norm_bytes_allow_one_step_at_boundaries_only():
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(64, 384, generator=g) * 3 + 1).bfloat16()
    gamma, beta = torch.rand(384, generator=g) + 0.5, torch.randn(384, generator=g) * 0.1
    y, err, rstd = FO.norm_reference(x, gamma, beta, 1e-5, rms=False)
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    yf = (xf - mu) * torch.rsqrt(((xf - mu) ** 2).mean(-1, keepdim=True) + 1e-5) * gamma + beta   # fp32, as the kernel
    s = 448.0 / float(y.abs().max())
    got = FO.cast(yf * s, FO.E4M3)
    assert not bool(FO.byte_errors(got, y * s, err * s, FO.E4M3).any())
    assert torch.allclose(rstd, torch.rsqrt(((xf - mu) ** 2).mean(-1) + 1e-5).double(), rtol=1e-6)
    bad = FO.plant_two_steps(got, y)
    assert bool(FO.byte_errors(bad, y * s, err * s, FO.E4M3).any())


def test_producers_and_wiring():
    p = FO.Producers()
    buf = torch.zeros(1024, dtype=torch.uint8)
    w = buf[:512]
    w.copy_(torch.arange(512) % 200)
    p.wrote(w, "colsum_quant", 5, 3.0)
    s3 = torch.tensor(3.0)
    col = torch.stack([s3, 1 / s3, torch.tensor(0.0)])
    src = p.source(buf[:512].view(16, 32))
    assert src[1] == 5 and not FO.wiring_errors("x", 5, col, src)
    assert FO.wiring_errors("x", 6, col, src)                               # another role
    assert FO.wiring_errors("x", 5, torch.stack([s3 * 1.5, 1 / (s3 * 1.5), s3]), src)   # another scale
    p.wrote(buf[256:768], "norm", 1, 2.0)                                   # overwritten in part: no longer one source
    assert p.source(buf[:512]) is None and p.source(buf[256:768])[1] == 1


def _engine_ring(amaxes, formats, H, margin):
    """The delayed-scaling kernel's arithmetic: an H-slot ring, max over it, fmax / (m · 2^margin) rounded to nearest in fp32."""
    n = len(formats)
    hist, scale, out = torch.zeros(n, H), torch.ones(n), []
    fmax = torch.tensor([FO.FMAX[f] for f in formats], dtype=torch.float32)
    for k, a in enumerate(amaxes):
        hist[:, k % H] = a
        m = hist.max(1).values
        ok = (m > 0) & (m < 3e38)
        scale = torch.where(ok, fmax / (m * 2.0 ** margin), scale)
        out.append(torch.stack([scale, 1 / scale]))
    return out


@pytest.mark.parametrize("H,margin", [(16, 0), (4, 1)])
def test_recipe_matches_the_ring_and_flags_a_short_history(H, margin):
    formats = FO.role_formats(2)
    g = torch.Generator().manual_seed(H)
    amaxes = [torch.zeros(len(formats))] + [torch.rand(len(formats), generator=g) * (50.0 if k == 4 else 1.0) for k in range(24)]
    ring = _engine_ring(amaxes, formats, H, margin)
    rec, short = FO.Recipe(formats, H, margin), FO.Recipe(formats, H - 1, margin)
    missed = False
    for k, a in enumerate(amaxes):
        assert not FO.scale_mismatches(ring[k], rec.observe(a)), k
        missed |= bool(FO.scale_mismatches(ring[k], short.observe(a)))
    assert missed
    # the spike holds for exactly H prologues
    held = torch.stack([r[0] for r in ring[5:5 + H]])
    assert torch.equal(held, held[:1].expand_as(held)) and bool((ring[5 + H][0] > held[0]).all())


def test_tile_report_locates_the_tile():
    err, bound = torch.zeros(300, 600, dtype=torch.float64), torch.ones(300, 600, dtype=torch.float64)
    err[260, 530] = 3.0
    r = FO.tile_report("x", err, bound)
    assert (r.where, r.bad_tiles, r.worst) == ((2, 2), 1, 3.0)
    assert FO.tile_report("nan", torch.full((2, 2), math.nan, dtype=torch.float64), bound[:2, :2]).bad_tiles == 1
