"""The fused memory-bound kernels (``csrc/fused_ops.cu``, ``csrc/fp8_ops.cu``) against the fp64 references of ``fused_oracle``, on
every dispatch path, with guard bands around every output buffer and a second run that must give the same bits (except where
the kernel accumulates with float atomics). The bound each output is held to is stated in ``fused_oracle``'s docstring."""
import math

import pytest
import torch

import fused_oracle as fo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
F64 = torch.float64
PAD = 64                                    # guard elements on each side of an output (keeps 16-byte alignment for any dtype)
SENTINEL = {torch.bfloat16: -1234.0, torch.float32: -7777.0, torch.uint8: 0xA5, torch.int32: -5}


def _ops():
    from photon_b200 import ops

    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, scale=1.0, offset=0.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device=DEV, generator=_gen(seed)) * scale + offset).to(dtype)


def _guarded(shape, dtype, init=None):
    """(whole buffer, view of ``shape`` inside it): PAD sentinel elements before and after; the view holds ``init`` or sentinel."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * PAD,), SENTINEL[dtype], dtype=dtype, device=DEV)
    view = buf[PAD:PAD + n].view(shape)
    if init is not None:
        view.copy_(init)
    return buf, view


def _guard_intact(buf, what):
    n = buf.numel() - 2 * PAD
    want = torch.full((PAD,), SENTINEL[buf.dtype], dtype=buf.dtype, device=DEV)
    assert torch.equal(buf[:PAD], want) and torch.equal(buf[PAD + n:], want), f"{what}: wrote outside its buffer"


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else (torch.uint8 if t.element_size() == 1 else torch.int32))


def _same_bits(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f"{what}: second run differs in {(_bits(a) != _bits(b)).sum().item()} elements"


# =============================================================================================== cross-entropy
def _ce_case(R, V, scale, seed):
    """logits with ignored (-100, >= V), edge (0, V-1) targets and two constant rows (argmax ties -> index 0)."""
    x = _randn(R, V, seed=seed, scale=scale)
    tgt = torch.randint(0, V, (R,), device=DEV, generator=_gen(seed + 1))
    if R >= 8:
        tgt[:6] = torch.tensor([-100, V, 0, V - 1, V + 7, -1], device=DEV)
        x[6] = 0.75
        x[7] = -3.0
        tgt[6], tgt[7] = 0, 1           # row 6: tie won by index 0 (correct); row 7: not the first maximum (wrong)
    else:
        tgt[0] = V - 1
    uni = torch.log_softmax(torch.randn(V, device=DEV, generator=_gen(seed + 2)), -1)
    return x, tgt, uni


def _ce_check(work, x, tgt, uni, gs, stats, lse, what, write_grad=True):
    """Chunked fp64 reference (the largest case is 4096 x 128256): row_lse, dlogits, row sums of dlogits, then the stats."""
    R, V = x.shape
    chunk = max(1, (1 << 26) // V)
    loss_sum, loss_tol, abs_uni, valid_n, correct_n = 0.0, 0.0, 0.0, 0, 0
    for lo in range(0, R, chunk):
        hi = min(R, lo + chunk)
        ref = fo.cross_entropy(x[lo:hi], tgt[lo:hi], gs, uni)
        fo.assert_within(lse[lo:hi], ref["lse"], ref["lse_tol"], f"{what} row_lse rows {lo}:{hi}")
        if write_grad:
            got = work[lo:hi].to(F64)
            fo.assert_within(got, ref["dlogits"], ref["dl_tol"], f"{what} dlogits rows {lo}:{hi}")
            rs = got.sum(-1)
            fo.assert_within(rs, torch.zeros_like(rs), ref["dl_tol"].sum(-1), f"{what} dlogits row sums rows {lo}:{hi}")
        loss_sum += ref["stats"][0].item()
        loss_tol += ref["loss_tol"].item()
        valid_n += int(ref["stats"][1].item())
        correct_n += int(ref["stats"][2].item())
        abs_uni += ref["stats"][3].item()
    s = stats.tolist()
    assert abs(s[0] - loss_sum) <= loss_tol + R * 2.0 ** -52 * abs(loss_sum), f"{what} stats[0] {s[0]!r} vs {loss_sum!r} (tol {loss_tol:.3g})"
    assert s[1] == valid_n, f"{what} #valid {s[1]} vs {valid_n}"
    assert s[2] == correct_n, f"{what} #correct {s[2]} vs {correct_n}"
    assert abs(s[3] - abs_uni) <= R * 2.0 ** -52 * abs(abs_uni) + 1e-300, f"{what} unigram sum {s[3]!r} vs {abs_uni!r}"


def _ce_run(x, tgt, uni, gs, write_grad=True, ld=None):
    """Run the kernel on a guarded copy of ``x`` (row stride ``ld``); returns (work view, buffers, stats, lse)."""
    R, V = x.shape
    ld = ld or V
    buf, full = _guarded((R, ld), torch.bfloat16)
    work = full[:, :V]
    work.copy_(x)
    lbuf, lse = _guarded((R,), torch.float32)
    stats = torch.zeros(4, dtype=F64, device=DEV)
    _ops().cross_entropy(work, tgt, gs, write_grad, stats, lse, uni)
    return work, full, buf, stats, lse, lbuf


@pytest.mark.parametrize("scale", [1.0, 30.0])
@pytest.mark.parametrize("R", [1, 300, 4096])
@pytest.mark.parametrize("V", [8, 16, 2048, 50368, 128256])
def test_cross_entropy(V, R, scale):
    """V <= 50368: ``ce_smem_kernel`` (the row staged in shared memory by bulk copies). V = 128256 (a row over 200 KiB):
    ``ce_kernel`` (two passes over HBM). Loss, row lse, in-place dlogits, the four stats, argmax ties."""
    x, tgt, uni = _ce_case(R, V, scale, seed=V + R)
    gs = 1.0 / 123.0
    what = f"cross_entropy V={V} rows={R} scale={scale}"
    work, full, buf, stats, lse, lbuf = _ce_run(x, tgt, uni, gs)
    torch.cuda.synchronize()
    _guard_intact(buf, what + " logits")
    _guard_intact(lbuf, what + " row_lse")
    _ce_check(work, x, tgt, uni, gs, stats, lse, what)
    work2, _, _, stats2, lse2, _ = _ce_run(x, tgt, uni, gs)
    _same_bits(work2, work, what + " dlogits")
    _same_bits(lse2, lse, what + " row_lse")
    assert stats2[1:3].tolist() == stats[1:3].tolist()


@pytest.mark.parametrize("V", [50368, 128256])
def test_cross_entropy_strided_rows_and_no_grad(V):
    """``logits[:, :V]`` of a ``[rows, V + 64]`` buffer (row stride != V) on both kernels (``ce_smem_kernel`` for 50368,
    ``ce_kernel`` for 128256): the 64 padding columns stay untouched. ``write_grad=False`` (the scoring path) leaves the logits
    bitwise unchanged and still produces row_lse and the stats."""
    R = 300
    x, tgt, uni = _ce_case(R, V, 2.0, seed=7)
    gs = 0.01
    what = f"cross_entropy V={V} ld={V + 64}"
    work, full, buf, stats, lse, _ = _ce_run(x, tgt, uni, gs, ld=V + 64)
    torch.cuda.synchronize()
    _guard_intact(buf, what)
    assert torch.equal(_bits(full[:, V:]), _bits(torch.full((R, 64), SENTINEL[torch.bfloat16], dtype=torch.bfloat16, device=DEV))), \
        f"{what}: padding columns written"
    _ce_check(work, x, tgt, uni, gs, stats, lse, what)
    work, full, buf, stats, lse, _ = _ce_run(x, tgt, uni, gs, write_grad=False, ld=V + 64)
    _same_bits(work, x, f"cross_entropy V={V} write_grad=False logits")
    _ce_check(work, x, tgt, uni, gs, stats, lse, f"cross_entropy V={V} write_grad=False", write_grad=False)


@pytest.mark.parametrize("V", [50368, 128256])
def test_cross_entropy_all_targets_ignored(V):
    """A batch with no valid target (``ce_smem_kernel`` / ``ce_kernel``): zero loss and counts, all-zero gradient rows, a finite
    lse that still matches fp64."""
    R = 300
    x, _, uni = _ce_case(R, V, 1.0, seed=11)
    tgt = torch.full((R,), -100, dtype=torch.long, device=DEV)
    tgt[::2] = V
    work, _, _, stats, lse, _ = _ce_run(x, tgt, uni, 1.0)
    assert stats.tolist() == [0.0, 0.0, 0.0, 0.0]
    assert torch.isfinite(lse).all()
    assert not _bits(work).any(), "ignored rows must get an all-zero gradient"
    _ce_check(work, x, tgt, uni, 1.0, stats, lse, f"cross_entropy V={V} all ignored")


@pytest.mark.parametrize("V", [2048, 50368, 128256])
def test_ce_argmax_agrees_with_argmax_advance(V):
    """Scoring reports hits with ``argmax_advance``, training with the CE argmax (``ce_smem_kernel`` / ``ce_kernel``): both must
    pick the first maximum, also on ties and on a ``[:, :V]`` slice of a wider buffer."""
    ops = _ops()
    R = 64
    wide = _randn(R, V + 64, seed=V, scale=3.0)
    x = wide[:, :V]
    x[0] = 1.0                                              # every index ties
    x[1, 5] = x[1, V - 3] = 40.0                           # two separated maxima
    x[2, V - 1] = 40.0                                     # maximum in the last column
    x[3, 8:16] = 40.0                                      # a whole 16-byte vector of maxima
    ref = fo.cross_entropy(x, torch.zeros(R, dtype=torch.long, device=DEV), 1.0)["argmax"]
    assert ref[0].item() == 0 and ref[1].item() == 5 and ref[2].item() == V - 1 and ref[3].item() == 8
    ids = torch.full((R,), -1, dtype=torch.int32, device=DEV)
    ops.argmax_advance(x, ids)
    assert torch.equal(ids.long(), ref), f"argmax_advance V={V}: rows {torch.nonzero(ids.long() != ref).flatten().tolist()} differ"
    for shift, want in ((0, R), (1, 0)):                    # target = first maximum: all correct; the next index: none
        stats = torch.zeros(4, dtype=F64, device=DEV)
        ops.cross_entropy(x.clone(), (ref + shift) % V, 1.0, False, stats)
        assert stats[2].item() == want, f"CE argmax V={V} shift {shift}: #correct {stats[2].item()} != {want}"


# =============================================================================================== LayerNorm
LN_SHAPES = [(d, T) for d in (768, 1024, 1032) for T in (1, 7, 9, 8192)] + \
            [(d, T) for d in (64, 200, 256, 1000, 2048, 2560, 3072, 4096) for T in (9, 8192)]
LN_EPS = 1e-5


def _ln_inputs(T, d, seed):
    """Rows with a large common offset (mean 30, std 0.5): a one-pass variance loses most of its digits there."""
    x = _randn(T, d, seed=seed, scale=0.5, offset=30.0)
    g = torch.rand(d, device=DEV, generator=_gen(seed + 1)) + 0.5
    b = torch.randn(d, device=DEV, generator=_gen(seed + 2)) * 0.1
    return x, g, b


def _ln_fwd(x, g, b):
    T, d = x.shape
    ybuf, y = _guarded((T, d), torch.bfloat16)
    mbuf, mean = _guarded((T,), torch.float32)
    rbuf, rstd = _guarded((T,), torch.float32)
    gbuf, gv = _guarded((d,), torch.float32, g)
    bv = _guarded((d,), torch.float32, b)[1] if b is not None else None
    _ops().layernorm_fwd(x, gv, bv, y, mean, rstd, LN_EPS)
    for buf, n in ((ybuf, "y"), (mbuf, "mean"), (rbuf, "rstd")):
        _guard_intact(buf, f"layernorm_fwd {n}")
    return y, mean, rstd


def _check_stats(x, mean, rstd, what):
    _, mu, rs = fo.layernorm_fwd(x, torch.ones(x.shape[-1], device=DEV), None, LN_EPS)
    fo.assert_within(mean, mu, fo.ln_mean_tol(x), f"{what} mean")
    fo.assert_within(rstd.to(F64) / rs, torch.ones_like(rs), fo.ln_rstd_rel_tol(x, rs), f"{what} rstd / fp64 rstd")


@pytest.mark.parametrize("d,T", LN_SHAPES)
def test_layernorm(d, T):
    """Forward (``ln_fwd_kernel``) with and without beta; backward on both paths: with dgamma and/or dbeta and d <= 1024 the
    one-pass ``ln_bwd_fused_kernel`` (persistent: at T = 8192 every warp loops over several rows), otherwise
    ``ln_bwd_dx_kernel`` + ``col_reduce`` (and always for dx only). Variants: dres / no dres, dgamma only, dbeta only, dgamma
    and dbeta accumulated into non-zero values."""
    ops = _ops()
    x, g, b = _ln_inputs(T, d, seed=d * 31 + T)
    what = f"layernorm d={d} T={T}"
    for beta in (b, None):
        tag = f"{what} beta={'yes' if beta is not None else 'None'}"
        y, mean, rstd = _ln_fwd(x, g, beta)
        _check_stats(x, mean, rstd, tag)
        ref, _, _ = fo.layernorm_fwd(x, g, beta, LN_EPS, mean=mean, rstd=rstd)
        fo.assert_within(y, ref, fo.bf16_tol(ref, fo.ln_fwd_floor(x, g, beta, mean, rstd)), f"{tag} y")
        y2, mean2, rstd2 = _ln_fwd(x, g, beta)
        _same_bits(y2, y, f"{tag} y")
        _same_bits(mean2, mean, f"{tag} mean")
        _same_bits(rstd2, rstd, f"{tag} rstd")
    dy = _randn(T, d, seed=d + T + 5)
    dres = _randn(T, d, seed=d + T + 6)
    for use_dres, want_dg, want_db in ((True, True, True), (False, True, False), (True, False, True), (False, False, False)):
        dr = dres if use_dres else None
        tag = f"{what} dres={use_dres} dgamma={want_dg} dbeta={want_db}"
        ref_dx, ref_dg, ref_db, floor, abs_dg, abs_db = fo.layernorm_bwd(dy, x, g, mean, rstd, dr)
        outs = []
        for _ in range(2):
            dxbuf, dx = _guarded((T, d), torch.bfloat16)
            g0 = torch.randn(d, device=DEV, generator=_gen(d)) if want_dg else None
            b0 = torch.randn(d, device=DEV, generator=_gen(d + 1)) if want_db else None
            dgbuf, dg = _guarded((d,), torch.float32, g0) if want_dg else (None, None)
            dbbuf, db = _guarded((d,), torch.float32, b0) if want_db else (None, None)
            ops.layernorm_bwd(dy, x, g, mean, rstd, dr, dx, dg, db)
            for buf, n in ((dxbuf, "dx"), (dgbuf, "dgamma"), (dbbuf, "dbeta")):
                if buf is not None:
                    _guard_intact(buf, f"{tag} {n}")
            fo.assert_within(dx, ref_dx, fo.bf16_tol(ref_dx, floor), f"{tag} dx")
            depth = fo.colsum_depth(T)
            if want_dg:
                fo.assert_within(dg, g0.to(F64) + ref_dg, fo.sum_tol(g0.to(F64).abs() + abs_dg, depth), f"{tag} dgamma")
            if want_db:
                fo.assert_within(db, b0.to(F64) + ref_db, fo.sum_tol(b0.to(F64).abs() + abs_db, depth), f"{tag} dbeta")
            outs.append(dx)
        _same_bits(outs[1], outs[0], f"{tag} dx")


@pytest.mark.parametrize("d", [64, 200, 768, 1000, 1032, 2048, 2560, 4096])
@pytest.mark.parametrize("with_beta", [True, False])
def test_layernorm_fwd_q8(d, with_beta):
    """``ln_fwd_q8_kernel``: E4M3 bytes within one E4M3 ulp of the fp64 LayerNorm times the scale (some values saturate at
    448), mean / rstd as the bf16 forward, and the amax of the unscaled fp32 output."""
    T = 1001
    x, g, b = _ln_inputs(T, d, seed=d + 3)
    beta = b if with_beta else None
    ref, mu, rs = fo.layernorm_fwd(x, g, beta, LN_EPS)
    amax_ref = ref.abs().max().item()
    s = 448.0 / amax_ref * 1.25
    meta = torch.zeros(3, 2, device=DEV)
    meta[0], meta[1] = s, 1.0 / s
    ybuf, y8 = _guarded((T, d), torch.uint8)
    mean, rstd = torch.empty(T, device=DEV), torch.empty(T, device=DEV)
    _ops().layernorm_fwd_q8(x, g, beta, y8, mean, rstd, LN_EPS, meta, 1)
    what = f"layernorm_fwd_q8 d={d} beta={with_beta}"
    _guard_intact(ybuf, what)
    _check_stats(x, mean, rstd, what)
    want = (ref * float(torch.tensor(s, dtype=torch.float32))).clamp(-448.0, 448.0)
    got = y8.view(torch.float8_e4m3fn).to(F64)
    fo.assert_within(got, want, fo.e4m3_ulp(want), f"{what} E4M3 bytes")
    err = (ref.abs() * fo.ln_rstd_rel_tol(x, rs)[:, None] + fo.ln_mean_tol(x)[:, None] * rs[:, None] * g.to(F64)
           + fo.ln_fwd_floor(x, g, beta, mu, rs)).max().item()
    assert abs(meta[2, 1].item() - amax_ref) <= err, f"{what} amax {meta[2, 1].item()!r} vs {amax_ref!r} (tol {err:.3g})"
    assert meta[2, 0].item() == 0.0


def test_layernorm_rejects_unsupported_rows():
    """d % 8 != 0 and d > 4096 raise in both directions instead of launching."""
    ops = _ops()
    for d in (100, 4104):
        x = _randn(4, d, seed=1)
        g = torch.ones(d, device=DEV)
        y, m, r = torch.empty_like(x), torch.empty(4, device=DEV), torch.empty(4, device=DEV)
        with pytest.raises(RuntimeError):
            ops.layernorm_fwd(x, g, None, y, m, r)
        with pytest.raises(RuntimeError):
            ops.layernorm_bwd(x, x, g, m, r, None, y, None, None)


# =============================================================================================== column sums
COL_T = [1, 7, 25, 33, 1000, 16384]
COL_D = [8, 264, 2304, 3080]


@pytest.mark.parametrize("T", COL_T)
@pytest.mark.parametrize("d", COL_D)
def test_col_sum(d, T):
    """``col_reduce_kernel`` without x (bias gradients): the 4-row unrolled loop and its tail, a strided ``dy`` ([:, :d] of a
    wider buffer) and accumulation into non-zero values."""
    dy = _randn(T, d + 24, seed=d * 7 + T)[:, :d]
    out0 = torch.randn(d, device=DEV, generator=_gen(T))
    buf, out = _guarded((d,), torch.float32, out0)
    _ops().col_sum(dy, out)
    what = f"col_sum d={d} T={T}"
    _guard_intact(buf, what)
    ref, tol = fo.col_sum(dy, out0)
    fo.assert_within(out, ref, tol, what)


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
@pytest.mark.parametrize("T", COL_T)
@pytest.mark.parametrize("d", COL_D)
def test_colsum_quant(d, T, fmt):
    """``colsum_quant_kernel``: column sums into non-zero values plus the fp8 copy of a strided ``dy`` into a ``y8`` with
    ``ld8 != d``. The bytes equal ``torch``'s saturating cast of the same fp32 product (the scale makes the largest values
    saturate); the padding bytes stay untouched; amax is the exact max |dy|."""
    ops = _ops()
    dt = torch.float8_e4m3fn if fmt == "e4m3" else torch.float8_e5m2
    dy = _randn(T, d + 24, seed=d * 11 + T, scale=3e-4)[:, :d]
    amax = dy.float().abs().max().item()
    s = fo.FP8_FMAX[fmt] / amax * 1.25
    meta = torch.zeros(3, 1, device=DEV)
    meta[0], meta[1] = s, 1.0 / s
    out0 = torch.randn(d, device=DEV, generator=_gen(T))
    what = f"colsum_quant {fmt} d={d} T={T}"
    runs = []
    for _ in range(2):
        meta[2] = 0.0
        obuf, out = _guarded((d,), torch.float32, out0)
        ybuf, yfull = _guarded((T, d + 16), torch.uint8)
        ops.colsum_quant(dy, out, yfull[:, :d], ops.E4M3 if fmt == "e4m3" else ops.E5M2, meta, 0)
        _guard_intact(obuf, what + " out_sum")
        _guard_intact(ybuf, what + " y8")
        assert (yfull[:, d:] == SENTINEL[torch.uint8]).all(), f"{what}: y8 padding columns written"
        ref, tol = fo.col_sum(dy, out0)
        fo.assert_within(out, ref, tol, what + " column sums")
        want = (dy.float() * meta[0, 0]).clamp(-fo.FP8_FMAX[fmt], fo.FP8_FMAX[fmt]).to(dt).view(torch.uint8)
        y8 = yfull[:, :d]
        assert torch.equal(y8, want), f"{what}: {(y8 != want).sum().item()} of {y8.numel()} bytes differ from torch's cast"
        assert meta[2, 0].item() == amax, f"{what} amax {meta[2, 0].item()!r} vs {amax!r}"
        runs.append(y8.clone())
    assert torch.equal(runs[0], runs[1]), f"{what}: second run differs"


def test_fp8_quantize_segments_bytes_exact():
    """``seg_amax_kernel`` + ``seg_quant_kernel``: per-segment current scaling; bytes identical to torch's saturating cast
    with the scale the kernel chose; the bytes between segments untouched."""
    ops = _ops()
    sizes, offs, total = [4096, 768 * 264, 8], [], 0
    for n in sizes:
        offs.append(total)
        total += n + 64
    src = torch.zeros(total, dtype=torch.bfloat16, device=DEV)
    for i, (o, n) in enumerate(zip(offs, sizes)):
        src[o:o + n] = _randn(n, seed=i, scale=10.0 ** (i - 1))
    seg = torch.tensor(list(zip(offs, sizes)), dtype=torch.int64, device=DEV)
    meta = torch.zeros(3, 3, device=DEV)
    buf, dst = _guarded((total,), torch.uint8)
    ops.fp8_quantize_segments(src, dst, seg, meta, 0)
    _guard_intact(buf, "fp8_quantize_segments")
    for i, (o, n) in enumerate(zip(offs, sizes)):
        a = src[o:o + n].float().abs().max().item()
        assert meta[2, i].item() == a
        assert abs(meta[0, i].item() * a / 448.0 - 1.0) <= 4 * fo.EPS32
        want = (src[o:o + n].float() * meta[0, i]).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
        assert torch.equal(dst[o:o + n], want), f"segment {i}: {(dst[o:o + n] != want).sum().item()} bytes differ"
        assert (dst[o + n:o + n + 64] == SENTINEL[torch.uint8]).all(), f"segment {i}: gap written"


# =============================================================================================== embedding
def _embed_ids(T, V, mode, seed):
    if mode == "equal":
        return torch.full((T,), 17, dtype=torch.long, device=DEV)
    ids = torch.randint(0, V, (T,), device=DEV, generator=_gen(seed))
    ids[::5] = -3
    ids[1::7] = V + 11
    ids[2::9] = V
    ids[3::11] = V - 1
    ids[4::13] = 0
    return ids


@pytest.mark.parametrize("mode", ["mixed", "equal"])
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("d", [64, 768, 2560])
def test_embedding(d, B, mode):
    """``embed_fwd_kernel`` (ids < 0 read row 0, ids >= V row V-1) with and without wpe, bit-exact; ``embed_bwd_wte_kernel``
    (vector RED; out-of-range ids are skipped; "equal": every token adds into one row) and ``embed_bwd_wpe_kernel`` (no atomics,
    bitwise reproducible), each also alone (the other embedding frozen). ``embed_pos`` (decoder) on the same rows."""
    ops = _ops()
    S, V = 32, 1000
    T = B * S
    ids = _embed_ids(T, V, mode, seed=d + B)
    wte, wpe = _randn(V, d, seed=d), _randn(S + 3, d, seed=d + 1)
    what = f"embed d={d} B={B} ids={mode}"
    for wp in (wpe, None):
        ref = fo.embed_fwd(ids, wte, wp, S)
        outs = []
        for _ in range(2):
            buf, out = _guarded((T, d), torch.bfloat16)
            ops.embed_fwd(ids, wte, wp, out, S)
            _guard_intact(buf, what)
            assert torch.equal(out, ref.float().bfloat16()), f"{what} wpe={wp is not None}: forward differs from the fp64 sum"
            outs.append(out.clone())
        _same_bits(outs[1], outs[0], f"{what} forward")
        pos = (torch.arange(T, device=DEV) % S).to(torch.int32)
        pbuf, pout = _guarded((T, d), torch.bfloat16)
        ops.embed_pos(ids.to(torch.int32), pos, wte, wp, pout)
        _guard_intact(pbuf, what + " embed_pos")
        assert torch.equal(pout, outs[0]), f"{what} wpe={wp is not None}: embed_pos differs from embed_fwd"
    dh = _randn(T, d, seed=d + B + 9)
    dwte0 = torch.randn(V, d, device=DEV, generator=_gen(3))
    dwpe0 = torch.randn(S + 3, d, device=DEV, generator=_gen(4))
    rwte, rwpe, twte, twpe = fo.embed_bwd(ids, dh, V, S, dwte0, dwpe0)
    for want_te, want_pe in ((True, True), (True, False), (False, True)):
        tag = f"{what} dwte={want_te} dwpe={want_pe}"
        pes = []
        for _ in range(2):
            tbuf, dwte = _guarded((V, d), torch.float32, dwte0) if want_te else (None, None)
            pbuf, dwpe = _guarded((S + 3, d), torch.float32, dwpe0) if want_pe else (None, None)
            ops.embed_bwd(ids, dh, dwte, dwpe, S)
            if want_te:
                _guard_intact(tbuf, tag + " dwte")
                fo.assert_within(dwte, rwte, twte, tag + " dwte")
            if want_pe:
                _guard_intact(pbuf, tag + " dwpe")
                fo.assert_within(dwpe[:S], rwpe, twpe, tag + " dwpe")
                assert torch.equal(dwpe[S:], dwpe0[S:]), f"{tag}: dwpe rows past seq_len written"
                pes.append(dwpe.clone())
        if want_pe:
            _same_bits(pes[1], pes[0], tag + " dwpe")


# =============================================================================================== optimizer
def _hyper(kind, step, lr=3e-2, b1=0.9, b2=0.99, eps=1e-6, wd=0.1, clip_exp=0.25, coupled=False):
    t = step + 1
    h = dict(first=False, lr=lr, beta1=b1, beta2=b2, eps=eps, decay=1.0, wd=0.0, clip=math.inf, step_size=0.0, inv_sqrt_bc2=1.0)
    if kind == 0:
        h["first"] = step == 0
        if coupled:                                    # decouple: false — wd * p joins the gradient
            h["wd"] = wd
        else:
            h["decay"] = 1.0 - lr * wd
        if step > 0:
            h["clip"] = float(step) ** clip_exp
    elif kind == 1:
        h["decay"] = 1.0 - wd
        h["step_size"] = lr / (1.0 - b1 ** t)
        h["inv_sqrt_bc2"] = 1.0 / math.sqrt(1.0 - b2 ** t)
    else:
        h["decay"] = 1.0 - lr * wd
    return h


def _optim_call(kind, p, g, m, v, shadow, h, gm):
    _ops().ext().fused_optimizer(p, g, m, v, shadow, kind, h["first"], h["lr"], h["beta1"], h["beta2"], h["eps"], h["decay"],
                                 h["clip"], h["step_size"], h["inv_sqrt_bc2"], gm, wd=h["wd"])


@pytest.mark.parametrize("with_shadow", [True, False])
@pytest.mark.parametrize("with_gm", [True, False])
@pytest.mark.parametrize("n", [4, 4100, (1 << 22) + 4])
@pytest.mark.parametrize("kind,coupled", [(0, False), (1, False), (2, False), (0, True)], ids=["adopt", "adamw", "sgd", "adopt_coupled"])
def test_fused_optimizer(kind, coupled, n, with_gm, with_shadow):
    """``optim_kernel`` for 5 steps against ``fused_oracle.optim_step`` from the kernel's own state each step: ADOPT's first
    step (only v is seeded) and a clip ``step**0.25`` that binds (v was seeded from small or zero gradients), AdamW's bias
    corrections, SGD without moment planes, weight decay (ADOPT's also coupled: added to the gradient), grad_mult, zero
    gradients (ADOPT's ``max(sqrt v, eps)``), a size that is not a multiple of the grid stride. The bf16 shadow equals
    ``p.to(bf16)`` bitwise."""
    p = torch.randn(n, device=DEV, generator=_gen(n))
    m = torch.zeros(n, device=DEV) if kind != 2 else torch.empty(0, device=DEV)
    v = torch.zeros(n, device=DEV) if kind != 2 else torch.empty(0, device=DEV)
    sbuf, shadow = _guarded((n,), torch.bfloat16) if with_shadow else (None, None)
    gm = torch.tensor([0.5], device=DEV) if with_gm else None
    what = f"fused_optimizer kind={kind} coupled={coupled} n={n} grad_mult={with_gm} shadow={with_shadow}"
    bound_seen = False
    for step in range(5):
        g = torch.randn(n, device=DEV, generator=_gen(step)) * (0.1 if step == 0 else 1.0)
        g[::7] = 0.0                                   # zero every step: v stays 0 there
        if step == 0:
            g[3::11] = 0.0                             # zero only at the seeding step: g / eps later, clipped
        h = _hyper(kind, step, coupled=coupled)
        state = (p.clone(), m.clone(), v.clone())
        P, M, V, tol = fo.optim_step(kind, p, g, m if kind != 2 else p, v if kind != 2 else p, h,
                                       grad_mult=0.5 if with_gm else None)
        if kind == 0 and step > 0:
            G = g.to(F64) * (0.5 if with_gm else 1.0) + h["wd"] * p.to(F64)
            bound_seen |= bool((G.abs() / v.to(F64).sqrt().clamp(min=h["eps"]) > h["clip"]).any())
        _optim_call(kind, p, g, m, v, shadow, h, gm)
        tag = f"{what} step {step}"
        fo.assert_within(p, P, tol["p"], tag + " p")
        if kind != 2:
            fo.assert_within(m, M, tol["m"], tag + " m")
            fo.assert_within(v, V, tol["v"], tag + " v")
        if with_shadow:
            _guard_intact(sbuf, tag + " shadow")
            assert torch.equal(_bits(shadow), _bits(p.to(torch.bfloat16))), f"{tag}: shadow != p.to(bf16)"
        if step == 4:                                   # the same step again from the same state: the same bits
            p2, m2, v2 = state
            _optim_call(kind, p2, g, m2, v2, None, h, gm)
            _same_bits(p2, p, tag + " p")
            if kind != 2:
                _same_bits(m2, m, tag + " m")
                _same_bits(v2, v, tag + " v")
    if kind == 0 and n > 4:
        assert bound_seen, "the ADOPT clip never bound: the test does not exercise it"


# =============================================================================================== flat helpers
@pytest.mark.parametrize("n", [4, 1000, 1001, (1 << 20) + 3, 1 << 26])
def test_flat_l2_norm(n):
    """``sqnorm_kernel``: float4 body plus the ``n % 4`` tail (the last three elements are large, so a dropped tail is far
    outside the bound); relative error <= 1e-6 against fp64."""
    x = torch.randn(n, device=DEV, generator=_gen(n))
    x[-3:] = 1000.0
    got = _ops().flat_l2_norm(x).item()
    want = x.to(F64).norm().item()
    assert abs(got - want) <= 1e-6 * want, f"flat_l2_norm n={n}: {got!r} vs {want!r} (rel err {abs(got - want) / want:.3g})"


def test_cast_bf16_special_values():
    """``cast_bf16_kernel`` gives the bits of ``torch``'s cast: signed zeros, infinities, NaN, round-to-nearest-even ties in
    both directions, overflow to inf, and fp32 subnormals (kept, not flushed, despite ``--use_fast_math``)."""
    vals = [0.0, -0.0, math.inf, -math.inf, math.nan, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 3.4028234e38,
            3.3961e38, 2.0 ** -140, -(2.0 ** -149), 1.5 * 2.0 ** -126, 2.0 ** -133 * 1.5, 2.0 ** -126 * (1 - 2.0 ** -9), 1.0]
    src = torch.tensor(vals, dtype=torch.float32).to(DEV)
    src = torch.cat([src, torch.randn(4096, device=DEV, generator=_gen(5)) * 1e-39])
    dst = torch.empty(src.numel(), dtype=torch.bfloat16, device=DEV)
    _ops().cast_bf16(src, dst)
    want = src.to(torch.bfloat16)
    diff = torch.nonzero(_bits(dst) != _bits(want)).flatten().tolist()
    assert not diff, f"cast_bf16 differs from torch at {diff[:8]}: got {[hex(int(_bits(dst)[i]) & 0xffff) for i in diff[:8]]}, " \
                     f"want {[hex(int(_bits(want)[i]) & 0xffff) for i in diff[:8]]}"
    assert (_bits(dst)[16:] != 0).sum() > 1000, "the subnormal inputs were flushed"


# =============================================================================================== operand guards
def test_vector_kernels_reject_misaligned_operands():
    """Every binding whose kernel moves rows in 16-byte vectors rejects, before any launch, a row stride that is not a
    multiple of 16 bytes and a base pointer one element off; the optimizer rejects planes of the wrong length."""
    ops = _ops()
    R, V = 16, 2048
    buf = _randn(R * (V + 8) + 8, seed=1)
    stats = torch.zeros(4, dtype=F64, device=DEV)
    tgt = torch.zeros(R, dtype=torch.long, device=DEV)
    odd_stride = buf[:R * (V + 1)].view(R, V + 1)[:, :V]
    off_base = buf[1:1 + R * V].view(R, V)
    for name, t in (("row stride", odd_stride), ("base", off_base)):
        with pytest.raises(RuntimeError, match="cross_entropy"):
            ops.cross_entropy(t, tgt, 1.0, True, stats)
        with pytest.raises(RuntimeError, match="col_sum"):
            ops.col_sum(t, torch.zeros(V, device=DEV))
        with pytest.raises(RuntimeError, match="colsum_quant"):
            ops.colsum_quant(t, torch.zeros(V, device=DEV), None)
    meta = torch.ones(3, 1, device=DEV)
    with pytest.raises(RuntimeError):
        y8 = torch.zeros(R, V + 4, dtype=torch.uint8, device=DEV)[:, :V]
        ops.colsum_quant(buf[:R * V].view(R, V), None, y8, ops.E5M2, meta, 0)
    x = buf[1:1 + R * 256].view(R, 256)
    g = torch.ones(256, device=DEV)
    y, m, r = torch.empty(R, 256, dtype=torch.bfloat16, device=DEV), torch.empty(R, device=DEV), torch.empty(R, device=DEV)
    with pytest.raises(RuntimeError, match="layernorm_fwd"):
        ops.layernorm_fwd(x, g, None, y, m, r)
    with pytest.raises(RuntimeError, match="layernorm_bwd"):
        ops.layernorm_bwd(x, x, g, m, r, None, y, None, None)
    with pytest.raises(RuntimeError, match="layernorm_fwd_q8"):
        ops.layernorm_fwd_q8(x, g, None, torch.empty(R, 256, dtype=torch.uint8, device=DEV), m, r, 1e-5, meta, 0)
    with pytest.raises(RuntimeError, match="layernorm_fwd"):
        ops.layernorm_fwd(y, torch.ones(255, device=DEV), None, y, m, r)               # gamma of the wrong length
    with pytest.raises(RuntimeError, match="embed_fwd"):
        ops.embed_fwd(tgt, buf[1:1 + 64 * 256].view(64, 256), None, y, R)
    with pytest.raises(RuntimeError, match="flat_l2_norm"):
        ops.flat_l2_norm(torch.zeros(1028, device=DEV)[1:1025])
    with pytest.raises(RuntimeError, match="flat_l2_norm"):
        ops.flat_l2_norm(torch.zeros(2048, device=DEV)[::2])
    n = 4100
    p = torch.zeros(n, device=DEV)
    h = _hyper(1, 0)
    for bad in ("g", "m", "v", "shadow"):
        args = dict(g=torch.zeros(n, device=DEV), m=torch.zeros(n, device=DEV), v=torch.zeros(n, device=DEV),
                    shadow=torch.zeros(n, dtype=torch.bfloat16, device=DEV))
        args[bad] = args[bad][:n - 4]
        with pytest.raises(RuntimeError, match="fused_optimizer"):
            _optim_call(1, p, args["g"], args["m"], args["v"], args["shadow"], h, None)
    torch.cuda.synchronize()


# =============================================================================================== second device
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_cross_entropy_on_a_second_device():
    """The shared-memory opt-in of ``ce_smem_kernel`` is a per-device attribute: after a call on cuda:0, the same process must
    run V = 50368 on cuda:1 and match the oracle."""
    R, V = 300, 50368
    x, tgt, uni = _ce_case(R, V, 1.0, seed=3)
    _ce_run(x, tgt, uni, 0.5)
    torch.cuda.synchronize(DEV)
    d1 = torch.device("cuda", 1)
    x1, tgt1, uni1 = x.to(d1), tgt.to(d1), uni.to(d1)
    work = x1.clone()
    lse = torch.empty(R, device=d1)
    stats = torch.zeros(4, dtype=F64, device=d1)
    with torch.cuda.device(d1):
        _ops().cross_entropy(work, tgt1, 0.5, True, stats, lse, uni1)
        torch.cuda.synchronize(d1)
    _ce_check(work, x1, tgt1, uni1, 0.5, stats, lse, "cross_entropy on cuda:1")
