"""Grouped-query attention kernels (n_kv_heads < n_heads) against the fp64 oracle of ``attention_oracle``.

The fused buffer is [B, S, (H + 2*H_kv) * dh]: H query heads, then H_kv key heads, then H_kv value heads; query head h reads kv
head h // G, G = H / H_kv. The oracle runs on K / V explicitly repeated to H heads, with dK / dV summed over each group; the
bf16 baseline is PyTorch autograd through ``repeat_interleave`` (so its group sums are bf16 too). The per-tile criterion is
``attention_oracle.check``.
"""
import math

import pytest
import torch

import attention_oracle as A

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN = float("nan")
LSE_ATOL = 1e-4   # as for the multi-head kernels (test_attention_gpu.py)
H = 8


def _gqa_inputs(case, B, S, Hq, Hkv, dh, seed):
    """The input cases of ``attention_oracle.make_inputs`` with only the first H_kv key / value heads kept."""
    x, dout = A.make_inputs(case, B, S, Hq, dh, DEV, seed=seed)
    x = x.view(B, S, 3, Hq, dh)
    qkv = torch.cat([x[:, :, 0].reshape(B, S, -1), x[:, :, 1, :Hkv].reshape(B, S, -1), x[:, :, 2, :Hkv].reshape(B, S, -1)], -1)
    return qkv.contiguous(), dout


def _split(qkv, Hq, Hkv):
    """[B, S, (H + 2 H_kv) dh] -> q [B, H, S, dh], k, v [B, H_kv, S, dh]."""
    B, S, W = qkv.shape
    dh = W // (Hq + 2 * Hkv)
    q = qkv[..., : Hq * dh].view(B, S, Hq, dh).transpose(1, 2)
    k = qkv[..., Hq * dh: (Hq + Hkv) * dh].view(B, S, Hkv, dh).transpose(1, 2)
    v = qkv[..., (Hq + Hkv) * dh:].view(B, S, Hkv, dh).transpose(1, 2)
    return q, k, v


def _slopes(Hq, alibi):
    from photon_b200.models.mpt import alibi_slopes

    return alibi_slopes(Hq).to(DEV) if alibi else None


def _fwd(qkv, Hq, Hkv, scale, slopes, ds=None):
    from photon_b200 import ops

    B, S, W = qkv.shape
    dh = W // (Hq + 2 * Hkv)
    out = torch.full((B, S, Hq * dh), NAN, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, Hq, S), NAN, dtype=torch.float32, device=DEV)
    ops.attention_fwd(qkv, out, lse, Hq, scale, True, slopes, ds, n_kv_heads=Hkv)
    return out, lse


def _bwd(qkv, out, dout, lse, Hq, Hkv, scale, slopes, ds=None, de=None):
    from photon_b200 import ops

    dqkv = torch.full_like(qkv, NAN)
    delta = torch.full_like(lse, NAN)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, Hq, scale, True, slopes, ds, de, n_kv_heads=Hkv)
    return dqkv


def _group_sum(t, Hkv):
    B, Hq, R, dh = t.shape
    return t.view(B, Hkv, Hq // Hkv, R, dh).sum(2)


def _baseline(q, k, v, scale, slopes, dout, G):
    """``attention_oracle``'s batched bf16 baseline, with K / V repeated inside autograd (bf16 group sums in the backward)."""
    B, Hq, S, dh = q.shape
    pos = torch.arange(S, device=q.device)
    with torch.enable_grad():
        leaves = [t.detach().bfloat16().requires_grad_(True) for t in (q, k, v)]
        kr, vr = (t.repeat_interleave(G, dim=1) for t in leaves[1:])
        s = (leaves[0] @ kr.transpose(-1, -2)) * scale
        if slopes is not None:
            s = s + torch.as_tensor(slopes, dtype=torch.float32).to(q.device).bfloat16()[:, None, None] * (pos[None, :] - pos[:, None]).bfloat16()
        s = s.masked_fill(pos[None, :] > pos[:, None], float("-inf"))
        o = torch.softmax(s, -1) @ vr
        grads = torch.autograd.grad(o, leaves, dout.bfloat16())
    return A.Result(o.detach().double(), None, *(t.double() for t in grads))


def _refs(qkv, dout, Hq, Hkv, scale, slopes, keep_fn=None):
    G = Hq // Hkv
    q, k, v = _split(qkv, Hq, Hkv)
    kr, vr = k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)
    do = A.heads(dout, Hq)
    sl = None if slopes is None else slopes.tolist()
    ref = A.oracle(q, kr, vr, scale, causal=True, slopes=sl, dout=do, keep_fn=keep_fn)
    ref.dk, ref.dv = _group_sum(ref.dk, Hkv), _group_sum(ref.dv, Hkv)
    if keep_fn is None:
        base = _baseline(q, k, v, scale, sl, do, G)
    else:   # the per-head bf16 baseline under the mask, its dK / dV summed over the group in bf16
        base = A._run(q, kr, vr, do, scale, True, sl, None, None, torch.bfloat16, keep_fn)   # noqa: SLF001
        base.dk, base.dv = (_group_sum(t.bfloat16(), Hkv).double() for t in (base.dk, base.dv))
    return ref, base


# (tensor, test id) -> a measured miss of the per-tile max bound with the tile and whole-tensor means inside theirs, reported as an
# expected failure after every other check of the test (as attention_oracle.KNOWN and test_doc_attention_gpu.KNOWN_DOC do).
# Measured on an H100 80GB HBM3 at 700 W.
KNOWN_GQA = {
    ("dq", "dh64-g1-alibi-s2048-normal"): "G = 1 is the multi-head kernel (its outputs are bitwise those of the multi-head "
                                          "build): worst dQ tile max 1.10x its bound (h=1, rows 1792-1919), worst tile mean "
                                          "0.65x, whole-tensor mean 0.57x the bf16 baseline's",
    ("dq", "dh128-g8-alibi-s2048-c4+c4"): "worst dQ tile max 1.01x its bound (b=1, h=4, rows 256-383), whole-tensor mean 0.50x "
                                          "the bf16 baseline's; the same tiles as the multi-head dQ miss of test_doc_attention_gpu "
                                          "(KNOWN_DOC, c4+c4, 1.17x)",
}


def _check_all(out, lse, dqkv, ref, base, Hq, Hkv, case, dev, test_id=""):
    A.check("o", A.heads(out, Hq), ref.o, base.o, case=case)
    A.check_lse(lse, ref.lse, LSE_ATOL, case=case)
    dq, dk, dv = _split(dqkv, Hq, Hkv)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        known = KNOWN_GQA.get((name, test_id))
        if known is not None:
            rep = A.tile_report(name, got, getattr(ref, name), getattr(base, name), case=case)
            print(rep["msg"])
            if rep["tile_ratio"] > 1.0 and math.isfinite(rep["tile_ratio"]) and rep["mean_ratio"] <= 1.0:
                dev.append(f"{known}: {rep['msg']}")
                continue
        A.check(name, got, getattr(ref, name), getattr(base, name), case=case, deviations=dev)


GROUPS = [1, 2, 4, H]
MATRIX = [pytest.param(dh, G, alibi, S, case, id=f"dh{dh}-g{G}{'-alibi' if alibi else ''}-s{S}-{case}")
          for dh in (64, 128) for G in GROUPS for alibi in (False, True) for S in (128, 1024, 2048) for case in A.CASES]


@pytest.mark.parametrize("dh,G,alibi,S,case", MATRIX)
def test_gqa_attention_fwd_bwd(dh, G, alibi, S, case):
    Hkv = H // G
    qkv, dout = _gqa_inputs(case, 1, S, H, Hkv, dh, seed=S + dh + G)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    out, lse = _fwd(qkv, H, Hkv, scale, slopes)
    dqkv = _bwd(qkv, out, dout, lse, H, Hkv, scale, slopes)
    dqkv2 = _bwd(qkv, out, dout, lse, H, Hkv, scale, slopes)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all() and torch.isfinite(lse).all() and torch.isfinite(dqkv).all()), "an output was never written"
    assert torch.equal(dqkv[..., H * dh:], dqkv2[..., H * dh:]), "dK / dV are not bitwise repeatable"
    ref, base = _refs(qkv, dout, H, Hkv, scale, slopes)
    dev = A.Deviations()
    _check_all(out, lse, dqkv, ref, base, H, Hkv, case, dev, f"dh{dh}-g{G}{'-alibi' if alibi else ''}-s{S}-{case}")
    dev.report()


@pytest.mark.parametrize("G", [2, 4, H])
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
def test_gqa_forward_equals_multi_head_on_repeated_kv(G, dh, alibi):
    """The forward reads the kv head's columns exactly as the multi-head kernel reads its own: O and LSE are bitwise those of
    a multi-head run on a buffer whose K / V heads are repeated."""
    B, S, Hkv = 2, 1024, H // G
    qkv, _ = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=G + dh)
    q, k, v = _split(qkv, H, Hkv)
    flat = lambda t: t.transpose(1, 2).reshape(B, S, -1)  # noqa: E731
    mha = torch.cat([flat(q), flat(k.repeat_interleave(G, 1)), flat(v.repeat_interleave(G, 1))], -1).contiguous()
    slopes = _slopes(H, alibi)
    out, lse = _fwd(qkv, H, Hkv, 0.125, slopes)
    out1, lse1 = _fwd(mha, H, H, 0.125, slopes)
    torch.cuda.synchronize()
    assert torch.equal(out, out1) and torch.equal(lse, lse1)


@pytest.mark.parametrize("G", [2, 4])
def test_gqa_nan_in_one_kv_head_stays_in_its_group(G):
    B, S, dh, Hkv = 2, 1024, 64, H // G
    qkv, dout = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=G)
    out, lse = _fwd(qkv, H, Hkv, 0.125, None)
    dqkv = _bwd(qkv, out, dout, lse, H, Hkv, 0.125, None)
    bad = qkv.clone()
    _, k, v = _split(bad, H, Hkv)
    k[1, 0, 300] = NAN                      # one key row of kv head 0, batch row 1
    v[1, 0, 500] = NAN
    out_b, lse_b = _fwd(bad, H, Hkv, 0.125, None)
    dqkv_b = _bwd(bad, out_b, dout, lse_b, H, Hkv, 0.125, None)
    torch.cuda.synchronize()
    o4, ob4 = A.heads(out, H), A.heads(out_b, H)
    assert torch.equal(ob4[:, G:], o4[:, G:]) and torch.equal(ob4[0], o4[0]), "NaN reached another group or batch row"
    assert torch.equal(lse_b[:, G:], lse[:, G:])
    dq, dk, dv = _split(dqkv, H, Hkv)
    dqb, dkb, dvb = _split(dqkv_b, H, Hkv)
    assert torch.equal(dkb[:, 1:], dk[:, 1:]) and torch.equal(dvb[:, 1:], dv[:, 1:]) and torch.equal(dkb[0], dk[0])
    assert bool(torch.isfinite(dqb[:, G:]).all() and torch.isfinite(dqb[0]).all())
    torch.testing.assert_close(dqb[:, G:], dq[:, G:], rtol=1e-2, atol=1e-3)   # dQ accumulates with float atomics
    assert bool(torch.isnan(ob4[1, :G]).any()), "the poisoned group did not see its NaN"


# ------------------------------------------------------------------------------------------------ document mask
DOC = [pytest.param(dh, G, alibi, S, pair, id=f"dh{dh}-g{G}{'-alibi' if alibi else ''}-s{S}-{pair[0]}+{pair[1]}")
       for dh in (64, 128) for G in (2, H) for alibi in (False, True) for S, pair in ((1024, ("tile_edges", "mid_tile")),
                                                                                       (2048, ("c4", "c4")))]


@pytest.mark.parametrize("dh,G,alibi,S,pair", DOC)
def test_gqa_doc_attention(dh, G, alibi, S, pair):
    from test_doc_attention_gpu import _bounds, _keep_fn, _sid

    Hkv = H // G
    qkv, dout = _gqa_inputs("normal", 2, S, H, Hkv, dh, seed=S + G + dh)
    sid = _sid(pair, S)
    ds, de = _bounds(sid)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    out, lse = _fwd(qkv, H, Hkv, scale, slopes, ds)
    dqkv = _bwd(qkv, out, dout, lse, H, Hkv, scale, slopes, ds, de)
    torch.cuda.synchronize()
    ref, base = _refs(qkv, dout, H, Hkv, scale, slopes, keep_fn=_keep_fn(sid))
    dev = A.Deviations()
    _check_all(out, lse, dqkv, ref, base, H, Hkv, f"normal, doc {pair}", dev,
               f"dh{dh}-g{G}{'-alibi' if alibi else ''}-s{S}-{pair[0]}+{pair[1]}")
    dev.report()


# ------------------------------------------------------------------------------------------------ RoPE and arguments
@pytest.mark.parametrize("Hkv", [1, 2])
def test_gqa_rope_kernel(Hkv):
    from photon_b200 import ops
    from photon_b200.models.mpt import apply_rope, rope_tables

    B, S, Hq, dh = 2, 256, 4, 64
    qkv = torch.randn(B, S, (Hq + 2 * Hkv) * dh, device=DEV).bfloat16()
    cos, sin = (t.contiguous() for t in rope_tables(S, dh, 10000.0, DEV))
    q, k, v = _split(qkv.float(), Hq, Hkv)
    work = qkv.clone()
    ops.rope_(work, cos, sin, Hq, n_kv_heads=Hkv)
    gq, gk, gv = _split(work.float(), Hq, Hkv)
    assert (gq - apply_rope(q, cos, sin)).abs().max().item() < 3e-2 and (gk - apply_rope(k, cos, sin)).abs().max().item() < 3e-2
    assert torch.equal(gv, v)
    ops.rope_(work, cos, sin, Hq, inverse=True, n_kv_heads=Hkv)
    assert (work.float() - qkv.float()).abs().max().item() < 6e-2


def test_gqa_bindings_reject_bad_head_counts():
    from photon_b200 import ops

    B, S, dh = 1, 128, 64
    qkv = torch.zeros(B, S, (4 + 2 * 2) * dh, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(B, S, 4 * dh, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, 4, S, dtype=torch.float32, device=DEV)
    n0 = ops.launch_count()
    for kv in (3, 0, -2, 1):   # does not divide, none, negative, a row width that does not fit
        with pytest.raises(RuntimeError):
            ops.attention_fwd(qkv, out, lse, 4, 0.125, True, n_kv_heads=kv)
        with pytest.raises(RuntimeError):
            ops.attention_bwd(qkv, out, out, lse, torch.zeros_like(qkv), torch.zeros_like(lse), 4, 0.125, True, n_kv_heads=kv)
        with pytest.raises(RuntimeError):
            ops.rope_(qkv, torch.zeros(S, dh // 2, device=DEV), torch.zeros(S, dh // 2, device=DEV), 4, n_kv_heads=kv)
    kc = torch.zeros(1, 2, 256, dh, dtype=torch.bfloat16, device=DEV)
    pos = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError):   # the cache holds 2 kv heads
        ops.decode_attention(qkv[:, 0], kc, kc, pos, out[:, 0].clone(), 4, 0.125, n_kv_heads=1)
    with pytest.raises(RuntimeError):
        ops.decode_append(qkv[:, 0].clone(), pos, kc, kc.clone(), None, 4, n_kv_heads=4)
    with pytest.raises(RuntimeError):
        ops.cache_attention(qkv[:, 0].clone(), kc, kc, ops.cache_tiles([(0, 0, 1, 0)], DEV), out[:, 0].clone(), 4, 0.125, n_kv_heads=1)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a kernel was launched before the argument check"
    ops.attention_fwd(qkv, out, lse, 4, 0.125, True, n_kv_heads=2)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 1


# ------------------------------------------------------------------------------------------------ decoding and scoring
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("G", [2, 3, 8, 16])
def test_gqa_decode_attention(dh, alibi, G):
    """As test_decode_gpu's ragged test, with a cache of H_kv heads; G = 16 runs the query heads in two passes of 8."""
    from photon_b200 import ops

    lens = [1, 2, 127, 128, 129, 1000, 2048]
    Hq = 6 if G == 3 else 16
    B, S, Hkv = len(lens), 2048, Hq // G
    slopes = _slopes(Hq, alibi)
    scale = 1.0 / math.sqrt(dh)
    pos = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=DEV)
    for case in ("normal", "peaked", "rising"):
        seq, _ = _gqa_inputs(case, B, S, Hq, Hkv, dh, seed=dh + alibi + G)
        q, k, v = _split(seq, Hq, Hkv)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = seq[torch.arange(B, device=DEV), pos.long()].contiguous()
        out = torch.empty(B, Hq * dh, dtype=torch.bfloat16, device=DEV)
        ops.decode_attention(qkv, kc, vc, pos, out, Hq, scale, slopes, n_kv_heads=Hkv)
        torch.cuda.synchronize()
        qr = qkv[:, : Hq * dh].view(B, Hq, 1, dh)
        kr, vr = kc.repeat_interleave(G, 1), vc.repeat_interleave(G, 1)
        kw = dict(causal=True, slopes=None if slopes is None else slopes.tolist(), q_pos=pos.long()[:, None], lengths=lens)
        ref, base = A.oracle(qr, kr, vr, scale, **kw), A.baseline(qr, kr, vr, scale, **kw)
        A.check("decode o", out.view(B, Hq, 1, dh), ref.o, base.o, rows=1, case=f"{case}, G {G}", whole_mean=True)


@pytest.mark.parametrize("use_rope", [False, True])
@pytest.mark.parametrize("Hkv", [1, 2])
def test_gqa_decode_append(use_rope, Hkv):
    from photon_b200 import ops
    from photon_b200.models.mpt import rope_tables

    Hq, dh, S, Bm, N = 4, 64, 256, 3, 5
    g = torch.Generator(device=DEV).manual_seed(3 + Hkv)
    kc = torch.randn(Bm, Hkv, S, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(Bm, Hkv, S, dh, device=DEV, generator=g).bfloat16()
    qkv = torch.randn(N, (Hq + 2 * Hkv) * dh, device=DEV, generator=g).bfloat16()
    slot = torch.tensor([2, 0, 1, 1, 0], dtype=torch.int32, device=DEV)
    pos = torch.tensor([5, 0, 100, 255, 17], dtype=torch.int32, device=DEV)
    rope = tuple(t.contiguous() for t in rope_tables(S, dh, 10000.0, DEV)) if use_rope else None
    k_want, v_want, q_in = kc.clone(), vc.clone(), qkv.clone()
    ops.decode_append(qkv, pos, kc, vc, rope, Hq, slot=slot, n_kv_heads=Hkv)
    torch.cuda.synchronize()
    q, k, v = (t[:, :, 0] for t in _split(q_in.float()[:, None], Hq, Hkv))   # [N, heads, dh]
    if use_rope:
        c, s = rope[0][pos.long()][:, None], rope[1][pos.long()][:, None]
        rot = lambda t: torch.cat([t[..., : dh // 2] * c - t[..., dh // 2:] * s, t[..., dh // 2:] * c + t[..., : dh // 2] * s], -1)  # noqa: E731
        q, k = rot(q), rot(k)
    for r in range(N):
        k_want[slot[r], :, pos[r]] = k[r].bfloat16()
        v_want[slot[r], :, pos[r]] = v[r].bfloat16()
    d = Hq * dh
    torch.testing.assert_close(qkv[:, :d].float(), q.reshape(N, d), rtol=1e-2, atol=1e-2)
    assert torch.equal(qkv[:, d:], q_in[:, d:])
    torch.testing.assert_close(kc.float(), k_want.float(), rtol=1e-2, atol=1e-2)
    assert torch.equal(vc, v_want)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("G", [2, 4])
def test_gqa_cache_attention(dh, G):
    from photon_b200 import ops
    from test_score_gpu import RUNS, SENTINEL, _layout

    Hq, S, Bm = 4, 2048, 6
    Hkv = Hq // G
    runs, N = _layout(RUNS)
    scale = 1.0 / math.sqrt(dh)
    tiles = ops.cache_tiles(runs, DEV)
    slopes = _slopes(Hq, True)
    for case in ("normal", "peaked", "rising"):
        seq, _ = _gqa_inputs(case, Bm, S, Hq, Hkv, dh, seed=dh + G)
        _, k, v = _split(seq, Hq, Hkv)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = torch.randn(N, (Hq + 2 * Hkv) * dh, device=DEV).bfloat16()
        for slot, r0, n, p in runs:
            qkv[r0: r0 + n] = seq[slot, p: p + n]
        out = torch.full((N, Hq * dh), SENTINEL, dtype=torch.bfloat16, device=DEV)
        ops.cache_attention(qkv, kc, vc, tiles, out, Hq, scale, slopes, n_kv_heads=Hkv)
        torch.cuda.synchronize()
        covered = torch.zeros(N, dtype=torch.bool)
        got, refs, bases = [], [], []
        for slot, r0, n, p in tiles.tolist():
            covered[r0: r0 + n] = True
            q = qkv[r0: r0 + n, : Hq * dh].view(1, n, Hq, dh).transpose(1, 2)
            kw = dict(causal=True, slopes=slopes.tolist(), q_pos=(p + torch.arange(n, device=DEV))[None], lengths=[p + n])
            ks, vs = (t[slot: slot + 1].repeat_interleave(G, 1) for t in (kc, vc))
            refs.append(A.oracle(q, ks, vs, scale, **kw).o)
            bases.append(A.baseline(q, ks, vs, scale, **kw).o)
            got.append(out[r0: r0 + n].view(1, n, Hq, dh).transpose(1, 2))
        A.check_tiles("cache o", got, refs, bases, case=f"{case}, G {G}")
        assert bool((out[~covered.to(DEV)] == SENTINEL).all()), "a row outside the tiles was written"
