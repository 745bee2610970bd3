"""Sliding-window attention kernels (``window`` W of ``attention_fwd`` / ``attention_bwd`` / ``decode_attention`` /
``cache_attention``) against the fp64 oracle of ``attention_oracle``.

Query q sees key k iff q - W <= k <= q, intersected with the document mask when ``doc_start`` / ``doc_end`` are given. The
oracle and the bf16 baseline take that mask as ``keep_fn``; the bounds are the per-tile criterion of ``attention_oracle``.
"""
import math

import pytest
import torch

import attention_oracle as A
from test_doc_attention_gpu import _bounds, _sid
from test_gqa_attention_gpu import _gqa_inputs, _group_sum, _slopes, _split

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN = float("nan")
LSE_ATOL = 1e-4   # as for the plain kernels (test_attention_gpu.py)
H = 4


def _fwd(qkv, Hkv, scale, slopes, ds=None, window=-1):
    from photon_b200 import ops

    B, S, W = qkv.shape
    dh = W // (H + 2 * Hkv)
    out = torch.full((B, S, H * dh), NAN, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, S), NAN, dtype=torch.float32, device=DEV)
    ops.attention_fwd(qkv, out, lse, H, scale, True, slopes, ds, n_kv_heads=Hkv, window=window)
    return out, lse


def _bwd(qkv, out, dout, lse, Hkv, scale, slopes, ds=None, de=None, window=-1):
    from photon_b200 import ops

    dqkv = torch.full_like(qkv, NAN)
    delta = torch.full_like(lse, NAN)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, slopes, ds, de, n_kv_heads=Hkv, window=window)
    return dqkv


def _keep_fn(W, sid=None):
    def keep(b, h, q_pos, n):
        k_pos = torch.arange(n, device=q_pos.device)
        m = (k_pos[None, :] <= q_pos[:, None]) & (k_pos[None, :] >= q_pos[:, None] - W)
        if sid is not None:
            s = sid[b].to(q_pos.device)
            m = m & (s[q_pos][:, None] == s[:n][None, :])
        return m
    return keep


def _refs(qkv, dout, Hkv, scale, slopes, keep_fn):
    G = H // Hkv
    q, k, v = _split(qkv, H, Hkv)
    kr, vr = k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)
    do = A.heads(dout, H)
    sl = None if slopes is None else slopes.tolist()
    ref = A.oracle(q, kr, vr, scale, causal=True, slopes=sl, dout=do, keep_fn=keep_fn)
    base = A._run(q, kr, vr, do, scale, True, sl, None, None, torch.bfloat16, keep_fn)   # noqa: SLF001
    ref.dk, ref.dv = _group_sum(ref.dk, Hkv), _group_sum(ref.dv, Hkv)
    base.dk, base.dv = (_group_sum(t.bfloat16(), Hkv).double() for t in (base.dk, base.dv))
    return ref, base


# (d_head, kv heads, ALiBi, document mask): each window and sequence length runs every combination once
FEATS = [(64, H, False, False), (64, 2, True, False), (64, H, True, True), (64, 1, False, True),
         (128, H, False, False), (128, 2, True, True), (128, 1, True, False), (128, H, False, True)]


def _windows(S):
    return sorted({0, 1, 127, 128, 129, 300, 1000, S - 1, S + 5})


# test id -> a measured miss of the per-tile max bound with the tile and whole-tensor means inside theirs, reported as an
# expected failure after every other check of the test (as attention_oracle.KNOWN and test_doc_attention_gpu.KNOWN_DOC do).
# Measured on an H100 80GB HBM3 at 700 W.
KNOWN_WINDOW = {
    ("dv", "s128-w129-dh128-kv4-doc"): "worst dV tile max 1.02x its bound (b=1, h=2, keys 0-127), worst tile mean 0.48x, "
                                       "whole-tensor mean 0.51x the bf16 baseline's; W = 129 >= S - 1, so this is the document "
                                       "mask alone",
    ("dq", "s2048-w128-dh64-kv2-alibi"): "worst dQ tile max 1.03x its bound (h=0, rows 1152-1279), worst tile mean 0.61x, "
                                         "whole-tensor mean 0.56x the bf16 baseline's",
    ("dq", "s2048-w127-dh64-kv1-doc"): "worst dQ tile max 1.06x its bound (h=3, rows 1408-1535), worst tile mean 0.50x, "
                                       "whole-tensor mean 0.52x the bf16 baseline's",
}


def _test_id(S, W, dh, Hkv, alibi, doc):
    return f"s{S}-w{W}-dh{dh}-kv{Hkv}{'-alibi' if alibi else ''}{'-doc' if doc else ''}"


MATRIX = [pytest.param(S, W, dh, Hkv, alibi, doc, id=_test_id(S, W, dh, Hkv, alibi, doc))
          for S in (128, 256, 2048) for W in _windows(S) for dh, Hkv, alibi, doc in FEATS]


@pytest.mark.parametrize("S,W,dh,Hkv,alibi,doc", MATRIX)
def test_window_attention_fwd_bwd(S, W, dh, Hkv, alibi, doc):
    B = 1 if S == 2048 else 2
    qkv, dout = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=S + W + dh + Hkv)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    sid = ds = de = None
    if doc:
        sid = _sid(("mid_tile", "tile_edges")[:B], S) if S == 2048 else _sid(("singletons", "before_tile_end")[:B], S)
        ds, de = _bounds(sid)
    out, lse = _fwd(qkv, Hkv, scale, slopes, ds, W)
    dqkv = _bwd(qkv, out, dout, lse, Hkv, scale, slopes, ds, de, W)
    dqkv2 = _bwd(qkv, out, dout, lse, Hkv, scale, slopes, ds, de, W)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all() and torch.isfinite(lse).all() and torch.isfinite(dqkv).all()), "an output was never written"
    assert torch.equal(dqkv[..., H * dh:], dqkv2[..., H * dh:]), "dK / dV are not bitwise repeatable"
    ref, base = _refs(qkv, dout, Hkv, scale, slopes, _keep_fn(W, sid))
    case = f"normal, W {W}{', doc' if doc else ''}"
    A.check("o", A.heads(out, H), ref.o, base.o, case=case)
    A.check_lse(lse, ref.lse, LSE_ATOL, case=case)
    dev = A.Deviations()
    for name, got in zip(("dq", "dk", "dv"), _split(dqkv, H, Hkv)):
        if W == 0 and name != "dv":
            # each row sees only its own key: P = 1, dS = dP - delta = 0 exactly, and so are the oracle's and the baseline's
            # dQ and dK; the kernel's are what is left of dP - delta after fp32 rounding
            assert got.abs().max().item() < 1e-3, name
            continue
        known = KNOWN_WINDOW.get((name, _test_id(S, W, dh, Hkv, alibi, doc)))
        if known is not None:
            rep = A.tile_report(name, got, getattr(ref, name), getattr(base, name), case=case)
            print(rep["msg"])
            if rep["tile_ratio"] > 1.0 and math.isfinite(rep["tile_ratio"]) and rep["mean_ratio"] <= 1.0:
                dev.append(f"{known}: {rep['msg']}")
                continue
        A.check(name, got, getattr(ref, name), getattr(base, name), case=case)
    dev.report()


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("doc", [False, True])
def test_wide_window_is_bitwise_causal(dh, alibi, doc):
    """W >= S - 1 hides no key: O, LSE, dK and dV are bitwise those of the run without a window (dQ leaves through float
    reduce-adds, whose order is not fixed)."""
    B, S, Hkv = 2, 1024, 2
    qkv, dout = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=dh + alibi)
    slopes = _slopes(H, alibi)
    ds, de = _bounds(_sid(("c4", "mid_tile"), S)) if doc else (None, None)
    out, lse = _fwd(qkv, Hkv, 0.125, slopes, ds)
    dqkv = _bwd(qkv, out, dout, lse, Hkv, 0.125, slopes, ds, de)
    for W in (S - 1, S, S + 5, 2 ** 31 - 1):
        out_w, lse_w = _fwd(qkv, Hkv, 0.125, slopes, ds, W)
        dqkv_w = _bwd(qkv, out_w, dout, lse_w, Hkv, 0.125, slopes, ds, de, W)
        torch.cuda.synchronize()
        assert torch.equal(out, out_w) and torch.equal(lse, lse_w), W
        assert torch.equal(dqkv[..., H * dh:], dqkv_w[..., H * dh:]), W
        torch.testing.assert_close(dqkv[..., : H * dh], dqkv_w[..., : H * dh], rtol=1e-2, atol=1e-3)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("W", [129, 300])
def test_key_tiles_before_every_window_are_never_read(dh, W):
    """NaN in the K / V rows of key tiles that lie before the window of a query tile's first row: that tile's O and LSE are
    bitwise those of a clean run (a tile that were loaded would spread NaN through P V even where masked)."""
    B, S, Hkv, P = 1, 2048, 2, 512
    qkv, _ = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=W)
    out, lse = _fwd(qkv, Hkv, 0.125, None, None, W)
    bad = qkv.clone()
    _, k, v = _split(bad, H, Hkv)
    k[:, :, :P] = NAN
    v[:, :, :P] = NAN
    out_b, lse_b = _fwd(bad, Hkv, 0.125, None, None, W)
    torch.cuda.synchronize()
    first = -(-(P + W) // 128) * 128   # first query tile whose first row's window starts at or after P
    assert torch.equal(out_b[:, first:], out[:, first:]) and torch.equal(lse_b[..., first:], lse[..., first:])
    assert bool(torch.isnan(out_b[:, P:P + 1]).any()), "the poisoned keys were not used where they are visible"


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("W", [129, 300])
def test_query_steps_past_every_window_are_never_read(dh, W):
    """NaN in Q and dO of the query rows from P on: dK and dV of every key tile whose last key's window ends before P are
    bitwise unchanged."""
    B, S, Hkv, P = 1, 2048, 2, 1024
    qkv, dout = _gqa_inputs("normal", B, S, H, Hkv, dh, seed=W + 1)
    out, lse = _fwd(qkv, Hkv, 0.125, None, None, W)
    dqkv = _bwd(qkv, out, dout, lse, Hkv, 0.125, None, window=W)
    bad, dbad = qkv.clone(), dout.clone()
    bad[:, P:, : H * dh] = NAN
    dbad[:, P:] = NAN
    dqkv_b = _bwd(bad, out, dbad, lse, Hkv, 0.125, None, window=W)
    torch.cuda.synchronize()
    n_keys = (P - 127 - W + 127) // 128 * 128   # key tiles jt with jt * 128 + 127 + W < P
    assert n_keys > 0
    assert torch.equal(dqkv_b[:, :n_keys, H * dh:], dqkv[:, :n_keys, H * dh:])
    assert bool(torch.isnan(dqkv_b[:, P - 1, H * dh:]).any()), "the poisoned queries were not used where they see the key"


def test_bindings_reject_bad_windows():
    from photon_b200 import ops

    B, S, dh = 1, 128, 64
    qkv = torch.zeros(B, S, 3 * H * dh, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(B, S, H * dh, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(B, H, S, dtype=torch.float32, device=DEV)
    kc = torch.zeros(1, H, 256, dh, dtype=torch.bfloat16, device=DEV)
    pos = torch.zeros(1, dtype=torch.int32, device=DEV)
    n0 = ops.launch_count()
    for causal, window in ((True, -2), (True, -100), (False, 0), (False, 64)):
        with pytest.raises(RuntimeError, match="window"):
            ops.attention_fwd(qkv, out, lse, H, 0.125, causal, window=window)
        with pytest.raises(RuntimeError, match="window"):
            ops.attention_bwd(qkv, out, out, lse, torch.zeros_like(qkv), torch.zeros_like(lse), H, 0.125, causal, window=window)
    with pytest.raises(RuntimeError, match="window"):
        ops.decode_attention(qkv[:, 0], kc, kc, pos, out[:, 0].clone(), H, 0.125, window=-2)
    with pytest.raises(RuntimeError, match="window"):
        ops.cache_attention(qkv[:, 0].clone(), kc, kc, ops.cache_tiles([(0, 0, 1, 0)], DEV), out[:, 0].clone(), H, 0.125, window=-3)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a kernel was launched before the argument check"


# ------------------------------------------------------------------------------------------------ decoding and scoring
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("G", [1, 4])
@pytest.mark.parametrize("W", [0, 1, 255, 256, 300, 1000])
def test_window_decode_attention(dh, alibi, G, W):
    """Positions below and beyond W (chunks of 256 keys wholly below the window, the chunk holding its first key, and a
    window that covers the whole sequence). Cache rows below each row's window hold NaN: they are never read."""
    from photon_b200 import ops

    lens = [1, 2, 127, 128, 129, 300, 1000, 1500, 2048]
    B, S, Hkv = len(lens), 2048, H // G
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    pos = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=DEV)
    for case in ("normal", "peaked"):
        seq, _ = _gqa_inputs(case, B, S, H, Hkv, dh, seed=dh + alibi + G + W)
        q, k, v = _split(seq, H, Hkv)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = seq[torch.arange(B, device=DEV), pos.long()].contiguous()
        out = torch.empty(B, H * dh, dtype=torch.bfloat16, device=DEV)
        ops.decode_attention(qkv, kc, vc, pos, out, H, scale, slopes, n_kv_heads=Hkv, window=W)
        kb, vb = kc.clone(), vc.clone()
        for b, n in enumerate(lens):
            kb[b, :, : max(0, n - 1 - W)] = NAN
            vb[b, :, : max(0, n - 1 - W)] = NAN
        out_b = torch.empty_like(out)
        ops.decode_attention(qkv, kb, vb, pos, out_b, H, scale, slopes, n_kv_heads=Hkv, window=W)
        torch.cuda.synchronize()
        assert torch.equal(out, out_b), "a key below the window was read"
        qr = qkv[:, : H * dh].view(B, H, 1, dh)
        kr, vr = kc.repeat_interleave(G, 1), vc.repeat_interleave(G, 1)
        sl = None if slopes is None else slopes.tolist()
        qp = pos.long()[:, None]
        ref = A.oracle(qr, kr, vr, scale, causal=True, slopes=sl, q_pos=qp, lengths=lens, keep_fn=_keep_fn(W))
        base = A._run(qr, kr, vr, None, scale, True, sl, qp, lens, torch.bfloat16, _keep_fn(W))   # noqa: SLF001
        A.check("decode o", out.view(B, H, 1, dh), ref.o, base.o, rows=1, case=f"{case}, G {G}, W {W}", whole_mean=True)


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("W", [0, 5, 127, 128, 300, 1000])
def test_window_cache_attention(dh, G, W):
    from photon_b200 import ops
    from test_score_gpu import RUNS, SENTINEL, _layout

    S, Bm = 2048, 6
    Hkv = H // G
    runs, N = _layout(RUNS)
    scale = 1.0 / math.sqrt(dh)
    tiles = ops.cache_tiles(runs, DEV)
    slopes = _slopes(H, True)
    for case in ("normal", "peaked"):
        seq, _ = _gqa_inputs(case, Bm, S, H, Hkv, dh, seed=dh + G + W)
        _, k, v = _split(seq, H, Hkv)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = torch.randn(N, (H + 2 * Hkv) * dh, device=DEV).bfloat16()
        for slot, r0, n, p in runs:
            qkv[r0: r0 + n] = seq[slot, p: p + n]
        out = torch.full((N, H * dh), SENTINEL, dtype=torch.bfloat16, device=DEV)
        ops.cache_attention(qkv, kc, vc, tiles, out, H, scale, slopes, n_kv_heads=Hkv, window=W)
        torch.cuda.synchronize()
        covered = torch.zeros(N, dtype=torch.bool)
        got, refs, bases = [], [], []
        for slot, r0, n, p in tiles.tolist():
            covered[r0: r0 + n] = True
            q = qkv[r0: r0 + n, : H * dh].view(1, n, H, dh).transpose(1, 2)
            qp = (p + torch.arange(n, device=DEV))[None]
            ks, vs = (t[slot: slot + 1].repeat_interleave(G, 1) for t in (kc, vc))
            refs.append(A.oracle(q, ks, vs, scale, causal=True, slopes=slopes.tolist(), q_pos=qp, lengths=[p + n], keep_fn=_keep_fn(W)).o)
            bases.append(A._run(q, ks, vs, None, scale, True, slopes.tolist(), qp, [p + n], torch.bfloat16, _keep_fn(W)).o)   # noqa: SLF001
            got.append(out[r0: r0 + n].view(1, n, H, dh).transpose(1, 2))
        assert all(bool(torch.isfinite(g).all()) for g in got)
        A.check_tiles("cache o", got, refs, bases, case=f"{case}, G {G}, W {W}")
        assert bool((out[~covered.to(DEV)] == SENTINEL).all()), "a row outside the tiles was written"
