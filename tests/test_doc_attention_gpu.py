"""Document-masked wgmma attention (``doc_start`` / ``doc_end`` from ``doc_bounds``) against the fp64 oracle.

Query q sees key k iff k <= q and both rows belong to the same document (a maximal run of equal ``sequence_id``). The
oracle and the bf16 baseline take that mask as ``keep_fn``; the bounds are the per-tile criterion of ``attention_oracle``.
"""
import math

import numpy as np
import pytest
import torch

import attention_oracle as A

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN = float("nan")
LSE_ATOL = 1e-4   # as for the plain kernels (test_attention_gpu.py)


# ------------------------------------------------------------------------------------------------ layouts
def _ids_from_starts(S, starts):
    sid = np.zeros(S, dtype=np.int64)
    for s in sorted(set(starts)):
        if 0 < s < S:
            sid[s:] += 1
    return sid


def layout(name, S, seed=0):
    """sequence_id [S] of one row (non-decreasing, as the collator emits them)."""
    if name == "tile_edges":          # every boundary on a 128-row tile edge
        return _ids_from_starts(S, range(128, S, 256))
    if name == "mid_tile":            # boundaries inside tiles
        return _ids_from_starts(S, [60, 200, 333, 700, 1000, 1500, 1900])
    if name == "before_tile_end":     # a document starting on the last row of a tile
        return _ids_from_starts(S, range(127, S, 128 * 3))
    if name == "singletons":          # runs of 1-token documents (row 0 of a tile, a tile edge and mid-tile)
        return _ids_from_starts(S, list(range(1, 40)) + list(range(120, 140)) + list(range(300, 310)))
    if name == "c4":                  # EOS positions of the synthetic C4 stream, llm-foundry's EOS-mode ids
        from photon_b200.data.streaming import sequence_ids
        from photon_b200.data.synthetic import EOS_ID, SyntheticC4

        row = torch.from_numpy(SyntheticC4(S, seed=seed)[0].astype(np.int64))[None]
        return sequence_ids(row, eos_token_id=EOS_ID)[0].numpy()
    if name == "one":
        return np.zeros(S, dtype=np.int64)
    raise ValueError(name)


PAIRS = [("tile_edges", "mid_tile"), ("before_tile_end", "singletons"), ("c4", "c4")]
MODES = [(64, 12, False), (64, 12, True), (128, 16, False), (128, 16, True)]
SEQS = [128, 384, 2048]
MATRIX = [pytest.param(dh, H, alibi, S, pair, id=f"dh{dh}-h{H}{'-alibi' if alibi else ''}-s{S}-{pair[0]}+{pair[1]}")
          for dh, H, alibi in MODES for S in SEQS for pair in PAIRS]


def _sid(names, S):
    return torch.from_numpy(np.stack([layout(n, S, seed=7 + i) for i, n in enumerate(names)])).to(DEV)


def _slopes(H, alibi):
    from photon_b200.models.mpt import alibi_slopes

    return alibi_slopes(H).to(DEV) if alibi else None


def _bounds(sid):
    from photon_b200 import ops

    B, S = sid.shape
    ds = torch.full((B * S,), -7, dtype=torch.int32, device=DEV)
    de = torch.full((B * S,), -7, dtype=torch.int32, device=DEV)
    ops.doc_bounds(sid, ds, de)
    return ds, de


def _fwd(qkv, H, scale, slopes, ds=None):
    from photon_b200 import ops

    B, S, d3 = qkv.shape
    out = torch.full((B, S, d3 // 3), NAN, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, S), NAN, dtype=torch.float32, device=DEV)
    ops.attention_fwd(qkv, out, lse, H, scale, True, slopes, ds)
    return out, lse


def _bwd(qkv, out, dout, lse, H, scale, slopes, ds=None, de=None):
    from photon_b200 import ops

    dqkv = torch.full_like(qkv, NAN)
    delta = torch.full_like(lse, NAN)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, slopes, ds, de)
    return dqkv


def _keep_fn(sid):
    def keep(b, h, q_pos, n):
        k_pos = torch.arange(n, device=q_pos.device)
        s = sid[b].to(q_pos.device)
        return (k_pos[None, :] <= q_pos[:, None]) & (s[q_pos][:, None] == s[:n][None, :])
    return keep


def _refs(qkv, dout, H, scale, slopes, sid):
    q, k, v = A.split_heads(qkv, H)
    do = A.heads(dout, H)
    sl = None if slopes is None else slopes.tolist()
    keep = _keep_fn(sid)
    ref = A.oracle(q, k, v, scale, causal=True, slopes=sl, dout=do, keep_fn=keep)
    base = A._run(q, k, v, do, scale, True, sl, None, None, torch.bfloat16, keep)   # the bf16 baseline under the same mask
    return ref, base


# (tensor, layout pair, d_head, S) -> a measured miss of the per-tile max bound, reported as an expected failure after every other
# check of the test has run (as attention_oracle.KNOWN does for the plain kernels). Measured on an H100 80GB HBM3 at 700 W.
KNOWN_DOC = {
    ("dk", "tile_edges+mid_tile", 64, 2048): "worst tile max 1.04x its bound (b=1, h=5, keys 640-767, a boundary at 700); "
                                             "whole-tensor mean error 0.49x the bf16 baseline's",
    ("dq", "c4+c4", 64, 2048): "worst tile max 1.17x its bound (b=1, h=2, rows 256-383); whole-tensor mean error 0.50x the bf16 "
                               "baseline's. dS uses delta = rowsum(dO * O) of the bf16 O, like the plain kernel (attention_oracle."
                               "KNOWN); an fp32 emulation of that math reaches 0.70x of this tile's bound, so part of the excess "
                               "is not explained",
}


def _check(name, got, ref, base, case, key, dev):
    rep = A.tile_report(name, got, ref, base, case=case)
    print(rep["msg"])
    ok = rep["tile_ratio"] <= 1.0 and rep["mean_ratio"] <= 1.0
    known = KNOWN_DOC.get((name, *key)) if key is not None else None
    if not ok and known and math.isfinite(rep["tile_ratio"]) and rep["mean_ratio"] <= 1.0:
        dev.append(f"{known}: {rep['msg']}")
        return
    assert ok, rep["msg"]


def _rows(t, lo):
    """[B, H, R, dh] -> rows lo.. (a whole number of 128-row tiles)."""
    return t[:, :, lo:]


# ------------------------------------------------------------------------------------------------ bounds
def test_doc_bounds_are_maximal_runs():
    """doc_bounds on rows with runs of every length, including ids that come back (runs, not equality classes)."""
    g = np.random.default_rng(3)
    for S in (1, 5, 128, 1000, 2048, 4100):
        rows = [layout("one", S), g.integers(0, 3, S), np.cumsum(g.random(S) < 0.01), np.arange(S)]
        sid = torch.from_numpy(np.stack(rows).astype(np.int64)).to(DEV)
        ds, de = _bounds(sid)
        torch.cuda.synchronize()
        for b, r in enumerate(rows):
            exp_s, exp_e = np.zeros(S, np.int64), np.zeros(S, np.int64)
            cur = 0
            for s in range(S):
                if s > 0 and r[s] != r[s - 1]:
                    cur = s
                exp_s[s] = cur
            cur = S - 1
            for s in range(S - 1, -1, -1):
                if s < S - 1 and r[s] != r[s + 1]:
                    cur = s
                exp_e[s] = cur
            assert (ds.view(-1, S)[b].cpu().numpy() == exp_s).all(), (S, b)
            assert (de.view(-1, S)[b].cpu().numpy() == exp_e).all(), (S, b)


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("dh,H,alibi,S,pair", MATRIX)
def test_doc_attention_matches_oracle(dh, H, alibi, S, pair):
    B = 2
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=S + dh + H + 11)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    sid = _sid(pair, S)
    ds, de = _bounds(sid)
    out, lse = _fwd(qkv, H, scale, slopes, ds)
    dqkv = _bwd(qkv, out, dout, lse, H, scale, slopes, ds, de)
    torch.cuda.synchronize()
    for name, t in (("o", out), ("lse", lse), ("dqkv", dqkv)):
        assert bool(torch.isfinite(t).all()), f"{name}: an element was never written or is not finite"
    ref, base = _refs(qkv, dout, H, scale, slopes, sid)
    case = f"{pair[0]}+{pair[1]}"
    dev = A.Deviations()
    A.check("o", A.heads(out, H), ref.o, base.o, case=case)
    A.check_lse(lse, ref.lse, LSE_ATOL, case=case)
    dq, dk, dv = A.split_heads(dqkv, H)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        _check(name, got, getattr(ref, name), getattr(base, name), case, (case, dh, S) if not alibi else None, dev)
    dev.report()


@pytest.mark.parametrize("dh,H,alibi", [(64, 12, False), (64, 12, True), (128, 16, False), (128, 16, True)])
@pytest.mark.parametrize("S", [384, 2048])
def test_one_document_per_row_equals_causal(dh, H, alibi, S):
    """The mask path with one document per row: O, LSE, dK and dV bitwise those of the plain causal kernel."""
    B = 2
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=S + dh + 5)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    sid = _sid(("one", "one"), S)
    ds, de = _bounds(sid)
    out, lse = _fwd(qkv, H, scale, slopes)
    out_d, lse_d = _fwd(qkv, H, scale, slopes, ds)
    dqkv = _bwd(qkv, out, dout, lse, H, scale, slopes)
    dqkv_d = _bwd(qkv, out_d, dout, lse_d, H, scale, slopes, ds, de)
    torch.cuda.synchronize()
    assert torch.equal(out, out_d) and torch.equal(lse, lse_d)
    d = H * dh
    assert torch.equal(dqkv[..., d:], dqkv_d[..., d:]), "dK / dV differ from the causal kernel"
    ref, base = _refs(qkv, dout, H, scale, slopes, sid)
    A.check("dq", A.split_heads(dqkv_d, H)[0], ref.dq, base.dq, case="one document")


@pytest.mark.parametrize("dh,H", [(64, 12), (128, 16)])
def test_documents_are_isolated(dh, H):
    """New q / k / v for one document leave the O rows of every other document, and the dK / dV rows of their keys,
    bitwise unchanged."""
    B, S = 2, 2048
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=dh + 3)
    scale = 1.0 / math.sqrt(dh)
    sid = _sid(("mid_tile", "c4"), S)
    ds, de = _bounds(sid)
    out, lse = _fwd(qkv, H, scale, None, ds)
    dqkv = _bwd(qkv, out, dout, lse, H, scale, None, ds, de)
    for b in range(B):
        doc = int(sid[b, S // 2])            # the document in the middle of the row
        rows = sid[b] == doc
        other = qkv.clone()
        g = torch.Generator(device="cpu").manual_seed(b)
        other[b, rows] = torch.randn(int(rows.sum()), qkv.shape[-1], generator=g).to(DEV).bfloat16()
        out2, lse2 = _fwd(other, H, scale, None, ds)
        dqkv2 = _bwd(other, out2, dout, lse2, H, scale, None, ds, de)
        torch.cuda.synchronize()
        keep = ~rows
        d = H * dh
        assert not torch.equal(out2[b, rows], out[b, rows])
        assert torch.equal(out2[b, keep], out[b, keep]), "O of another document changed"
        assert torch.equal(dqkv2[b, keep, d:], dqkv[b, keep, d:]), "dK / dV of another document's keys changed"
        assert torch.equal(out2[1 - b], out[1 - b]) and torch.equal(dqkv2[1 - b, :, d:], dqkv[1 - b, :, d:])


@pytest.mark.parametrize("dh,H,alibi", [(64, 12, False), (128, 16, True)])
def test_skipped_key_tiles_are_never_read(dh, H, alibi):
    """A document ending on a 128-row edge gets NaN keys and values. Every later document must not see them, forward or
    backward: the plain causal kernel would (P = 0 times a NaN V is still NaN), the masked one skips those tiles."""
    B, S, edge = 2, 2048, 512
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=dh + 9)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    starts = [[100, edge, edge + 70, 1300], [edge, 900]]   # the NaN document: [100, 512) in row 0, [0, 512) in row 1
    sid = torch.from_numpy(np.stack([_ids_from_starts(S, s) for s in starts])).to(DEV)
    ds, de = _bounds(sid)
    d = H * dh
    poisoned = qkv.clone()
    poisoned[0, 100:edge, d:] = NAN
    poisoned[1, :edge, d:] = NAN
    out, lse = _fwd(poisoned, H, scale, slopes, ds)
    dqkv = _bwd(poisoned, out, dout, lse, H, scale, slopes, ds, de)
    torch.cuda.synchronize()
    later = slice(edge, S)
    assert bool(torch.isfinite(out[:, later]).all()) and bool(torch.isfinite(lse[:, :, later]).all())
    assert bool(torch.isfinite(dqkv[:, later]).all()), "dQ / dK / dV of later documents saw the NaN tiles"
    # the later documents do not depend on the poisoned keys: the references come from the clean inputs
    ref, base = _refs(qkv, dout, H, scale, slopes, sid)
    A.check("o", _rows(A.heads(out, H), edge), _rows(ref.o, edge), _rows(base.o, edge), case="after NaN document")
    A.check_lse(lse[:, :, later], ref.lse[:, :, later], LSE_ATOL, case="after NaN document")
    dq, dk, dv = A.split_heads(dqkv, H)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        A.check(name, _rows(got, edge), _rows(getattr(ref, name), edge), _rows(getattr(base, name), edge), case="after NaN document")


# ------------------------------------------------------------------------------------------------ bindings
def test_bindings_reject_malformed_document_masks():
    from photon_b200 import ops

    B, S, H, dh = 1, 256, 4, 64
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV)
    out = torch.empty(B, S, H * dh, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, S, device=DEV)
    ds, de = _bounds(torch.zeros(B, S, dtype=torch.int64, device=DEV))
    ops.attention_fwd(qkv, out, lse, H, 0.125, True, None, ds)
    bad = {
        "dtype": ds.long(),
        "shape": ds[:-1],
        "device": ds.cpu(),
        "strides": torch.zeros(2 * B * S, dtype=torch.int32, device=DEV)[::2],
    }
    for why, t in bad.items():
        with pytest.raises(RuntimeError):
            ops.attention_fwd(qkv, out, lse, H, 0.125, True, None, t)
        with pytest.raises(RuntimeError):
            ops.attention_bwd(qkv, out, dout, lse, torch.empty_like(qkv), torch.empty_like(lse), H, 0.125, True, None, t, de)
        with pytest.raises(RuntimeError):
            ops.attention_bwd(qkv, out, dout, lse, torch.empty_like(qkv), torch.empty_like(lse), H, 0.125, True, None, ds, t)
    with pytest.raises(RuntimeError, match="causal"):
        ops.attention_fwd(qkv, out, lse, H, 0.125, False, None, ds)
    with pytest.raises(RuntimeError, match="causal"):
        ops.attention_bwd(qkv, out, dout, lse, torch.empty_like(qkv), torch.empty_like(lse), H, 0.125, False, None, ds, de)
    with pytest.raises(RuntimeError, match="doc_end without doc_start"):
        ops.attention_bwd(qkv, out, dout, lse, torch.empty_like(qkv), torch.empty_like(lse), H, 0.125, True, None, None, de)
    with pytest.raises(RuntimeError):
        ops.attention_bwd(qkv, out, dout, lse, torch.empty_like(qkv), torch.empty_like(lse), H, 0.125, True, None, ds, None)
    sid = torch.zeros(B, S, dtype=torch.int64, device=DEV)
    strided = torch.zeros(B, 2 * S, dtype=torch.int64, device=DEV)[:, ::2]
    for args in ((sid.int(), ds, de), (sid, ds[:-1], de), (sid, ds, de.long()), (strided, ds, de), (sid.cpu(), ds, de)):
        with pytest.raises(RuntimeError):
            ops.doc_bounds(*args)
    torch.cuda.synchronize()
