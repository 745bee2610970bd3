"""wgmma flash attention (fwd + bwd) tile by tile against an fp64 oracle, with a bf16 baseline setting each tile's bound.

See ``attention_oracle`` for the criterion. Every run also checks coverage (outputs start as NaN and must all be written),
isolation (NaN in the other batch rows and heads must not change a clean (b, h)) and repeatability (forward, dK and dV
bitwise; dQ accumulates with float atomics, so it only has to stay within the criterion).
"""
import math

import pytest
import torch

import attention_oracle as A

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN = float("nan")
# fp32 LSE vs the fp64 oracle. Scores come from exact bf16 products summed in fp32 and the softmax runs in exp2 with fp32
# sums, so the LSE error is a few fp32 ulps of |LSE| (<= 40 for the peaked inputs at S = 2048).
LSE_ATOL = 1e-4

# (d_head, heads, causal, alibi): the four template instances, causal and not, at the head counts of the real models
MODES = [(64, 12, True, False), (64, 12, True, True), (64, 12, False, False),
         (128, 16, True, False), (128, 20, True, True), (128, 16, False, False)]
# one diagonal tile, an odd tile count, the configs' max_seq_len
SEQS = [128, 384, 2048]
MATRIX = [pytest.param(dh, H, causal, alibi, S, case, id=f"dh{dh}-h{H}-{'causal' if causal else 'full'}{'-alibi' if alibi else ''}-s{S}-{case}")
          for dh, H, causal, alibi in MODES for S in SEQS for case in A.CASES]


def _slopes(H, alibi):
    from photon_b200.models.mpt import alibi_slopes

    return alibi_slopes(H).to(DEV) if alibi else None


def _fwd(qkv, H, scale, causal, slopes):
    from photon_b200 import ops

    B, S, d3 = qkv.shape
    out = torch.full((B, S, d3 // 3), NAN, dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, S), NAN, dtype=torch.float32, device=DEV)
    ops.attention_fwd(qkv, out, lse, H, scale, causal, slopes)
    return out, lse


def _bwd(qkv, out, dout, lse, H, scale, causal, slopes):
    from photon_b200 import ops

    dqkv = torch.full_like(qkv, NAN)
    delta = torch.full_like(lse, NAN)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, causal, slopes)
    return dqkv, delta


def _refs(qkv, dout, H, scale, causal, slopes):
    q, k, v = A.split_heads(qkv, H)
    do = None if dout is None else A.heads(dout, H)
    sl = None if slopes is None else slopes.tolist()
    kw = dict(causal=causal, slopes=sl, dout=do)
    return A.oracle(q, k, v, scale, **kw), A.baseline(q, k, v, scale, **kw)


def _grads(dqkv, H):
    return A.split_heads(dqkv, H)


def _check_grads(dqkv, ref, base, H, case, dev):
    dq, dk, dv = _grads(dqkv, H)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        A.check(name, got, getattr(ref, name), getattr(base, name), case=case, deviations=dev)


def _all_finite(name, *ts):
    for t in ts:
        assert bool(torch.isfinite(t).all()), f"{name}: an output element was never written (NaN left from the fill) or is not finite"


@pytest.mark.parametrize("dh,H,causal,alibi,S,case", MATRIX)
def test_attention_fwd(dh, H, causal, alibi, S, case):
    B = 1
    qkv, _ = A.make_inputs(case, B, S, H, dh, DEV, seed=S + dh + H)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    out, lse = _fwd(qkv, H, scale, causal, slopes)
    out2, lse2 = _fwd(qkv, H, scale, causal, slopes)
    torch.cuda.synchronize()
    _all_finite("fwd", out, lse)
    assert torch.equal(out, out2) and torch.equal(lse, lse2), "the forward is not bitwise repeatable"
    ref, base = _refs(qkv, None, H, scale, causal, slopes)
    A.check("o", A.heads(out, H), ref.o, base.o, case=case)
    A.check_lse(lse, ref.lse, LSE_ATOL, case=case)


@pytest.mark.parametrize("dh,H,causal,alibi,S,case", MATRIX)
def test_attention_bwd(dh, H, causal, alibi, S, case):
    B = 1
    qkv, dout = A.make_inputs(case, B, S, H, dh, DEV, seed=S + dh + H + 1)
    slopes = _slopes(H, alibi)
    scale = 1.0 / math.sqrt(dh)
    out, lse = _fwd(qkv, H, scale, causal, slopes)
    dqkv, delta = _bwd(qkv, out, dout, lse, H, scale, causal, slopes)
    dqkv2, _ = _bwd(qkv, out, dout, lse, H, scale, causal, slopes)
    torch.cuda.synchronize()
    _all_finite("bwd", dqkv, delta)
    ref, base = _refs(qkv, dout, H, scale, causal, slopes)
    dev = A.Deviations()
    _check_grads(dqkv, ref, base, H, case, dev)
    _check_grads(dqkv2, ref, base, H, case + ", second run", dev)
    d = H * dh
    assert torch.equal(dqkv[..., d:], dqkv2[..., d:]), "dK / dV are not bitwise repeatable"
    _check_isolation(qkv, dout, H, scale, causal, slopes, ref, base, case, dev)
    dev.report()


def _check_isolation(qkv, dout, H, scale, causal, slopes, ref, base, case, dev, b0=None, h0=None):
    """NaN everywhere but one (b, h): its outputs must equal, bit for bit, those of a run holding that (b, h) alone."""
    B, S, d3 = qkv.shape
    d = d3 // 3
    dh = d // H
    b0 = B - 1 if b0 is None else b0
    h0 = H - 1 if h0 is None else h0
    x5, g4 = qkv.view(B, S, 3, H, dh), dout.view(B, S, H, dh)
    poisoned = torch.full_like(x5, NAN)
    poisoned[b0, :, :, h0] = x5[b0, :, :, h0]
    dpois = torch.full_like(g4, NAN)
    dpois[b0, :, h0] = g4[b0, :, h0]
    poisoned, dpois = poisoned.view(B, S, d3), dpois.view(B, S, d)
    out, lse = _fwd(poisoned, H, scale, causal, slopes)
    dqkv, _ = _bwd(poisoned, out, dpois, lse, H, scale, causal, slopes)
    alone = x5[b0:b0 + 1, :, :, h0:h0 + 1].reshape(1, S, 3 * dh).contiguous()
    dalone = g4[b0:b0 + 1, :, h0:h0 + 1].reshape(1, S, dh).contiguous()
    s1 = None if slopes is None else slopes[h0:h0 + 1].contiguous()
    out1, lse1 = _fwd(alone, 1, scale, causal, s1)
    dqkv1, _ = _bwd(alone, out1, dalone, lse1, 1, scale, causal, s1)
    torch.cuda.synchronize()
    got = dqkv.view(B, S, 3, H, dh)[b0, :, :, h0]
    want = dqkv1.view(S, 3, dh)
    assert torch.equal(out.view(B, S, H, dh)[b0, :, h0], out1.view(S, dh)), f"O of (b={b0}, h={h0}) depends on other heads or rows"
    assert torch.equal(lse[b0, h0], lse1[0, 0]), f"LSE of (b={b0}, h={h0}) depends on other heads or rows"
    assert torch.equal(got[:, 1:], want[:, 1:]), f"dK / dV of (b={b0}, h={h0}) depend on other heads or rows"
    sl = (slice(b0, b0 + 1), slice(h0, h0 + 1))
    A.check("dq", got[:, 0][None, None], ref.dq[sl], base.dq[sl], case=case + f", isolated (b={b0}, h={h0})", deviations=dev)


# (B, S, H, causal, dh): more CTAs than SMs, so several waves of (tile, batch*head) CTAs run, causal and not
MANY = [(4, 1024, 12, True, 64), (8, 512, 12, True, 64), (3, 768, 5, True, 64), (4, 512, 12, False, 64), (2, 1024, 3, False, 64),
        (4, 1024, 16, True, 128), (2, 512, 8, False, 128), (2, 2048, 20, True, 128), (2, 2048, 20, False, 128)]


@pytest.mark.parametrize("B,S,H,causal,dh", MANY)
def test_attention_persistent_many_items(B, S, H, causal, dh):
    """Multi-wave grids (B = 2, H = 20, S = 2048 is 640 CTAs on 132 SMs): every (b, h) and tile checked, plus coverage,
    repeatability and the isolation of one (b, h) in the middle of the grid."""
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=B * S + H)
    scale = 1.0 / math.sqrt(dh)
    out, lse = _fwd(qkv, H, scale, causal, None)
    dqkv, delta = _bwd(qkv, out, dout, lse, H, scale, causal, None)
    out2, lse2 = _fwd(qkv, H, scale, causal, None)
    dqkv2, _ = _bwd(qkv, out, dout, lse, H, scale, causal, None)
    torch.cuda.synchronize()
    _all_finite("fwd / bwd", out, lse, dqkv, delta)
    assert torch.equal(out, out2) and torch.equal(lse, lse2), "the forward is not bitwise repeatable"
    assert torch.equal(dqkv[..., H * dh:], dqkv2[..., H * dh:]), "dK / dV are not bitwise repeatable"
    ref, base = _refs(qkv, dout, H, scale, causal, None)
    A.check("o", A.heads(out, H), ref.o, base.o, case="normal")
    A.check_lse(lse, ref.lse, LSE_ATOL, case="normal")
    _check_grads(dqkv, ref, base, H, "normal", None)
    _check_grads(dqkv2, ref, base, H, "normal, second run", None)
    _check_isolation(qkv, dout, H, scale, causal, None, ref, base, "normal", None, b0=B // 2, h0=H // 2)


@pytest.mark.parametrize("B,S,H,dh", [(2, 512, 4, 64), (1, 1024, 3, 128), (2, 2048, 12, 64), (1, 2048, 16, 128)])
def test_attention_alibi_fwd_bwd(B, S, H, dh):
    """attn_config.alibi: score += slope_h * (key - query) inside both kernels, with the slopes the models use (bias max 8),
    at several batch rows and head counts (the input cases at one batch row are in test_attention_fwd / _bwd)."""
    slopes = _slopes(H, True)
    scale = 1.0 / math.sqrt(dh)
    qkv, dout = A.make_inputs("normal", B, S, H, dh, DEV, seed=B + S + H)
    out, lse = _fwd(qkv, H, scale, True, slopes)
    dqkv, delta = _bwd(qkv, out, dout, lse, H, scale, True, slopes)
    torch.cuda.synchronize()
    _all_finite("fwd / bwd", out, lse, dqkv, delta)
    ref, base = _refs(qkv, dout, H, scale, True, slopes)
    A.check("o", A.heads(out, H), ref.o, base.o, case="normal")
    A.check_lse(lse, ref.lse, LSE_ATOL, case="normal")
    _check_grads(dqkv, ref, base, H, "normal", None)


# ------------------------------------------------------------------------------------------------ argument checks
def _args(B=1, S=128, H=2, dh=64):
    d = H * dh
    qkv = torch.zeros(B, S, 3 * d, dtype=torch.bfloat16, device=DEV)
    return dict(qkv=qkv, out=torch.zeros(B, S, d, dtype=torch.bfloat16, device=DEV),
                lse=torch.zeros(B, H, S, dtype=torch.float32, device=DEV), dout=torch.zeros(B, S, d, dtype=torch.bfloat16, device=DEV),
                dqkv=torch.zeros_like(qkv), delta=torch.zeros(B, H, S, dtype=torch.float32, device=DEV), H=H, causal=True, slopes=None)


def _bad(kind):
    a = _args()
    if kind == "out_shape":
        a["out"] = a["out"][:, :, :64]
    elif kind == "out_strided":
        a["out"] = torch.zeros(1, 256, 128, dtype=torch.bfloat16, device=DEV)[:, ::2]
    elif kind == "dout_shape":
        a["dout"] = torch.zeros(1, 128, 64, dtype=torch.bfloat16, device=DEV)
    elif kind == "lse_shape":
        a["lse"] = torch.zeros(1, 128, 2, dtype=torch.float32, device=DEV)
    elif kind == "lse_strided":
        a["lse"] = torch.zeros(1, 128, 2, dtype=torch.float32, device=DEV).transpose(1, 2)
    elif kind == "delta_shape":
        a["delta"] = torch.zeros(1, 2, 64, dtype=torch.float32, device=DEV)
    elif kind == "dqkv_shape":
        a["dqkv"] = torch.zeros(1, 128, 2 * 128, dtype=torch.bfloat16, device=DEV)
    elif kind == "dqkv_strided":
        a["dqkv"] = torch.zeros(1, 256, 3 * 128, dtype=torch.bfloat16, device=DEV)[:, ::2]
    elif kind == "heads_do_not_divide_d":
        a["H"] = 3
        a["lse"] = torch.zeros(1, 3, 128, dtype=torch.float32, device=DEV)
        a["delta"] = torch.zeros(1, 3, 128, dtype=torch.float32, device=DEV)
    elif kind == "alibi_not_causal":
        a["causal"] = False
        a["slopes"] = torch.ones(2, dtype=torch.float32, device=DEV)
    return a


FWD_BAD = ["out_shape", "out_strided", "lse_shape", "lse_strided", "heads_do_not_divide_d", "alibi_not_causal"]
BWD_BAD = FWD_BAD + ["dout_shape", "delta_shape", "dqkv_shape", "dqkv_strided"]


@pytest.mark.parametrize("kind", BWD_BAD)
def test_attention_bindings_reject_bad_arguments(kind):
    from photon_b200 import ops

    a = _bad(kind)
    n0 = ops.launch_count()
    if kind in FWD_BAD:
        with pytest.raises(RuntimeError):
            ops.attention_fwd(a["qkv"], a["out"], a["lse"], a["H"], 0.125, a["causal"], a["slopes"])
    with pytest.raises(RuntimeError):
        ops.attention_bwd(a["qkv"], a["out"], a["dout"], a["lse"], a["dqkv"], a["delta"], a["H"], 0.125, a["causal"], a["slopes"])
    torch.cuda.synchronize()
    assert ops.launch_count() == n0, "a kernel was launched before the argument check"
    good = _args()   # the same call with well-formed arguments goes through
    ops.attention_fwd(good["qkv"], good["out"], good["lse"], 2, 0.125, True)
    ops.attention_bwd(good["qkv"], good["out"], good["dout"], good["lse"], good["dqkv"], good["delta"], 2, 0.125, True)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 4


def test_rope_kernel_matches_oracle_and_inverts():
    from photon_b200 import ops
    from photon_b200.models.mpt import apply_rope, rope_tables

    B, S, H, dh = 2, 256, 4, 64
    d = H * dh
    qkv = torch.randn(B, S, 3 * d, device="cuda:0").to(torch.bfloat16)
    cos, sin = rope_tables(S, dh, 10000.0, "cuda:0")
    ref = qkv.float().view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)            # [3, B, H, S, dh]
    rq, rk = apply_rope(ref[0], cos, sin), apply_rope(ref[1], cos, sin)
    work = qkv.clone()
    ops.rope_(work, cos.contiguous(), sin.contiguous(), H)
    got = work.float().view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    assert (got[0] - rq).abs().max().item() < 3e-2 and (got[1] - rk).abs().max().item() < 3e-2
    assert torch.equal(got[2], ref[2])                                        # v untouched
    ops.rope_(work, cos.contiguous(), sin.contiguous(), H, inverse=True)      # rotation is orthogonal
    assert (work.float() - qkv.float()).abs().max().item() < 6e-2
