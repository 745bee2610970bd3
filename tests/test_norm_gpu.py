"""RMSNorm (``model.norm_type``) on the sm_90a kernels: the RMS instances of the row kernels against fp64 references on every
dispatch path, their launches, the engine against the fp32 PyTorch model, its own paths (checkpointing, CUDA graphs, amp_fp8,
full parameter sharding) and the KV-cached decoder and scorer."""
import pytest
import torch

import fused_oracle as fo
from test_ffn_gpu import LOGP_TOL, _ids, _match, _pair, _prompts
from test_fused_ops_gpu import _guard_intact, _guarded, _randn, _same_bits
from test_launch_count_gpu import _kernels_and_count

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
F64 = torch.float64
EPS = 1e-5


def _ops():
    from photon_b200 import ops

    return ops


# ------------------------------------------------------------------------------------------------ fp64 references
def rmsnorm_fwd_ref(x, g, eps, rstd=None):
    """y, rstd of ``y = x · rstd · g``, ``rstd = rsqrt(mean(x²) + eps)``; given ``rstd`` (the kernel's), y uses it."""
    xd = x.to(F64)
    rs = torch.rsqrt((xd * xd).mean(-1) + eps)
    r_use = rs if rstd is None else rstd.to(F64).reshape(rs.shape)
    return xd * r_use[..., None] * g.to(F64), rs


def rstd_rel_tol(d):
    """The per-lane chain of x² sums (as ``fo.ln_chain``), the squares, and rsqrtf (2 ulp)."""
    return (fo.ln_chain(d) + 10) * fo.EPS32


def fwd_floor(x, g, rstd):
    """fp32 error of ``x * rstd * g`` (two roundings, with the slack of ``fo.ln_fwd_floor``)."""
    return 4 * fo.EPS32 * (x.to(F64) * rstd.to(F64)[:, None] * g.to(F64)).abs()


def rmsnorm_bwd_ref(dy, x, g, rstd, dres=None):
    """dx (+ dres) and dgamma for the given rstd, the fp32 floor of dx and the sum of |terms| of each dgamma column."""
    d = x.shape[-1]
    xd, dyd, gd, rs = x.to(F64), dy.to(F64), g.to(F64), rstd.to(F64)[:, None]
    xh = xd * rs
    dyg = dyd * gd
    c2 = (dyg * xh).mean(-1, keepdim=True)
    dx = rs * (dyg - xh * c2)
    if dres is not None:
        dx = dx + dres.to(F64)
    c2_err = (fo.ln_chain(d) + 5) * fo.EPS32 * (dyg * xh).abs().mean(-1, keepdim=True)
    floor = rs * (4 * fo.EPS32 * (dyg.abs() + (xh * c2).abs()) + xh.abs() * c2_err) + 2 * fo.EPS32 * dx.abs()
    return dx, (dyd * xh).sum(0), floor, (dyd * xh).abs().sum(0)


# ------------------------------------------------------------------------------------------------ kernels
NORM_D = [256, 768, 1024, 2048, 2560, 4096]
NORM_T = [9, 8193]


def _inputs(T, d, seed):
    x = _randn(T, d, seed=seed, scale=1.5, offset=0.3)
    g = torch.rand(d, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + 1)) + 0.5
    return x, g


def _fwd(x, g):
    T, d = x.shape
    ybuf, y = _guarded((T, d), torch.bfloat16)
    rbuf, rstd = _guarded((T,), torch.float32)
    gbuf, gv = _guarded((d,), torch.float32, g)
    _ops().rmsnorm_fwd(x, gv, y, rstd, EPS)
    for buf, n in ((ybuf, "y"), (rbuf, "rstd"), (gbuf, "gamma")):
        _guard_intact(buf, f"rmsnorm_fwd {n}")
    return y, rstd


@pytest.mark.parametrize("T", NORM_T)
@pytest.mark.parametrize("d", NORM_D)
def test_rmsnorm_fwd_and_bwd(d, T):
    """Forward (``ln_fwd_kernel<N, true>``); backward with dgamma at d <= 1024 on the one-pass ``ln_bwd_fused_kernel<N, true>``
    (persistent at T = 8193), otherwise and without dgamma on ``ln_bwd_dx_kernel<N, true>`` (+ ``col_reduce_kernel<true>``).
    Every combination of dres and dgamma; dgamma accumulates into a non-zero value."""
    ops = _ops()
    x, g = _inputs(T, d, seed=d * 7 + T)
    what = f"rmsnorm d={d} T={T}"
    y, rstd = _fwd(x, g)
    _, rs = rmsnorm_fwd_ref(x, g, EPS)
    fo.assert_within(rstd.to(F64) / rs, torch.ones_like(rs), rstd_rel_tol(d), f"{what} rstd / fp64 rstd")
    ref, _ = rmsnorm_fwd_ref(x, g, EPS, rstd=rstd)
    fo.assert_within(y, ref, fo.bf16_tol(ref, fwd_floor(x, g, rstd)), f"{what} y")
    y2, rstd2 = _fwd(x, g)
    _same_bits(y2, y, f"{what} y")
    _same_bits(rstd2, rstd, f"{what} rstd")
    dy = _randn(T, d, seed=d + T + 5)
    dres = _randn(T, d, seed=d + T + 6)
    for use_dres in (True, False):
        for want_dg in (True, False):
            dr = dres if use_dres else None
            tag = f"{what} dres={use_dres} dgamma={want_dg}"
            ref_dx, ref_dg, floor, abs_dg = rmsnorm_bwd_ref(dy, x, g, rstd, dr)
            outs = []
            for _ in range(2):
                dxbuf, dx = _guarded((T, d), torch.bfloat16)
                g0 = torch.randn(d, device=DEV, generator=torch.Generator(device=DEV).manual_seed(d)) if want_dg else None
                dgbuf, dg = _guarded((d,), torch.float32, g0) if want_dg else (None, None)
                ops.rmsnorm_bwd(dy, x, g, rstd, dr, dx, dg)
                for buf, n in ((dxbuf, "dx"), (dgbuf, "dgamma")):
                    if buf is not None:
                        _guard_intact(buf, f"{tag} {n}")
                fo.assert_within(dx, ref_dx, fo.bf16_tol(ref_dx, floor), f"{tag} dx")
                if want_dg:
                    fo.assert_within(dg, g0.to(F64) + ref_dg, fo.sum_tol(g0.to(F64).abs() + abs_dg, fo.colsum_depth(T)),
                                     f"{tag} dgamma")
                outs.append(dx)
            _same_bits(outs[1], outs[0], f"{tag} dx")


@pytest.mark.parametrize("d", NORM_D)
def test_rmsnorm_fwd_q8(d):
    """``ln_fwd_q8_kernel<N, true>``: E4M3 bytes within one E4M3 ulp of the fp64 RMSNorm times the scale (some values saturate
    at 448), rstd as the bf16 forward, the amax of the unscaled output, and the same bytes from a second run."""
    T = 1001
    x, g = _inputs(T, d, seed=d + 3)
    ref, rs = rmsnorm_fwd_ref(x, g, EPS)
    amax_ref = ref.abs().max().item()
    s = 448.0 / amax_ref * 1.25
    what = f"rmsnorm_fwd_q8 d={d}"
    runs = []
    for _ in range(2):
        meta = torch.zeros(3, 2, device=DEV)
        meta[0], meta[1] = s, 1.0 / s
        ybuf, y8 = _guarded((T, d), torch.uint8)
        rbuf, rstd = _guarded((T,), torch.float32)
        _ops().rmsnorm_fwd_q8(x, g, y8, rstd, EPS, meta, 1)
        _guard_intact(ybuf, what)
        _guard_intact(rbuf, f"{what} rstd")
        runs.append((y8, rstd, meta))
    y8, rstd, meta = runs[0]
    fo.assert_within(rstd.to(F64) / rs, torch.ones_like(rs), rstd_rel_tol(d), f"{what} rstd / fp64 rstd")
    want = (ref * float(torch.tensor(s, dtype=torch.float32))).clamp(-448.0, 448.0)
    fo.assert_within(y8.view(torch.float8_e4m3fn).to(F64), want, fo.e4m3_ulp(want), f"{what} E4M3 bytes")
    err = (ref.abs() * rstd_rel_tol(d) + fwd_floor(x, g, rs)).max().item()
    assert abs(meta[2, 1].item() - amax_ref) <= err, f"{what} amax {meta[2, 1].item()!r} vs {amax_ref!r} (tol {err:.3g})"
    assert meta[2, 0].item() == 0.0
    _same_bits(runs[1][0], y8, f"{what} bytes")
    _same_bits(runs[1][1], rstd, f"{what} rstd")


def test_rmsnorm_bindings_reject_unsupported_rows():
    ops = _ops()
    meta = torch.ones(3, 2, device=DEV)
    for d in (100, 4104):   # d % 8 != 0, d > 4096
        x = _randn(4, d, seed=1)
        g, r = torch.ones(d, device=DEV), torch.empty(4, device=DEV)
        y = torch.empty_like(x)
        with pytest.raises(RuntimeError, match="rmsnorm"):
            ops.rmsnorm_fwd(x, g, y, r)
        with pytest.raises(RuntimeError, match="rmsnorm"):
            ops.rmsnorm_bwd(x, x, g, r, None, y, None)
        with pytest.raises(RuntimeError, match="rmsnorm"):
            ops.rmsnorm_bwd(x, x, g, r, None, y, torch.zeros(d, device=DEV))
        with pytest.raises(RuntimeError, match="rmsnorm_fwd_q8"):
            ops.rmsnorm_fwd_q8(x, g, torch.empty(4, d, dtype=torch.uint8, device=DEV), r, 1e-5, meta, 0)
    x = _randn(4, 256, seed=2)
    y, r = torch.empty_like(x), torch.empty(4, device=DEV)
    short = torch.ones(248, device=DEV)   # gamma of the wrong length
    with pytest.raises(RuntimeError, match="rmsnorm_fwd"):
        ops.rmsnorm_fwd(x, short, y, r)
    with pytest.raises(RuntimeError, match="rmsnorm_bwd"):
        ops.rmsnorm_bwd(x, x, short, r, None, y, None)
    with pytest.raises(RuntimeError, match="rmsnorm_bwd"):
        ops.rmsnorm_bwd(x, x, torch.ones(256, device=DEV), r, None, y, torch.zeros(248, device=DEV))
    with pytest.raises(RuntimeError, match="rmsnorm_fwd_q8"):
        ops.rmsnorm_fwd_q8(x, short, torch.empty(4, 256, dtype=torch.uint8, device=DEV), r, 1e-5, meta, 0)
    with pytest.raises(RuntimeError, match="rmsnorm_fwd"):
        ops.rmsnorm_fwd(x, torch.ones(256, device=DEV), y, torch.empty(3, device=DEV))   # rstd of the wrong length


# ------------------------------------------------------------------------------------------------ launch counts
@pytest.mark.parametrize("d,dgamma,n", [(768, True, 1), (768, False, 1), (2048, True, 2), (2048, False, 1)])
def test_rms_ops_launch_what_their_layernorm_counterparts_do(d, dgamma, n):
    ops = _ops()
    T = 256
    x, dy = _randn(T, d, seed=3), _randn(T, d, seed=4)
    g = torch.ones(d, device=DEV)
    y, mean, rstd = torch.empty_like(x), torch.empty(T, device=DEV), torch.empty(T, device=DEV)
    dg = torch.zeros(d, device=DEV) if dgamma else None
    meta = torch.ones(3, 2, device=DEV)
    y8 = torch.empty(T, d, dtype=torch.uint8, device=DEV)
    pairs = {"fwd": (lambda: ops.layernorm_fwd(x, g, None, y, mean, rstd), lambda: ops.rmsnorm_fwd(x, g, y, rstd)),
             "fwd_q8": (lambda: ops.layernorm_fwd_q8(x, g, None, y8, mean, rstd, EPS, meta, 0),
                        lambda: ops.rmsnorm_fwd_q8(x, g, y8, rstd, EPS, meta, 0)),
             "bwd": (lambda: ops.layernorm_bwd(dy, x, g, mean, rstd, None, y, dg, None),
                     lambda: ops.rmsnorm_bwd(dy, x, g, rstd, None, y, dg))}
    for op, (ln, rms) in pairs.items():
        k_ln, n_ln = _kernels_and_count(ln)
        k_rms, n_rms = _kernels_and_count(rms)
        assert n_rms == n_ln == len(k_rms) == len(k_ln), (op, k_ln, k_rms)
        assert all("true>" in k for k in k_rms) and not any("true>" in k for k in k_ln), (op, k_rms)
    assert _kernels_and_count(pairs["bwd"][1])[1] == n


# ------------------------------------------------------------------------------------------------ engine vs fp32 model
VARIANTS = {"plain": {}, "qkln_gqa_rope": dict(qk_ln=True, kv_n_heads=2, rope=True, learned_pos_emb=False),
            "llama": dict(ffn_type="mptglu", ffn_act="silu", rope=True, learned_pos_emb=False, kv_n_heads=2, no_bias=True),
            "llama_doc": dict(ffn_type="mptglu", ffn_act="silu", rope=True, learned_pos_emb=False, kv_n_heads=2, no_bias=True,
                              attn_uses_sequence_id=True)}
NORM_WEIGHTS = ["transformer.blocks.0.norm_1.weight", "transformer.blocks.1.norm_2.weight", "transformer.norm_f.weight",
                "transformer.blocks.0.attn.q_ln.weight", "transformer.blocks.1.attn.k_ln.weight"]


def _cfg(norm_type="rmsnorm", **kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=512, n_heads=8, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch", norm_type=norm_type,
                norm_eps=1e-6)
    return MPTConfig(**{**base, **kw})


def _check_norm_grads(ref, eng, tol=0.08):
    """Per-tensor relative distance of the norm weights' gradients (after ``_match``); returns how many were checked."""
    lay = eng.flat.layout
    checked = 0
    for name in NORM_WEIGHTS:
        if name in lay.names:
            a, b = lay.view(ref.flat.grads, name), lay.view(eng.flat.grads, name)
            assert a.norm() > 0 and ((a - b).norm() / a.norm()).item() < tol, name
            checked += 1
    return checked


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_rmsnorm_engine_matches_torch(variant):
    cfg = _cfg(**VARIANTS[variant])
    ref, eng = _pair(cfg)
    assert eng.attn_mode == "b200" and eng.layers[0].b1 is None and eng.bf is None
    sid = None
    if cfg.attn_uses_sequence_id:
        from test_doc_engine_gpu import _batch

        ids, sid = _batch(4, 256, seed=1)
    else:
        ids = _ids(4, 256, 1)
    _match(ref, eng, ids, sid)
    assert _check_norm_grads(ref, eng) == (5 if cfg.qk_ln else 3)
    es = None if sid is None else sid[:2]
    a, b = ref.eval_stats(ids[:2], es), eng.eval_stats(ids[:2], es)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3


def test_rmsnorm_engine_with_frozen_norm_weights():
    """Frozen norm weights are read from the frozen planes and get no gradient; everything around them still trains."""
    frozen = ["transformer.blocks.0.norm_1.weight", "transformer.blocks.1.norm_2.weight", "transformer.norm_f.weight",
              "transformer.blocks.0.attn.q_ln.weight"]
    ref, eng = _pair(_cfg(qk_ln=True), frozen_layers=frozen)
    assert set(eng.frozen_layout.names) == set(frozen) and eng.flat.layout.names == ref.flat.layout.names
    assert eng.layers[0].d_g1 is None and eng.layers[1].d_g2 is None and eng.d_gf is None and eng.layers[0].d_qk_g[0] is None
    _match(ref, eng, _ids(4, 256, 3))
    assert _check_norm_grads(ref, eng) == 1   # blocks.1 k_ln


def test_rmsnorm_engine_launches_what_layernorm_does():
    """A LayerNorm's dbeta comes out of the launch of its dgamma, so dropping the norm bias removes no launch."""
    from photon_b200.models.engine import B200Engine

    for kw in ({}, dict(qk_ln=True, kv_n_heads=2)):
        n = {}
        for norm_type in ("layernorm", "rmsnorm"):
            e = B200Engine(_cfg(norm_type, **kw), DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
            e.fwd_bwd(_ids(2, 256, 0), 510.0)
            n[norm_type] = e.launches_per_microbatch
        assert n["rmsnorm"] == n["layernorm"] > 0, (kw, n)


# ------------------------------------------------------------------------------------------------ the engine's own paths
def test_rmsnorm_engine_activation_checkpointing_and_graphs():
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(n_layers=3, qk_ln=True, ffn_type="mptglu", ffn_act="silu", no_bias=True)
    eager = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
    ckpt = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5, activation_checkpointing=True)
    graph = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": True}, seed=5)
    denom = float(2 * 255)
    for e in (eager, ckpt, graph):
        e.flat.zero_grad()
    for s in range(3):
        ids = _ids(2, 256, 10 + s)
        losses = [float(e.fwd_bwd(ids, denom)[0]) for e in (eager, ckpt, graph)]
        torch.cuda.synchronize()
        assert losses[0] == losses[1], losses
        assert abs(losses[0] - losses[2]) <= 1e-3 * abs(losses[0]), losses
    assert len(graph._graphs) == 1   # noqa: SLF001
    assert graph.launches_per_microbatch == eager.launches_per_microbatch
    for e in (ckpt, graph):
        rel = ((eager.flat.grads - e.flat.grads).norm() / eager.flat.grads.norm()).item()
        assert rel < 1e-3, rel


@pytest.mark.parametrize("graph", [False, True])
def test_rmsnorm_engine_amp_fp8_tracks_bf16(graph):
    """Same weights, same batch: the fp8 engine (``rmsnorm_fwd_q8`` for both block norms) follows the bf16 engine as
    test_fp8_gpu.py's LayerNorm case does, the norm weights' gradients included."""
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(d_model=256, n_heads=4)
    e8 = B200Engine(cfg, DEV, "amp_fp8", {"cuda_graph": graph}, seed=3)
    e16 = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": graph}, seed=3)
    e8.flat.params.copy_(e16.flat.params)
    e8.params_updated()
    ids = _ids(4, 256, 7)
    for _ in range(2):
        for e in (e8, e16):
            e.flat.zero_grad()
        l8, n8 = e8.fwd_bwd(ids, 4.0 * 255)
        l16, n16 = e16.fwd_bwd(ids, 4.0 * 255)
    assert float(n8) == float(n16)
    assert abs(float(l8) - float(l16)) / float(l16) < 2e-2
    lay = e8.flat.layout
    for i, name in enumerate(lay.names):
        a, b = lay.view(e8.flat.grads, i).flatten().double(), lay.view(e16.flat.grads, i).flatten().double()
        cos = float((a @ b) / (a.norm() * b.norm()))
        if lay.numels[i] >= 256 * 256:
            assert cos > 0.95, (name, cos)
        elif "norm" in name:
            assert cos > 0.9, (name, cos)
    assert float((e8.fp8_meta[0, : e8._n_dyn] != 1.0).float().mean()) == 1.0   # noqa: SLF001


@pytest.mark.parametrize("precision", ["amp_bf16", "amp_fp8"])
def test_rmsnorm_sharded_engine_equals_plain_engine(precision):
    """A world-size-1 ZeRO-3 engine against the plain one (as test_zero3.py / test_zero3_fp8_gpu.py): the RMSNorm weights are
    1-D parameters like any other, so no special case is involved."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import NvlZero3Comm

    cfg = _cfg(d_model=256, n_heads=4, n_layers=3, attn_impl="flash", qk_ln=True)
    plain = B200Engine(cfg, DEV, precision, {"cuda_graph": False}, seed=5)
    comm = NvlZero3Comm(plain.flat.layout, cfg.n_layers, rank=0, world_size=1, device=DEV, fp8=precision == "amp_fp8")
    shard = B200Engine(cfg, DEV, precision, {}, seed=5, zero3=comm)
    assert torch.equal(shard.flat.full_params(), plain.flat.params)
    denom = float(4 * (cfg.max_seq_len - 1))
    plain.flat.zero_grad(), shard.flat.zero_grad()
    for s in range(2):
        ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device=DEV, generator=torch.Generator("cuda").manual_seed(s))
        la, na = plain.fwd_bwd(ids, denom)
        lb, nb = shard.fwd_bwd(ids, denom)
        assert float(na) == float(nb) and abs(float(la) - float(lb)) <= 1e-5 * abs(float(la)), (float(la), float(lb))
    torch.cuda.synchronize()
    full = torch.zeros_like(plain.flat.grads)
    comm.plan.shard_to_full(shard.flat.grads, 0, full)
    assert plain.flat.grads.abs().max() > 0
    rel = ((full - plain.flat.grads).norm() / plain.flat.grads.norm()).item()
    assert rel < (2e-3 if precision == "amp_fp8" else 1e-5), rel
    lay = plain.flat.layout
    for i, n in enumerate(lay.names):
        a, b = lay.view(plain.flat.grads, i), lay.view(full, i)
        assert (a - b).norm() <= (2e-2 if precision == "amp_fp8" else 1e-4) * a.norm() + 1e-9, n
    comm.close()


# ------------------------------------------------------------------------------------------------ decoding and scoring
LLAMA_QK = dict(ffn_type="mptglu", ffn_act="silu", rope=True, learned_pos_emb=False, kv_n_heads=2, no_bias=True, qk_ln=True)


def test_rmsnorm_decoder_follows_the_model():
    ref, eng = _pair(_cfg(**LLAMA_QK), kernels={"cuda_graph": True})
    prompts = _prompts()
    dec = eng.decoder(len(prompts))
    assert dec is not None
    seqs = [list(p) for p in prompts]
    follow = [True] * len(seqs)
    toks = dec.start(prompts, 16)
    for t in range(16):
        got = torch.log_softmax(dec.logits.float(), -1)
        for i, s in enumerate(seqs):
            with torch.no_grad():
                want = torch.log_softmax(ref.logits(torch.tensor([s], device=DEV))[0, -1].float(), -1)
            assert (got[i] - want).abs().max().item() < LOGP_TOL, (t, i)
            top2 = want.topk(2).values
            if follow[i] and (top2[0] - top2[1]).item() < LOGP_TOL:
                follow[i] = False
            if follow[i]:
                assert toks[i] == int(want.argmax()), (t, i)
            s.append(toks[i])
        if t < 15:
            toks = dec.step()


def test_rmsnorm_score_matches_the_model():
    from test_score_gpu import _fp32_stats, _pairs

    ref, eng = _pair(_cfg(**LLAMA_QK))
    pairs = _pairs(eng.cfg)
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (i, lp, want_lp)
        if clear:
            assert hit == want_hit, i
