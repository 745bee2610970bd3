"""Gated (``mptglu``) and SiLU feed-forward blocks on the sm_90a kernels: the new GEMM and skinny-GEMM epilogues against fp64
references, the engine against the fp32 PyTorch model, checkpointing / CUDA graphs / freeze lists, the decoder and scorer, and
the cases the engine refuses."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
EPI_BF16, EPI_RESIDUAL, EPI_SILU_GRAD, EPI_MUL2 = 0, 1, 8, 9
LOGP_TOL = 0.15   # as test_decode_gpu.py


# ------------------------------------------------------------------------------------------------ GEMM epilogues
# (A MN-major, B MN-major, epilogue, with bias): SiLU + derivative (forward), the two-multiplier epilogue as the gated up
# projection (K-major B, bias) and as the down projection's dgrad (MN-major B, no bias), the accumulating dgrad
CASES = [(0, 0, EPI_SILU_GRAD, True), (0, 0, EPI_MUL2, True), (0, 1, EPI_MUL2, False), (0, 1, EPI_RESIDUAL, False)]
SHAPES = [(520, 328, 208), (72, 584, 144)]   # the M / N / K tails of test_gemm_epilogue_gpu.py
OFF = 32


def _silu(z):
    return z * torch.sigmoid(z)


def _silu_grad(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def _run(amn, bmn, epi, with_bias, M, N, K, cluster):
    from photon_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(11)
    a = torch.randn(*((K, M) if amn else (M, K)), device=DEV, generator=g).bfloat16()
    b = (torch.randn(*((K, N) if bmn else (N, K)), device=DEV, generator=g) * 0.05).bfloat16()
    acc = (a.double().t() if amn else a.double()) @ (b.double() if bmn else b.double().t())
    bias = torch.randn(N, device=DEV, generator=g) * 0.1 if with_bias else None
    z = acc + (bias.double() if bias is not None else 0)
    aux = torch.randn(M, N, device=DEV, generator=g).bfloat16() if epi in (EPI_MUL2, EPI_RESIDUAL) else None
    aux2 = torch.randn(M, N, device=DEV, generator=g).bfloat16() if epi == EPI_MUL2 else None
    pad = 64 - N % 16
    outs = {"D": torch.full((M + 8, N + pad), -7.0, device=DEV, dtype=torch.bfloat16)}
    if epi in (EPI_SILU_GRAD, EPI_MUL2):
        outs["D2"] = torch.full((M + 8, N + pad), -5.0, device=DEV, dtype=torch.bfloat16)
    guards = {k: v.clone() for k, v in outs.items()}
    view = {k: v[:M, OFF:OFF + N] for k, v in outs.items()}
    ops.gemm(a, b, view["D"], a_mn=bool(amn), b_mn=bool(bmn), epi=epi, bias=bias, aux=aux, aux2=aux2, out2=view.get("D2"),
             cluster=cluster)
    torch.cuda.synchronize()
    if epi == EPI_SILU_GRAD:
        refs = {"D": _silu(z), "D2": _silu_grad(z)}
    elif epi == EPI_MUL2:
        refs = {"D": z * aux.double(), "D2": z * aux2.double()}
    else:
        refs = {"D": z + aux.double()}
    return outs, guards, view, refs


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("amn,bmn,epi,with_bias", CASES)
def test_ffn_gemm_epilogue(amn, bmn, epi, with_bias, cluster, M, N, K):
    outs, guards, view, refs = _run(amn, bmn, epi, with_bias, M, N, K, cluster)
    for k, buf in outs.items():
        inside = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
        inside[:M, OFF:OFF + N] = True
        assert torch.equal(buf[~inside], guards[k][~inside]), f"{k}: the epilogue wrote outside its output"
    for k, ref in refs.items():
        err = (view[k].double() - ref).abs()
        bad = int((err > 3e-2 + 2e-2 * ref.abs()).sum())
        assert bad == 0, f"{k}: {bad} of {err.numel()} elements out of tolerance, max err {err.max().item():.4g}"
    outs2, _, _, _ = _run(amn, bmn, epi, with_bias, M, N, K, cluster)
    for k in outs:
        assert torch.equal(outs[k], outs2[k]), f"{k}: two runs differ"


def test_mul2_needs_the_second_multiplier():
    from photon_b200 import ops

    a = torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV)
    b = torch.zeros(256, 64, dtype=torch.bfloat16, device=DEV)
    d, d2, aux = (torch.empty(128, 256, dtype=torch.bfloat16, device=DEV) for _ in range(3))
    with pytest.raises(RuntimeError, match="aux2"):
        ops.gemm(a, b, d, epi=EPI_MUL2, aux=aux, out2=d2)


@pytest.mark.parametrize("M", [1, 3, 16, 64])
@pytest.mark.parametrize("K,N", [(768, 2048), (2048, 5632), (776, 1000)])
def test_skinny_silu_and_mul(M, K, N):
    from photon_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(M * 7 + K + N)
    x = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    mul = torch.randn(M, N, device=DEV, generator=g).bfloat16()
    z = x.double() @ w.double().t() + bias.double()
    for name, kw, want in (("silu", dict(silu=True), _silu(z)), ("mul", dict(mul=mul), z * mul.double())):
        buf = torch.full((M + 2, N + 40), -3.0, dtype=torch.bfloat16, device=DEV)
        guard = buf.clone()
        out = buf[1:M + 1, 16:16 + N]
        ops.skinny_gemm(x, w, out, bias, **kw)
        again = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        ops.skinny_gemm(x, w, again, bias, **kw)
        torch.cuda.synchronize()
        inside = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
        inside[1:M + 1, 16:16 + N] = True
        assert torch.equal(buf[~inside], guard[~inside]), f"{name}: wrote outside its output"
        err = (out.double() - want).abs()
        assert int((err > 3e-2 + 2e-2 * want.abs()).sum()) == 0, f"{name}: max err {err.max().item():.4g}"
        assert torch.equal(out, again), f"{name}: two runs differ"


# ------------------------------------------------------------------------------------------------ engine vs fp32 model
FFNS = {"mlp_silu": dict(ffn_act="silu"), "glu_gelu": dict(ffn_type="mptglu"), "glu_silu": dict(ffn_type="mptglu", ffn_act="silu")}
VARIANTS = {"plain": {}, "no_bias": dict(no_bias=True), "f1408": dict(ffn_hidden_size=1408),
            "gqa_rope_qkln": dict(kv_n_heads=2, rope=True, learned_pos_emb=False, qk_ln=True),
            "doc_mask": dict(attn_uses_sequence_id=True, rope=True, learned_pos_emb=False)}
FFN_WEIGHTS = [f"transformer.blocks.0.ffn.{k}_proj.weight" for k in ("gate", "up", "down")]


def _cfg(ffn, **kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=512, n_heads=8, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch")
    return MPTConfig(**{**base, **FFNS[ffn], **kw})


def _pair(cfg, kernels=None, **eng_kw):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    ref = TorchBackend(cfg, DEV, "fp32", seed=3, **eng_kw)
    eng = B200Engine(cfg, DEV, "amp_bf16", dict(kernels or {"cuda_graph": False}), seed=3, **eng_kw)
    if not eng_kw:
        eng.flat.params.copy_(ref.flat.params)
        eng.params_updated()
    return ref, eng


def _ids(b, S, seed):
    return torch.randint(0, 2048, (b, S), device=DEV, generator=torch.Generator("cuda").manual_seed(seed))


def _match(ref, eng, ids, sid=None, tol=(5e-3, 0.995, 0.08, 0.08)):
    """As test_gqa_engine_gpu.py::_match, with the per-tensor check on block 0's FFN weight gradients."""
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, n_ref = ref.fwd_bwd(ids, denom, sequence_id=sid)
    l_eng, n_eng = eng.fwd_bwd(ids, denom, sequence_id=sid)
    torch.cuda.synchronize()
    assert int(n_ref) == int(n_eng)
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < tol[0], (float(l_ref), float(l_eng))
    g_ref, g_eng = ref.flat.grads, eng.flat.grads
    cos = torch.nn.functional.cosine_similarity(g_ref, g_eng, dim=0).item()
    rel = ((g_ref - g_eng).norm() / g_ref.norm()).item()
    assert cos > tol[1] and rel < tol[2], (cos, rel)
    lay = eng.flat.layout
    checked = 0
    for name in FFN_WEIGHTS:
        if name in lay.names:
            a, b = lay.view(g_ref, name), lay.view(g_eng, name)
            assert ((a - b).norm() / a.norm()).item() < tol[3], name
            checked += 1
    return checked


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("ffn", list(FFNS))
def test_ffn_engine_matches_torch(ffn, variant):
    cfg = _cfg(ffn, **VARIANTS[variant])
    ref, eng = _pair(cfg)
    assert eng.attn_mode == "b200"
    assert eng.layers[0].wup.shape == (cfg.ffn_hidden, 512) and (eng.layers[0].wgate is not None) == cfg.ffn_gated
    sid = None
    if cfg.attn_uses_sequence_id:
        from test_doc_engine_gpu import _batch

        ids, sid = _batch(4, 256, seed=1)
    else:
        ids = _ids(4, 256, 1)
    assert _match(ref, eng, ids, sid) == (3 if cfg.ffn_gated else 2)
    es = None if sid is None else sid[:2]
    a, b = ref.eval_stats(ids[:2], es), eng.eval_stats(ids[:2], es)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3


@pytest.mark.parametrize("ffn", ["glu_silu", "mlp_silu"])
def test_ffn_engine_activation_checkpointing_and_graphs(ffn):
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(ffn, n_layers=3, ffn_hidden_size=1408)
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


def test_ffn_engine_freeze_list_with_gate_tensors():
    """Frozen gate tensors are read from the frozen planes; the up stage still runs for the trainable up projection."""
    frozen = ["transformer.blocks.0.ffn.gate_proj.weight", "transformer.blocks.1.ffn.gate_proj.bias", "transformer.wte.weight"]
    ref, eng = _pair(_cfg("glu_silu"), frozen_layers=frozen)
    assert eng.flat.layout.names == ref.flat.layout.names and set(eng.frozen_layout.names) == set(frozen)
    assert eng.layers[0].d_wgate is None and eng.layers[0].d_bgate is not None and eng.layers[1].d_bgate is None
    assert _match(ref, eng, _ids(4, 256, 3)) == 2


def test_ffn_engine_only_gate_trainable():
    from photon_b200.models.mpt import MPTForCausalLM

    cfg = _cfg("glu_gelu")
    names = [n for n, _ in MPTForCausalLM(cfg, device="meta", init=False).named_parameters()]
    frozen = [n for n in names if ".blocks.1.ffn.gate_proj." not in n]
    ref, eng = _pair(cfg, frozen_layers=frozen)
    assert list(eng.flat.layout.names) == ["transformer.blocks.1.ffn.gate_proj.bias", "transformer.blocks.1.ffn.gate_proj.weight"]
    denom = float(4 * 255)
    ids = _ids(4, 256, 4)
    ref.flat.zero_grad(), eng.flat.zero_grad()
    ref.fwd_bwd(ids, denom)
    eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    rel = ((ref.flat.grads - eng.flat.grads).norm() / ref.flat.grads.norm()).item()
    assert rel < 0.08, rel


def test_ffn_engine_launch_count():
    """Per block, a gated FFN adds the gate GEMM to the forward and, to the backward, the gate's bias column sum and wgrad and
    the second input-gradient dgrad: four launches per block more than mptmlp. SiLU launches what GELU does."""
    from photon_b200.models.engine import B200Engine

    n = {}
    for ffn in ("mlp_silu", "glu_silu"):
        e = B200Engine(_cfg(ffn), DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
        e.fwd_bwd(_ids(2, 256, 0), 510.0)
        n[ffn] = e.launches_per_microbatch
    mlp = B200Engine(_cfg("mlp_silu", ffn_act="gelu"), DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
    mlp.fwd_bwd(_ids(2, 256, 0), 510.0)
    assert n["mlp_silu"] == mlp.launches_per_microbatch
    assert n["glu_silu"] == n["mlp_silu"] + 4 * 2


@pytest.mark.parametrize("ffn", list(FFNS))
def test_ffn_engine_refuses_fp8_and_full_sharding(ffn):
    from photon_b200.models.engine import B200Engine

    with pytest.raises(NotImplementedError, match="amp_fp8 or full parameter sharding"):
        B200Engine(_cfg(ffn), DEV, "amp_fp8", {"cuda_graph": False})
    with pytest.raises(NotImplementedError, match="amp_fp8 or full parameter sharding"):
        B200Engine(_cfg(ffn), DEV, "amp_bf16", {}, zero3=object())


def test_ffn_engine_rejects_unaligned_width_at_construction():
    from photon_b200.models.engine import B200Engine

    with pytest.raises(ValueError, match="multiple of 8"):
        B200Engine(_cfg("glu_silu", ffn_hidden_size=1412), DEV, "amp_bf16", {"cuda_graph": False})
    B200Engine(_cfg("glu_silu", ffn_hidden_size=1416), DEV, "amp_bf16", {"cuda_graph": False})


# ------------------------------------------------------------------------------------------------ decoding and scoring
def _prompts(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 2048, (n,), generator=g).tolist() for n in (3, 50, 129, 200)]


@pytest.mark.parametrize("ffn", ["glu_silu", "mlp_silu"])
def test_ffn_decoder_follows_the_model(ffn):
    ref, eng = _pair(_cfg(ffn, kv_n_heads=2, rope=True, learned_pos_emb=False), kernels={"cuda_graph": True})
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


def test_ffn_score_matches_the_model():
    from test_score_gpu import _fp32_stats, _pairs

    ref, eng = _pair(_cfg("glu_silu", rope=True, learned_pos_emb=False))
    pairs = _pairs(eng.cfg)
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (i, lp, want_lp)
        if clear:
            assert hit == want_hit, i
