"""The LM head on the sm_90a engine: the fused cross-entropy kernels with the logit transform (``logit_scale`` /
``final_logit_softcapping``) against float64, and the engine with tied / untied heads against the fp32 PyTorch model (bf16,
amp_fp8, a Llama-style combination under activation checkpointing and CUDA graphs, freeze lists, ZeRO-3), decoding and scoring,
and launch counts."""
import math

import pytest
import torch

from test_gqa_engine_gpu import LOGP_TOL, _ids, _match

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
LLAMA = dict(rope=True, learned_pos_emb=False, kv_n_heads=2, norm_type="rmsnorm", ffn_type="mptglu", ffn_act="silu", no_bias=True,
             tie_word_embeddings=False)


# ------------------------------------------------------------------------------------------------------------- kernels
def _ce_fp64(x, tgt, scale, cap, grad_scale):
    """(loss per valid row summed, #valid, #correct, row_lse, dlogits) in float64 from the bf16 logits ``x``."""
    xd = x.double()
    y = xd * (scale if scale is not None else 1.0)
    if cap is not None:
        y = cap * torch.tanh(y / cap)
    lse = torch.logsumexp(y, -1)
    valid = tgt >= 0
    t = tgt.clamp(min=0)
    loss = (lse - y.gather(1, t[:, None])[:, 0])[valid].sum()
    idx = torch.arange(xd.shape[1], device=xd.device).expand_as(xd)
    first = torch.where(xd == xd.max(-1, keepdim=True).values, idx, xd.shape[1]).min(-1).values   # lowest index among ties
    correct = (first == tgt)[valid].sum()
    p = torch.softmax(y, -1)
    p[torch.arange(len(t)), t] -= 1.0
    dy = (scale if scale is not None else 1.0) * (1 - (torch.tanh(xd * scale / cap) ** 2 if cap is not None else 0.0))
    g = p * dy * grad_scale * valid[:, None]
    return float(loss), int(valid.sum()), int(correct), lse, g


@pytest.mark.parametrize("V", [50368, 102408])   # the shared-memory kernel, and the two-read kernel above 200 KiB rows
@pytest.mark.parametrize("scale,cap", [(None, None), (0.3, None), (1.0, 30.0), (0.3, 30.0), (1 / math.sqrt(768), 5.0), (2.0, 5.0)])
def test_cross_entropy_with_the_head_transform_against_fp64(V, scale, cap):
    """Tolerances: loss sum 2e-5 relative (fp32 per-row math, fp64 atomics); row_lse 2e-5 absolute per unit of |lse|;
    dlogits are bf16, so 1/128 of the row's largest gradient plus one bf16 ulp; #correct exact."""
    from photon_b200 import ops

    rows = 96
    g = torch.Generator("cuda").manual_seed(V + int(1000 * (scale or 0)) + int(cap or 0))
    x = (torch.randn(rows, V, device=DEV, generator=g) * 8.0).to(torch.bfloat16)
    x[:4, :64] = 200.0   # saturated rows (ties of y under the cap, never of x)
    x[:4, 7] = 250.0
    tgt = torch.randint(0, V, (rows,), device=DEV, generator=g)
    tgt[::7] = -100                 # ignored rows
    tgt[1] = 7                      # a saturated row whose target is the argmax
    grad_scale = 1.0 / 300
    want = _ce_fp64(x, tgt, scale, cap, grad_scale)
    stats = torch.zeros(4, dtype=torch.float64, device=DEV)
    lse = torch.empty(rows, dtype=torch.float32, device=DEV)
    xw = x.clone()
    ops.cross_entropy(xw, tgt, grad_scale, True, stats, row_lse=lse, logit_scale=scale, softcap=cap)
    torch.cuda.synchronize()
    assert abs(float(stats[0]) - want[0]) <= 2e-5 * abs(want[0]), (float(stats[0]), want[0])
    assert int(stats[1]) == want[1] and int(stats[2]) == want[2]
    assert ((lse.double() - want[3]).abs() <= 2e-5 * want[3].abs().clamp(min=1)).all()
    gmax = want[4].abs().max(dim=1, keepdim=True).values
    err = (xw.double() - want[4]).abs()
    assert (err <= gmax / 128 + want[4].abs() / 128 + 1e-12).all(), float((err - gmax / 128).max())
    assert float(xw[::7].abs().max()) == 0.0
    # the same call without write_grad leaves the logits alone and gives the same statistics
    st2 = torch.zeros(4, dtype=torch.float64, device=DEV)
    xr = x.clone()
    ops.cross_entropy(xr, tgt, 0.0, False, st2, logit_scale=scale, softcap=cap)
    assert torch.equal(xr, x) and abs(float(st2[0]) - float(stats[0])) <= 1e-6 * abs(float(stats[0]))


def test_cross_entropy_default_transform_is_the_plain_kernel():
    from photon_b200 import ops

    x = (torch.randn(64, 50368, device=DEV) * 4).to(torch.bfloat16)
    tgt = torch.randint(0, 50368, (64,), device=DEV)
    outs = []
    for kw in ({}, dict(logit_scale=1.0), dict(logit_scale=None, softcap=None)):
        st, xw = torch.zeros(4, dtype=torch.float64, device=DEV), x.clone()
        ops.cross_entropy(xw, tgt, 0.01, True, st, **kw)
        outs.append((st.cpu(), xw))
    assert all(torch.equal(outs[0][1], o[1]) for o in outs[1:])


@pytest.mark.parametrize("kw", [dict(logit_scale=0.0), dict(logit_scale=-1.0), dict(logit_scale=float("inf")), dict(softcap=-5.0),
                                dict(softcap=float("nan"))])
def test_cross_entropy_rejects_bad_transforms(kw):
    from photon_b200 import ops

    x = torch.zeros(4, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="logit"):
        ops.cross_entropy(x, torch.zeros(4, dtype=torch.long, device=DEV), 1.0, True, torch.zeros(4, dtype=torch.float64, device=DEV), **kw)


# -------------------------------------------------------------------------------------------------------------- engine
def _cfg(**kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=512, n_heads=8, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch")
    return MPTConfig(**{**base, **kw})


def _pair(cfg, precision="amp_bf16", kernels=None, **eng_kw):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    ref = TorchBackend(cfg, DEV, "fp32", seed=3)
    eng = B200Engine(cfg, DEV, precision, dict(kernels or {"cuda_graph": False}), seed=5, **eng_kw)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return ref, eng


def _head_grad_close(ref, eng, tol=0.08):
    lay = eng.flat.layout
    for name in ("lm_head.weight", "transformer.wte.weight"):
        if name in lay.names:
            a, b = lay.view(ref.flat.grads, name), lay.view(eng.flat.grads, name)
            assert ((a - b).norm() / a.norm()).item() < tol, name


HEADS = {"tied": dict(), "untied": dict(tie_word_embeddings=False), "tied_scale": dict(logit_scale=0.3),
         "untied_cap": dict(tie_word_embeddings=False, final_logit_softcapping=5.0),
         "untied_scale_cap": dict(tie_word_embeddings=False, logit_scale="inv_sqrt_d_model", final_logit_softcapping=30.0),
         "tied_cap": dict(final_logit_softcapping=2.0), "llama": dict(LLAMA, logit_scale=0.5, final_logit_softcapping=30.0)}


@pytest.mark.parametrize("variant", list(HEADS))
def test_engine_head_matches_torch(variant):
    ref, eng = _pair(_cfg(**HEADS[variant]))
    if HEADS[variant].get("tie_word_embeddings") is False:
        assert eng.head16.data_ptr() != eng.wte16.data_ptr()
    _match(ref, eng, _ids(4, 256, 1))
    _head_grad_close(ref, eng)
    a, b = ref.eval_stats(_ids(2, 256, 2)), eng.eval_stats(_ids(2, 256, 2))
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3
    assert abs(float(a["n_correct"]) - float(b["n_correct"])) <= 0.02 * float(a["n_tokens"])


@pytest.mark.parametrize("variant", ["untied_cap", "llama"])   # with scale 1/sqrt(d) the head's gradient is too flat for fp8
def test_engine_head_amp_fp8(variant):
    cfg = _cfg(**HEADS[variant])
    if cfg.ffn_type != "mptmlp":
        cfg = _cfg(**{**HEADS[variant], "ffn_type": "mptmlp", "ffn_act": "gelu"})   # amp_fp8 covers the mptmlp block
    ref, eng = _pair(cfg, precision="amp_fp8")
    _, bf = _pair(cfg)
    ids, denom = _ids(4, 256, 1), float(4 * 255)
    for e in (eng, bf):
        e.flat.zero_grad()
    l8, lb = float(eng.fwd_bwd(ids, denom)[0]), float(bf.fwd_bwd(ids, denom)[0])
    torch.cuda.synchronize()
    assert abs(l8 - lb) / lb < 2e-2, (l8, lb)
    cos = torch.nn.functional.cosine_similarity(eng.flat.grads, bf.flat.grads, dim=0).item()
    assert cos > 0.97, cos
    _match(ref, eng, ids, tol=(2e-2, 0.97, 0.25, 0.35))


def test_llama_head_under_checkpointing_and_graphs():
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(n_layers=3, **HEADS["llama"])
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
    for e in (ckpt, graph):
        rel = ((eager.flat.grads - e.flat.grads).norm() / eager.flat.grads.norm()).item()
        assert rel < 1e-3, rel


FREEZE = {"lm_head_frozen": dict(frozen_layers=["lm_head.weight"]), "only_lm_head": dict(unfrozen_layers=["lm_head.weight"]),
          "only_wte": dict(unfrozen_layers=["transformer.wte.weight"])}


@pytest.mark.parametrize("case", list(FREEZE))
def test_engine_freeze_lists_with_an_untied_head(case):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    cfg = _cfg(tie_word_embeddings=False, final_logit_softcapping=30.0)
    ref = TorchBackend(cfg, DEV, "fp32", seed=5)
    eng = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5, **FREEZE[case])
    ids, denom = _ids(4, 256, 1), float(4 * 255)
    ref.flat.zero_grad(), eng.flat.zero_grad()
    la, lb = float(ref.fwd_bwd(ids, denom)[0]), float(eng.fwd_bwd(ids, denom)[0])
    torch.cuda.synchronize()
    assert abs(la - lb) / la < 5e-3, (la, lb)
    rl, el = ref.flat.layout, eng.flat.layout
    assert ("lm_head.weight" in el.names) == (case == "only_lm_head")
    for name in el.names:
        a, b = rl.view(ref.flat.grads, name), el.view(eng.flat.grads, name)
        assert ((a - b).norm() / a.norm()).item() < 0.08, name
    if case == "lm_head_frozen":
        assert eng.frozen_layout is not None and "lm_head.weight" in eng.frozen_layout.names and not eng.plan.head_wgrad


@pytest.mark.parametrize("precision", ["amp_bf16", "amp_fp8"])
def test_engine_full_sharding_with_an_untied_head_equals_unsharded(precision):
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import NvlZero3Comm

    cfg = _cfg(n_layers=3, tie_word_embeddings=False, logit_scale=0.5, final_logit_softcapping=30.0)
    plain = B200Engine(cfg, DEV, precision, {"cuda_graph": False}, seed=5)
    comm = NvlZero3Comm(plain.flat.layout, cfg.n_layers, rank=0, world_size=1, device=DEV, fp8=precision == "amp_fp8")
    assert comm.plan.head is not None
    shard = B200Engine(cfg, DEV, precision, {}, seed=5, zero3=comm)
    assert torch.equal(shard.flat.full_params(), plain.flat.params)
    denom = float(4 * 255)
    plain.flat.zero_grad(), shard.flat.zero_grad()
    for s in range(2):
        ids = _ids(4, 256, s)
        la, _ = plain.fwd_bwd(ids, denom)
        lb, _ = shard.fwd_bwd(ids, denom)
        torch.cuda.synchronize()
        assert abs(float(la) - float(lb)) <= 1e-4 * abs(float(la)), (precision, float(la), float(lb))
    full = torch.zeros_like(plain.flat.grads)
    comm.plan.shard_to_full(shard.flat.grads, 0, full)
    rel = ((full - plain.flat.grads).norm() / plain.flat.grads.norm()).item()
    assert rel < 2e-3, (precision, rel)
    lay = plain.flat.layout
    a, b = lay.view(plain.flat.grads, "lm_head.weight"), lay.view(full, "lm_head.weight")
    assert a.norm() > 0 and ((a - b).norm() / a.norm()).item() < 1e-5
    comm.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_fully_sharded_untied_head_match_ddp(tmp_path):
    """torchrun, 2 GPUs: an untied, soft-capped head under kernels.param_sharding=zero3 ends on the parameters of plain DDP."""
    from test_multiproc_gpu import _torchrun

    _torchrun(tmp_path, 2, """
        from photon_b200.config import compose
        from photon_b200.centralised_train import run_centralised
        rank = dist.get_rank(); dev = torch.device('cuda', rank)
        outs = {}
        head = ['++llm_config.model.tie_word_embeddings=false', '++llm_config.model.final_logit_softcapping=30.0']
        for name, extra in (('zero3', ['kernels.param_sharding=zero3']), ('ddp', ['~llm_config.fsdp_config'])):
            cfg = compose(TINY + ['run_uuid=z3h', 'dataset/streams@dataset.train.streams=centralised', 'dataset.train.root_local=synthetic://7',
                                  'llm_config.model.n_layers=3'] + head + extra)
            tr = run_centralised(cfg, device=dev, rank=rank, world_size=dist.get_world_size(), duration='3ba')
            if name == 'zero3':
                assert tr.grad_comm.plan.head is not None
            outs[name] = tr.state.flat.full_params().clone()
            tr.close()
        rel = ((outs['zero3'] - outs['ddp']).norm() / outs['ddp'].norm()).item()
        assert rel < 2e-3, rel
        if rank == 0: print('RESULT_OK', rel)
    """, 29561)


def test_launch_count_untied_equals_tied():
    from photon_b200 import ops
    from photon_b200.models.engine import B200Engine

    counts = []
    for kw in (dict(), dict(tie_word_embeddings=False), dict(tie_word_embeddings=False, logit_scale=0.5, final_logit_softcapping=30.0)):
        e = B200Engine(_cfg(**kw), DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
        e.fwd_bwd(_ids(2, 256, 20), 510.0)
        torch.cuda.synchronize()
        ops.reset_launch_count()
        e.fwd_bwd(_ids(2, 256, 21), 510.0)
        torch.cuda.synchronize()
        counts.append(ops.launch_count())
    assert counts[0] == counts[1] == counts[2], counts


# ------------------------------------------------------------------------------------------------ decoding and scoring
@pytest.mark.parametrize("variant", ["untied_scale_cap", "tied_cap", "llama"])
def test_decoder_follows_the_model(variant):
    from test_window_engine_gpu import _follow

    ref, eng = _pair(_cfg(**HEADS[variant]), kernels={"cuda_graph": True})
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, 2048, (n,), generator=g).tolist() for n in (3, 40, 130)]
    dec = eng.decoder(len(prompts))

    class Raw:   # the decoder's logits are the raw head logits: compare against the module's before its transform
        def logits(self, ids):
            m = ref.model
            with torch.no_grad():
                h = m.hidden_states(ids)
                w = m.transformer.wte.weight if m.cfg.tie_word_embeddings else m.lm_head.weight
                return torch.nn.functional.linear(h, w)

    _follow(Raw(), dec, prompts, 12)


@pytest.mark.parametrize("variant", ["untied_scale_cap", "tied_cap", "llama"])
def test_score_matches_the_model(variant):
    from test_score_gpu import _fp32_stats, _pairs

    ref, eng = _pair(_cfg(**HEADS[variant]))
    pairs = _pairs(eng.cfg)
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (i, lp, want_lp)
        if clear:
            assert hit == want_hit, i
