"""Partly frozen models on the sm_90a engine (``fl.frozen_layers`` / ``fl.unfrozen_layers``): gradients against the fp32 torch
backend and the unfrozen engine, frozen storage, skipped backward work, graph replay, fp8 weight copies, the optional token
embedding gradient of ``embed_bwd``, decoding and a one-GPU federation."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
L = 4


def _cfg(**kw):
    from photon_b200.models.mpt import MPTConfig

    return MPTConfig(d_model=256, n_heads=4, n_layers=L, max_seq_len=256, vocab_size=2048, attn_impl="flash", **kw)


def _names(cfg):
    from photon_b200.models.mpt import MPTForCausalLM

    return [n for n, _ in MPTForCausalLM(cfg, device="meta", init=False).named_parameters()]


def _freeze(kind, cfg):
    """The freeze lists under test, as Trainer / backend keyword arguments."""
    names = _names(cfg)
    emb = [n for n in ("transformer.wte.weight", "transformer.wpe.weight") if n in names]
    return {
        "wte": dict(frozen_layers=["transformer.wte.weight"]),
        "wpe": dict(frozen_layers=["transformer.wpe.weight"]),
        "lower": dict(frozen_layers=emb + [n for n in names if any(f".blocks.{i}." in n for i in range(L // 2))]),
        "ffn1": dict(unfrozen_layers=[n for n in names if ".blocks.1.ffn." in n]),
        "norms_biases": dict(frozen_layers=[n for n in names if ".norm_" in n or ".norm_f." in n or n.endswith(".bias")]),
        "only_wte": dict(unfrozen_layers=["transformer.wte.weight"]),
    }[kind]


def _engine(cfg, precision="amp_bf16", ckpt=False, graph=True, **freeze):
    from photon_b200.models.engine import B200Engine

    return B200Engine(cfg, DEV, precision, {"cuda_graph": graph}, seed=5, activation_checkpointing=ckpt, **freeze)


def _ids(cfg, b=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg.vocab_size, (b, cfg.max_seq_len), generator=g).to(DEV)


def _cos(a, b):
    a, b = a.flatten().double(), b.flatten().double()
    return float((a @ b) / (a.norm() * b.norm()))


GRAD_CASES = [(k, p, c) for k in ("wte", "wpe", "lower", "ffn1", "norms_biases", "only_wte")
              for p, c in (("amp_bf16", False), ("amp_bf16", True), ("amp_fp8", False))]
VARIANTS = {"alibi": dict(alibi=True, learned_pos_emb=False), "rope_qkln_clip": dict(rope=True, learned_pos_emb=False, qk_ln=True, clip_qkv=6.0),
            "no_bias": dict(no_bias=True)}
GRAD_CASES += [(k, "amp_bf16", False, v) for v in VARIANTS for k in ("lower", "ffn1")]


@pytest.mark.parametrize("case", GRAD_CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_frozen_gradients_match_torch_and_unfrozen_engine(case):
    from photon_b200.train.backend import TorchBackend

    kind, precision, ckpt = case[:3]
    cfg = _cfg(**VARIANTS[case[3]]) if len(case) > 3 else _cfg()
    freeze = _freeze(kind, cfg)
    ref = TorchBackend(cfg, DEV, "fp32", seed=5, **freeze)
    full = _engine(cfg, precision, ckpt)
    eng = _engine(cfg, precision, ckpt, **freeze)
    assert eng.flat.layout.names == ref.flat.layout.names
    assert not set(eng.flat.layout.names) & set(eng.frozen_layout.names)
    ids = _ids(cfg)
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    for be in (ref, full, eng):
        be.flat.zero_grad()
    l_ref, _ = ref.fwd_bwd(ids, denom)
    l_full, _ = full.fwd_bwd(ids, denom)
    l_eng, _ = eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert float(l_eng) == float(l_full)                       # the forward is untouched by freezing
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < (2e-2 if precision == "amp_fp8" else 5e-3)
    lay, flay = eng.flat.layout, full.flat.layout
    g_ref, g_eng = ref.flat.grads, eng.flat.grads
    if precision == "amp_fp8":   # the fp8 recipe's own tolerance against higher precision (tests/test_fp8_gpu.py)
        for i, n in enumerate(lay.names):
            if lay.numels[i] >= 256 * 256:
                assert _cos(lay.view(g_ref, i), lay.view(g_eng, i)) > 0.95, n
    else:
        assert _cos(g_ref, g_eng) > 0.995 and float((g_ref - g_eng).norm() / g_ref.norm()) < 0.08
        for i, n in enumerate(lay.names):
            a = lay.view(g_ref, i)
            if a.norm() > 1e-6:
                assert _cos(a, lay.view(g_eng, i)) > 0.98, n
    # against the unfrozen engine, sliced to the trainable names: the same kernels on the same values, up to the float
    # atomics of attention dQ / embedding / split-K wgrad (and, in fp8, an occasional E5M2 rounding they flip)
    a = torch.cat([flay.view(full.flat.grads, n).flatten() for n in lay.names])
    b = torch.cat([lay.view(g_eng, n).flatten() for n in lay.names])
    rel = float((a - b).norm() / a.norm())
    assert rel < (3e-2 if precision == "amp_fp8" else 5e-3), rel
    for n in lay.names:
        x = flay.view(full.flat.grads, n)
        if x.norm() > 1e-6:
            assert _cos(x, lay.view(g_eng, n)) > (0.995 if precision == "amp_fp8" else 0.9999), n


def test_trainer_keeps_frozen_values_and_tracks_torch():
    from photon_b200.data.synthetic import synthetic_batch
    from photon_b200.train.trainer import Trainer

    cfg = _cfg()
    freeze = _freeze("lower", cfg)

    class Loader:
        def __iter__(self):
            k = 0
            while True:
                ids = torch.from_numpy(synthetic_batch(8, cfg.max_seq_len, seed=1, start=8 * k) % cfg.vocab_size)
                yield {"input_ids": ids.pin_memory(), "labels": ids}
                k += 1

    def make(kernels):
        return Trainer(cfg, optimizer_cfg=dict(name="adopt", lr=1e-3, betas=[0.9, 0.9999], eps=1e-6, weight_decay=0.0),
                       scheduler_cfg=dict(name="constant_with_warmup", t_warmup="1ba"), train_loader=Loader(), global_train_batch_size=8,
                       device_train_microbatch_size=4, precision="amp_bf16", max_duration="10ba", grad_clip_norm=1.0, device=DEV,
                       kernels=kernels, seed=5, **freeze)

    et = make({})
    tt = make({k: "torch" for k in ("gemm", "attention", "norm", "loss", "optimizer")})
    e, t = et.state.backend, tt.state.backend
    assert e.kind == "b200" and t.kind == "torch"
    assert set(e.frozen_layout.names) == set(freeze["frozen_layers"]) and not set(e.flat.layout.names) & set(freeze["frozen_layers"])
    mod = dict(e.model.named_parameters())
    for n in e.frozen_layout.names:
        assert mod[n].data_ptr() == e.frozen_layout.view(e.frozen_params, n).data_ptr()   # the module reads the frozen plane
    p32, p16 = e.frozen_params.clone(), e.frozen_bf16.clone()
    et.fit("5ba")
    tt.fit("5ba")
    torch.cuda.synchronize()
    assert torch.equal(e.frozen_params, p32) and torch.equal(e.frozen_bf16, p16)
    tm = dict(t.model.named_parameters())
    for n in e.frozen_layout.names:
        assert torch.equal(e.frozen_layout.view(e.frozen_params, n), tm[n].detach()), n
    le = [v for _, v in et.loggers[0].data["loss/train/total"]]
    lt = [v for _, v in tt.loggers[0].data["loss/train/total"]]
    assert len(le) == len(lt) == 5
    for a, b in zip(le, lt):
        assert abs(a - b) / abs(b) < 2e-2, (le, lt)
    assert le[-1] < le[0]


def test_frozen_lower_half_skips_backward_launches():
    from photon_b200 import ops

    cfg = _cfg()
    full = _engine(cfg, graph=False)
    eng = _engine(cfg, graph=False, **_freeze("lower", cfg))
    ids = _ids(cfg, b=2)
    b, S = ids.shape
    denom = float(b * (S - 1))
    full.fwd_bwd(ids, denom)
    eng.fwd_bwd(ids, denom)
    # the backward launches of the skipped blocks and of the embedding gradient, counted on the unfrozen engine
    ws = full._workspace(b, S)
    n0 = ops.launch_count()
    for i in range(L // 2):
        full._block_bwd(i, ws, b, S)
    ops.embed_bwd(ids.reshape(-1), ws["dh"], full.d_wte, full.d_wpe, S)
    skipped = ops.launch_count() - n0
    torch.cuda.synchronize()
    assert skipped > 0
    assert eng.launches_per_microbatch <= full.launches_per_microbatch - skipped, (eng.launches_per_microbatch, full.launches_per_microbatch, skipped)


def test_frozen_graph_replay_matches_eager():
    cfg = _cfg()
    freeze = _freeze("lower", cfg)
    a = _engine(cfg, graph=False, **freeze)
    g = _engine(cfg, graph=True, **freeze)
    assert g.use_graph and not a.use_graph
    denom = float(2 * (cfg.max_seq_len - 1))
    a.flat.zero_grad(), g.flat.zero_grad()
    for k in range(3):   # capture, then two replays with fresh token ids
        ids = _ids(cfg, b=2, seed=10 + k)
        la, _ = a.fwd_bwd(ids, denom)
        lg, _ = g.fwd_bwd(ids, denom)
        torch.cuda.synchronize()
        assert float(la) == float(lg)
    rel = float((a.flat.grads - g.flat.grads).norm() / a.flat.grads.norm())
    assert rel < 1e-3, rel
    assert g.launches_per_microbatch == a.launches_per_microbatch


def test_fp8_frozen_graph_replay_matches_unfrozen_graph():
    """amp_fp8: capturing runs one eager warm-up microbatch, which advances the delayed-scaling history, so a graphed engine's
    scales run one microbatch ahead of an eager one whatever is frozen. Against an unfrozen graphed engine the replays of the
    shortened schedule give the same losses, bitwise, and the same trainable gradients."""
    cfg = _cfg()
    freeze = _freeze("lower", cfg)
    full = _engine(cfg, "amp_fp8", graph=True)
    g = _engine(cfg, "amp_fp8", graph=True, **freeze)
    denom = float(2 * (cfg.max_seq_len - 1))
    full.flat.zero_grad(), g.flat.zero_grad()
    for k in range(3):
        ids = _ids(cfg, b=2, seed=10 + k)
        lf, _ = full.fwd_bwd(ids, denom)
        lg, _ = g.fwd_bwd(ids, denom)
        torch.cuda.synchronize()
        assert float(lf) == float(lg)
    lay, flay = g.flat.layout, full.flat.layout
    a = torch.cat([flay.view(full.flat.grads, n).flatten() for n in lay.names])
    b = torch.cat([lay.view(g.flat.grads, n).flatten() for n in lay.names])
    assert float((a - b).norm() / a.norm()) < 3e-2
    assert g.launches_per_microbatch < full.launches_per_microbatch


def test_fp8_frozen_weights_are_quantised_once_and_match_per_microbatch_quantisation():
    from photon_b200 import ops

    cfg = _cfg()
    freeze = _freeze("lower", cfg)
    full = _engine(cfg, "amp_fp8")
    eng = _engine(cfg, "amp_fp8", **freeze)
    frozen_w = [(i, k) for i in range(L) for k in eng._W_ROLES if eng.w8t_views[i].get(k) is not None]
    assert len(frozen_w) == 4 * (L // 2) and eng._n_w8 == 4 * (L - L // 2)
    roles = [eng._role(k, i) for i, k in frozen_w]
    # a fresh quantisation of the frozen bf16 plane gives the same bytes and scales
    w8, meta = torch.zeros_like(eng.w8f), eng.fp8_meta.clone()
    ops.fp8_quantize_segments(eng.frozen_bf16, w8, eng.w8f_seg, meta, eng._n_dyn + eng._n_w8)
    torch.cuda.synchronize()
    assert torch.equal(w8, eng.w8f) and torch.equal(meta[:2, roles], eng.fp8_meta[:2, roles])
    before, meta0 = eng.w8f.clone(), eng.fp8_meta[:2, roles].clone()
    ids = _ids(cfg, b=2)
    for k in range(3):
        full.fwd_bwd(ids, 510.0)
        eng.fwd_bwd(ids, 510.0)
    torch.cuda.synchronize()
    # no per-microbatch quantisation touches them ...
    assert torch.equal(eng.w8f, before) and torch.equal(eng.fp8_meta[:2, roles], meta0)
    # ... and they equal the unfrozen engine's per-microbatch quantisation of the same tensors, bitwise; the K-major copy the
    # dgrad GEMMs read is their exact transpose
    for i, k in frozen_w:
        assert torch.equal(eng.w8_views[i][k], full.w8_views[i][k]), (i, k)
        assert torch.equal(eng.fp8_meta[:2, eng._role(k, i)], full.fp8_meta[:2, full._role(k, i)]), (i, k)
        assert torch.equal(eng.w8t_views[i][k], eng.w8_views[i][k].t().contiguous()), (i, k)
    # a loaded fp8 state keeps the frozen bytes paired with their scales
    eng.load_fp8_state_dict(full.fp8_state_dict())
    torch.cuda.synchronize()
    assert torch.equal(eng.w8f, before) and torch.equal(eng.fp8_meta[:2, roles], meta0)


def test_embed_bwd_without_token_embedding_gradient():
    from photon_b200 import ops

    B, S, d, V = 3, 64, 768, 1000
    ids = torch.randint(0, V, (B * S,), device=DEV)
    dh = torch.randn(B * S, d, device=DEV).to(torch.bfloat16)
    dwpe = torch.zeros(S, d, device=DEV)
    n0 = ops.launch_count()
    ops.embed_bwd(ids, dh, None, dwpe, S)
    assert ops.launch_count() - n0 == 1        # the token-embedding scatter is not launched
    torch.cuda.synchronize()
    torch.testing.assert_close(dwpe, dh.float().view(B, S, d).sum(0), rtol=1e-3, atol=1e-3)
    dwte = torch.zeros(V, d, device=DEV)
    n0 = ops.launch_count()
    ops.embed_bwd(ids, dh, dwte, None, S)
    assert ops.launch_count() - n0 == 1
    torch.cuda.synchronize()
    torch.testing.assert_close(dwte, torch.zeros(V, d, device=DEV).index_add_(0, ids, dh.float()), rtol=1e-3, atol=1e-3)


def test_decoding_and_scoring_on_a_frozen_engine_match_the_unfrozen_engine():
    cfg = _cfg()
    full = _engine(cfg)
    eng = _engine(cfg, **_freeze("lower", cfg))     # same seed: the same values, held in the frozen planes
    g = torch.Generator().manual_seed(3)
    rnd = lambda n: torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist()  # noqa: E731
    prompts = [rnd(n) for n in (5, 64, 130)]
    pairs = [(rnd(20), rnd(n)) for n in (1, 4, 17)] + [(rnd(129), rnd(3))]

    def run(e):
        dec = e.decoder(len(pairs))
        toks = [dec.start(prompts, 6)] + [dec.step() for _ in range(5)]
        return toks, e.decoder(len(pairs)).score(pairs)

    assert run(eng) == run(full)


def test_one_gpu_nvl_federation_with_frozen_layers_runs_on_the_engine():
    from photon_b200.config import compose
    from photon_b200.federation import FederationRuntime
    from photon_b200.models.mpt import MPTForCausalLM
    from photon_b200.server_app import run_server

    frozen = ["transformer.wte.weight", "transformer.blocks.0.attn.Wqkv.weight"]
    tiny = ["llm_config.model.d_model=256", "llm_config.model.n_heads=4", "llm_config.model.n_layers=2", "llm_config.max_seq_len=256",
            "llm_config.model.vocab_size=50368", "llm_config.global_train_batch_size=8", "llm_config.device_train_microbatch_size=4",
            "llm_config.local_steps=2ba", "llm_config.log_to_console=false", "~llm_config.loggers.wandb", "~llm_config.loggers.tensorboard",
            "~llm_config.callbacks", "llm_config.save_folder=null", "llm_config.optimizer.lr=1.0e-3",
            "llm_config.scheduler.schedulers.lr.t_warmup=1ba", "fl.eval_period=null", "photon.resume_round=null", "fl.n_total_clients=4",
            "fl.n_clients_per_round=3", "fl.n_rounds=2", "dataset.train.root_local=synthetic://c", "run_uuid=g-frozen",
            "photon.comm_stack.shm=false", "photon.comm_stack.nvl=true", f"fl.frozen_layers=[{','.join(frozen)}]"]
    cfg = compose(tiny)
    rt = FederationRuntime(cfg, device=DEV, rank=0, world_size=1)
    h = run_server(cfg, runtime=rt)
    try:
        fit = h.metrics_distributed_fit
        assert [v for _, v in fit["server/n_failures"]] == [0, 0]
        e = rt.trainer.state.backend
        assert e.kind == "b200"
        assert not set(frozen) & set(rt.model_layout.names) and set(e.frozen_layout.names) == set(frozen)
        x = rt.round_backend.global_params()
        assert x.numel() == rt.model_layout.total and torch.isfinite(x).all()
        # every client trains on the same frozen values: the initial ones, never exchanged, never changed
        init = dict(MPTForCausalLM(rt.trainer.model_cfg, device=DEV, seed=rt.trainer.seed).named_parameters())
        for n in frozen:
            assert torch.equal(e.frozen_layout.view(e.frozen_params, n), init[n].detach()), n
    finally:
        rt.close()
