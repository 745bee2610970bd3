"""B200Engine (explicit fwd/bwd on our kernels) vs the stock-PyTorch backend on the same parameters."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(attn):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    dev = torch.device("cuda", 0)
    ref = TorchBackend(cfg, dev, "fp32", seed=3)
    eng = B200Engine(cfg, dev, "amp_bf16", {"attention": attn}, seed=5)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return cfg, ref, eng


@pytest.mark.parametrize("attn", ["torch", "b200"])
def test_engine_loss_and_grads_match_torch(attn):
    cfg, ref, eng = _mk(attn)
    ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device="cuda:0")
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, n_ref = ref.fwd_bwd(ids, denom)
    l_eng, n_eng = eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert int(n_ref) == int(n_eng)
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < 5e-3, (float(l_ref), float(l_eng))
    g_ref, g_eng = ref.flat.grads, eng.flat.grads
    cos = torch.nn.functional.cosine_similarity(g_ref, g_eng, dim=0).item()
    rel = ((g_ref - g_eng).norm() / g_ref.norm()).item()
    assert cos > 0.995 and rel < 0.08, (cos, rel)
    # per-tensor check catches a single wrong gradient hiding in the global norm
    lay = eng.flat.layout
    for i, n in enumerate(lay.names):
        a, b = lay.view(g_ref, i).flatten(), lay.view(g_eng, i).flatten()
        if a.norm() > 1e-6:
            c = torch.nn.functional.cosine_similarity(a, b, dim=0).item()
            assert c > 0.98, (n, c)
    assert eng.launches_per_microbatch > 0


def test_engine_eval_stats_match():
    cfg, ref, eng = _mk("torch")
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device="cuda:0")
    a, b = ref.eval_stats(ids), eng.eval_stats(ids)
    assert float(a["n_tokens"]) == float(b["n_tokens"])
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3


def test_trainer_on_engine_trains():
    from photon_b200.data.synthetic import synthetic_batch
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.trainer import Trainer

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048)

    class Loader:
        def __iter__(self):
            i = 0
            while True:
                ids = torch.from_numpy(synthetic_batch(8, 256, seed=1, start=0) % 2048)  # same batch -> must overfit
                yield {"input_ids": ids.pin_memory(), "labels": ids}
                i += 1

    tr = Trainer(cfg, optimizer_cfg=dict(name="adopt", lr=3e-3, betas=[0.9, 0.9999], eps=1e-6, weight_decay=0.0),
                 scheduler_cfg=dict(name="constant_with_warmup", t_warmup="2ba"), train_loader=Loader(), global_train_batch_size=8,
                 device_train_microbatch_size=4, precision="amp_bf16", max_duration="30ba", grad_clip_norm=1.0,
                 device="cuda:0", kernels={"attention": "torch"})
    assert tr.state.backend.kind == "b200"
    tr.fit("3ba")
    first = tr.loggers[0].data["loss/train/total"][0][1]
    tr.fit("25ba")
    last = tr.loggers[0].data["loss/train/total"][-1][1]
    assert last < first - 1.0, (first, last)


def test_engine_activation_checkpointing_is_exact():
    """Recomputing block internals from h[i] gives bit-identical gradients with 1/L of the block activations."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=3, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    dev = torch.device("cuda", 0)
    a = B200Engine(cfg, dev, "amp_bf16", {}, seed=5)
    b = B200Engine(cfg, dev, "amp_bf16", {}, seed=5, activation_checkpointing=True)
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device=dev)
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    a.flat.zero_grad(), b.flat.zero_grad()
    la, _ = a.fwd_bwd(ids, denom)
    lb, _ = b.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert float(la) == float(lb)
    ws = b._workspace(2, cfg.max_seq_len)
    assert ws["layers"][0] is ws["layers"][2]
    rel = ((a.flat.grads - b.flat.grads).norm() / a.flat.grads.norm()).item()
    assert rel < 1e-3, rel   # split-K reduce-add order is the only non-determinism
    assert b.launches_per_microbatch > a.launches_per_microbatch


def test_engine_cuda_graph_replay_matches_eager():
    """kernels.cuda_graph: the captured microbatch schedule accumulates the same gradients as eager launches, for
    fresh token ids on every replay."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    dev = torch.device("cuda", 0)
    a = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": False}, seed=5)
    b = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": True}, seed=5)
    assert not a.use_graph and b.use_graph
    a.flat.zero_grad(), b.flat.zero_grad()
    denom = float(2 * (cfg.max_seq_len - 1))
    for i in range(3):   # first call captures, the next two replay with different inputs
        ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device=dev)
        la, na = a.fwd_bwd(ids, denom)
        lb, nb = b.fwd_bwd(ids, denom)
        torch.cuda.synchronize()
        assert int(na) == int(nb) and abs(float(la) - float(lb)) <= 1e-3 * abs(float(la)), (i, float(la), float(lb))
    assert len(b._graphs) == 1
    rel = ((a.flat.grads - b.flat.grads).norm() / a.flat.grads.norm()).item()
    assert rel < 1e-3, rel
    assert b.launches_per_microbatch == a.launches_per_microbatch > 0


def test_engine_graph_replay_after_a_larger_attention_backward():
    """A captured graph keeps its own dQ accumulator: an attention backward at a larger shape elsewhere in the process,
    between capture and replay, must not move or free the memory the graph's nodes point at."""
    from photon_b200 import ops
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    dev = torch.device("cuda", 0)
    a = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": False}, seed=5)
    b = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": True}, seed=5)
    a.flat.zero_grad(), b.flat.zero_grad()
    denom = float(cfg.max_seq_len - 1)
    ids = torch.randint(0, cfg.vocab_size, (1, cfg.max_seq_len), device=dev)
    a.fwd_bwd(ids, denom)
    b.fwd_bwd(ids, denom)   # captures the b = 1 graph
    assert len(b._graphs) == 1
    # a larger attention backward: [8 x 2048] rows x 2048 columns of fp32 accumulator, 64x the engine's
    B, S, H, dh = 8, 2048, 16, 128
    qkv = torch.randn(B, S, 3 * H * dh, device=dev).bfloat16()
    out = torch.empty(B, S, H * dh, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(B, H, S, device=dev)
    ops.attention_fwd(qkv, out, lse, H, dh ** -0.5, True)
    ops.attention_bwd(qkv, out, torch.randn_like(out), lse, torch.empty_like(qkv), torch.empty_like(lse), H, dh ** -0.5, True)
    torch.cuda.synchronize()
    del qkv, out, lse
    for _ in range(2):   # replays of the b = 1 graph after it
        ids = torch.randint(0, cfg.vocab_size, (1, cfg.max_seq_len), device=dev)
        la, _ = a.fwd_bwd(ids, denom)
        lb, _ = b.fwd_bwd(ids, denom)
        torch.cuda.synchronize()
        assert abs(float(la) - float(lb)) <= 1e-3 * abs(float(la)), (float(la), float(lb))
    assert len(b._graphs) == 1
    assert bool(torch.isfinite(b.flat.grads).all())
    rel = ((a.flat.grads - b.flat.grads).norm() / a.flat.grads.norm()).item()
    assert rel < 1e-3, rel


def test_engine_d_head_128_runs_on_own_attention():
    """MPT-1B/3B/7B geometry (d_head = 128): forward and backward attention stay on the wgmma kernels."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    cfg = MPTConfig(d_model=256, n_heads=2, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    assert cfg.d_head == 128
    dev = torch.device("cuda", 0)
    ref = TorchBackend(cfg, dev, "fp32", seed=3)
    eng = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": False}, seed=5)
    assert eng.attn_mode == "b200"
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device=dev)
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, _ = ref.fwd_bwd(ids, denom)
    l_eng, _ = eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < 5e-3
    cos = torch.nn.functional.cosine_similarity(ref.flat.grads, eng.flat.grads, dim=0).item()
    rel = ((ref.flat.grads - eng.flat.grads).norm() / ref.flat.grads.norm()).item()
    assert cos > 0.995 and rel < 0.08, (cos, rel)


@pytest.mark.parametrize("variant", ["alibi", "rope", "no_bias", "clip_qkv", "qk_ln"])
def test_engine_positional_variants_match_torch(variant):
    """ALiBi / RoPE (no learned positions), no_bias, clip_qkv and qk_ln run on the engine's own kernels and match the PyTorch model."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    extra = {"alibi": dict(alibi=True, learned_pos_emb=False), "rope": dict(rope=True, learned_pos_emb=False),
             "no_bias": dict(no_bias=True), "clip_qkv": dict(clip_qkv=0.5), "qk_ln": dict(qk_ln=True)}[variant]
    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch", **extra)
    dev = torch.device("cuda", 0)
    ref = TorchBackend(cfg, dev, "fp32", seed=3)
    eng = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": False}, seed=5)
    assert eng.attn_mode == "b200" and (eng.alibi is not None) == (variant == "alibi") and (eng.rope is not None) == (variant == "rope")
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device=dev)
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, _ = ref.fwd_bwd(ids, denom)
    l_eng, _ = eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < 5e-3, (float(l_ref), float(l_eng))
    cos = torch.nn.functional.cosine_similarity(ref.flat.grads, eng.flat.grads, dim=0).item()
    rel = ((ref.flat.grads - eng.flat.grads).norm() / ref.flat.grads.norm()).item()
    assert cos > 0.995 and rel < 0.08, (cos, rel)


def test_engine_sequence_length_not_multiple_of_128_uses_library_attention():
    """The wgmma attention kernels need S % 128 == 0; any other length runs attention through SDPA inside the same engine
    step (everything else stays on our kernels) and still matches the PyTorch model."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=200, vocab_size=2048, attn_impl="torch")
    dev = torch.device("cuda", 0)
    ref = TorchBackend(cfg, dev, "fp32", seed=3)
    eng = B200Engine(cfg, dev, "amp_bf16", {}, seed=5)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    ids = torch.randint(0, cfg.vocab_size, (4, 200), device=dev)
    denom = float(4 * 199)
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, _ = ref.fwd_bwd(ids, denom)
    l_eng, _ = eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < 5e-3
    rel = ((ref.flat.grads - eng.flat.grads).norm() / ref.flat.grads.norm()).item()
    assert rel < 0.08, rel
