"""B200Engine with ``attn_config.attn_uses_sequence_id``: document-masked attention against the PyTorch model."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _cfg(**kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch", attn_uses_sequence_id=True)
    return MPTConfig(**{**base, **kw})


def _batch(b, S, seed, vocab=2048):
    """Synthetic C4 rows (EOS = 0 every ~400 tokens, plus one forced early boundary) and their EOS-mode sequence ids."""
    from photon_b200.data.streaming import sequence_ids
    from photon_b200.data.synthetic import synthetic_batch

    ids = torch.from_numpy(synthetic_batch(b, S, seed=seed) % vocab)
    g = np.random.default_rng(seed)
    for r in range(b):   # more than one document per row even at S = 256
        for p in g.integers(1, S - 1, 3):
            ids[r, int(p)] = 0
    return ids.to(DEV), sequence_ids(ids, eos_token_id=0).to(DEV)


def _pair(cfg, kernels=None, **eng_kw):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    ref = TorchBackend(cfg, DEV, "fp32", seed=3)
    eng = B200Engine(cfg, DEV, "amp_bf16", dict(kernels or {}), seed=5, **eng_kw)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return ref, eng


def _match(ref, eng, ids, sid):
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    ref.flat.zero_grad(), eng.flat.zero_grad()
    l_ref, n_ref = ref.fwd_bwd(ids, denom, sequence_id=sid)
    l_eng, n_eng = eng.fwd_bwd(ids, denom, sequence_id=sid)
    torch.cuda.synchronize()
    assert int(n_ref) == int(n_eng)
    assert abs(float(l_ref) - float(l_eng)) / float(l_ref) < 5e-3, (float(l_ref), float(l_eng))
    cos = torch.nn.functional.cosine_similarity(ref.flat.grads, eng.flat.grads, dim=0).item()
    rel = ((ref.flat.grads - eng.flat.grads).norm() / ref.flat.grads.norm()).item()
    assert cos > 0.995 and rel < 0.08, (cos, rel)
    return float(l_ref)


@pytest.mark.parametrize("variant", ["learned", "alibi", "rope", "d_head_128"])
def test_doc_engine_matches_torch(variant):
    extra = {"learned": {}, "alibi": dict(alibi=True, learned_pos_emb=False), "rope": dict(rope=True, learned_pos_emb=False),
             "d_head_128": dict(n_heads=2)}[variant]
    ref, eng = _pair(_cfg(**extra), {"cuda_graph": False})
    assert eng.attn_mode == "b200"
    ids, sid = _batch(4, 256, seed=1)
    masked = _match(ref, eng, ids, sid)
    # the mask changes the model: the same batch as one document per row gives another loss
    plain = float(ref.fwd_bwd(ids, 1.0, sequence_id=torch.zeros_like(sid))[0])
    assert abs(masked - plain) > 1e-3 * abs(plain)
    # eval: with ids the mask applies, without them the plain causal mask
    a, b = ref.eval_stats(ids, sequence_id=sid), eng.eval_stats(ids, sequence_id=sid)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3
    a, b = ref.eval_stats(ids), eng.eval_stats(ids)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3


def test_doc_engine_activation_checkpointing_is_exact():
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(n_layers=3)
    a = B200Engine(cfg, DEV, "amp_bf16", {}, seed=5)
    b = B200Engine(cfg, DEV, "amp_bf16", {}, seed=5, activation_checkpointing=True)
    ids, sid = _batch(2, 256, seed=2)
    denom = float(ids.shape[0] * (ids.shape[1] - 1))
    a.flat.zero_grad(), b.flat.zero_grad()
    la, _ = a.fwd_bwd(ids, denom, sequence_id=sid)
    lb, _ = b.fwd_bwd(ids, denom, sequence_id=sid)
    torch.cuda.synchronize()
    assert float(la) == float(lb)
    rel = ((a.flat.grads - b.flat.grads).norm() / a.flat.grads.norm()).item()
    assert rel < 1e-3, rel


def test_doc_engine_cuda_graph_replay_matches_eager():
    """The captured graph reads sequence_id as a static input: a new document layout on every replay."""
    from photon_b200.models.engine import B200Engine

    cfg = _cfg()
    a = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
    b = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": True}, seed=5)
    a.flat.zero_grad(), b.flat.zero_grad()
    denom = float(2 * 255)
    for i in range(3):
        ids, sid = _batch(2, 256, seed=10 + i)
        la, _ = a.fwd_bwd(ids, denom, sequence_id=sid)
        lb, _ = b.fwd_bwd(ids, denom, sequence_id=sid)
        torch.cuda.synchronize()
        assert abs(float(la) - float(lb)) <= 1e-3 * abs(float(la)), (i, float(la), float(lb))
    assert list(b._graphs) == [(2, 256, 1.0 / denom, "doc")]
    rel = ((a.flat.grads - b.flat.grads).norm() / a.flat.grads.norm()).item()
    assert rel < 1e-3, rel
    assert b.launches_per_microbatch == a.launches_per_microbatch > 0


def test_flag_off_ignores_sequence_id():
    """Without attn_uses_sequence_id a batch's sequence_id changes nothing: the same launches, bitwise the same eval
    statistics, and training gradients within the spread of two identical runs (dQ and the embedding gradients
    accumulate with float atomics)."""
    from photon_b200 import ops
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(attn_uses_sequence_id=False)
    ids, sid = _batch(2, 256, seed=4)
    denom = float(2 * 255)
    runs = []
    for kw in ({}, {}, {"sequence_id": sid}):
        eng = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
        eng.flat.zero_grad()
        ops.reset_launch_count()
        loss, _ = eng.fwd_bwd(ids, denom, **kw)
        n = ops.launch_count()
        ev = eng.eval_stats(ids, **kw)
        torch.cuda.synchronize()
        runs.append((float(loss), n, eng.flat.grads.clone(), {k: float(v) for k, v in ev.items()}))
    (l0, n0, g0, e0), (l1, n1, g1, e1), (l2, n2, g2, e2) = runs
    assert n0 == n1 == n2
    assert e0 == e1 == e2
    noise = (g0 - g1).norm().item()
    assert (g0 - g2).norm().item() <= max(4 * noise, 1e-6 * g0.norm().item()), ((g0 - g2).norm().item(), noise)


def test_flag_on_training_without_sequence_id_raises():
    from photon_b200.models.engine import B200Engine

    eng = B200Engine(_cfg(), DEV, "amp_bf16", {}, seed=5)
    ids, _ = _batch(2, 256, seed=5)
    with pytest.raises(ValueError, match="sequence_id"):
        eng.fwd_bwd(ids, 1.0)


def test_doc_engine_library_attention_fallback_matches_torch():
    """S % 128 != 0: attention runs through SDPA with the boolean document mask."""
    ref, eng = _pair(_cfg(max_seq_len=200))
    ids, sid = _batch(4, 200, seed=6)
    _match(ref, eng, ids, sid)


def test_doc_engine_fp8_one_document_matches_flag_off():
    """amp_fp8 (attention stays bf16): one document per row with the flag on is the plain causal model."""
    from photon_b200.models.engine import B200Engine

    ids, _ = _batch(2, 256, seed=7)
    sid = torch.zeros_like(ids)
    denom = float(2 * 255)
    out = []
    for on, kw in ((False, {}), (False, {}), (True, {"sequence_id": sid})):
        eng = B200Engine(_cfg(attn_uses_sequence_id=on), DEV, "amp_fp8", {"cuda_graph": False}, seed=5)
        eng.flat.zero_grad()
        loss, _ = eng.fwd_bwd(ids, denom, **kw)
        torch.cuda.synchronize()
        out.append((float(loss), eng.flat.grads.clone()))
    (l0, g0), (l1, g1), (l2, g2) = out
    assert abs(l0 - l2) <= abs(l0 - l1), (l0, l1, l2)   # bitwise whenever two identical runs agree bitwise
    noise = (g0 - g1).norm().item()
    assert (g0 - g2).norm().item() <= max(4 * noise, 1e-6 * g0.norm().item()), ((g0 - g2).norm().item(), noise)


def test_doc_engine_zero3_world_size_one_matches_unsharded():
    """Full parameter sharding goes through the same attention calls: one rank matches the unsharded engine at the
    tolerance of test_zero3.py."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import NvlZero3Comm

    cfg = _cfg(n_layers=3)
    ids, sid = _batch(4, 256, seed=8)
    denom = float(4 * 255)
    plain = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=5)
    comm = NvlZero3Comm(plain.flat.layout, cfg.n_layers, rank=0, world_size=1, device=DEV)
    shard = B200Engine(cfg, DEV, "amp_bf16", {}, seed=5, zero3=comm)
    plain.flat.zero_grad(), shard.flat.zero_grad()
    la, _ = plain.fwd_bwd(ids, denom, sequence_id=sid)
    lb, _ = shard.fwd_bwd(ids, denom, sequence_id=sid)
    torch.cuda.synchronize()
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(la)), (float(la), float(lb))
    full = torch.zeros_like(plain.flat.grads)
    comm.plan.shard_to_full(shard.flat.grads, 0, full)
    rel = ((full - plain.flat.grads).norm() / plain.flat.grads.norm()).item()
    assert rel < 1e-5, rel
    comm.close()
