"""B200Engine with grouped-query (kv_n_heads 2 of 8 heads) and multi-query (1 of 8) attention against the PyTorch model, and the
KV-cached decoder / scorer over the smaller cache."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
KV = [pytest.param(2, id="gqa2"), pytest.param(1, id="mqa")]
LOGP_TOL = 0.15   # as test_decode_gpu.py


def _cfg(kv, **kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=512, n_heads=8, kv_n_heads=kv, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch")
    return MPTConfig(**{**base, **kw})


def _pair(cfg, precision="amp_bf16", kernels=None, **eng_kw):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    ref = TorchBackend(cfg, DEV, "fp32", seed=3)
    eng = B200Engine(cfg, DEV, precision, dict(kernels or {"cuda_graph": False}), seed=5, **eng_kw)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return ref, eng


def _ids(b, S, seed):
    return torch.randint(0, 2048, (b, S), device=DEV, generator=torch.Generator("cuda").manual_seed(seed))


def _match(ref, eng, ids, sid=None, tol=(5e-3, 0.995, 0.08, 0.08)):
    """tol: loss relative error, whole-gradient cosine and relative L2 error, relative L2 error of each trainable fused QKV
    gradient."""
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
    for name in ("transformer.blocks.0.attn.Wqkv.weight", "transformer.blocks.1.attn.Wqkv.bias"):
        if name in lay.names:
            a, b = lay.view(g_ref, name), lay.view(g_eng, name)
            assert ((a - b).norm() / a.norm()).item() < tol[3], name


VARIANTS = {"plain": {}, "rope_qkln_clip": dict(rope=True, learned_pos_emb=False, qk_ln=True, clip_qkv=0.8),
            "alibi": dict(alibi=True, learned_pos_emb=False), "d_head_128": dict(n_heads=4)}


@pytest.mark.parametrize("kv", KV)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_gqa_engine_matches_torch(kv, variant):
    ref, eng = _pair(_cfg(kv, **VARIANTS[variant]))
    assert eng.attn_mode == "b200"
    assert eng.layers[0].wqkv.shape == (eng.cfg.qkv_dim, 512)
    _match(ref, eng, _ids(4, 256, 1))
    a, b = ref.eval_stats(_ids(2, 256, 2)), eng.eval_stats(_ids(2, 256, 2))
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3


@pytest.mark.parametrize("kv", KV)
def test_gqa_engine_document_mask(kv):
    from test_doc_engine_gpu import _batch

    ref, eng = _pair(_cfg(kv, attn_uses_sequence_id=True, rope=True, learned_pos_emb=False))
    ids, sid = _batch(4, 256, seed=1)
    _match(ref, eng, ids, sid)


@pytest.mark.parametrize("kv", KV)
def test_gqa_engine_amp_fp8(kv):
    """As test_fp8_gpu's engine check: fp8 GEMMs against the fp32 model, with the looser fp8 bounds."""
    ref, eng = _pair(_cfg(kv), precision="amp_fp8")
    assert eng.fp8 and tuple(eng.w8_views[0]["wqkv"].shape) == (eng.cfg.qkv_dim, 512)
    _match(ref, eng, _ids(4, 256, 1), tol=(2e-2, 0.97, 0.25, 0.35))


@pytest.mark.parametrize("kv", KV)
def test_gqa_engine_activation_checkpointing_and_graphs(kv):
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(kv, n_layers=3, qk_ln=True, rope=True, learned_pos_emb=False)
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


@pytest.mark.parametrize("kv", KV)
def test_gqa_engine_freeze_list(kv):
    """Frozen tensors of the GQA shapes (the fused projection, the narrower k_ln) live in the frozen planes; the same seed gives
    the engine and the model the same frozen values."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    frozen = ["transformer.blocks.0.attn.Wqkv.weight", "transformer.blocks.0.attn.k_ln.weight", "transformer.wte.weight"]
    cfg = _cfg(kv, qk_ln=True)
    ref = TorchBackend(cfg, DEV, "fp32", seed=3, frozen_layers=frozen)
    eng = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=3, frozen_layers=frozen)
    assert eng.flat.layout.names == ref.flat.layout.names and set(eng.frozen_layout.names) == set(frozen)
    assert eng.frozen_layout.shapes[eng.frozen_layout.index(frozen[1])] == (kv * 64,)
    _match(ref, eng, _ids(4, 256, 3))


def test_gqa_engine_full_sharding_equals_unsharded():
    """One rank's ZeRO-3 communicator (world size 1): the unit plan and the bf16 / E4M3 pieces take the GQA shapes from the
    layout, and training matches the unsharded engine."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import NvlZero3Comm

    cfg = _cfg(2, n_layers=3)
    for precision in ("amp_bf16", "amp_fp8"):
        plain = B200Engine(cfg, DEV, precision, {"cuda_graph": False}, seed=5)
        comm = NvlZero3Comm(plain.flat.layout, cfg.n_layers, rank=0, world_size=1, device=DEV, fp8=precision == "amp_fp8")
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
        g = shard.flat.grads[: plain.flat.grads.numel()]
        rel = ((g - plain.flat.grads).norm() / plain.flat.grads.norm()).item()
        assert rel < 2e-3, (precision, rel)
        comm.close()


# ------------------------------------------------------------------------------------------------ decoding and scoring
def _prompts(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 2048, (n,), generator=g).tolist() for n in (3, 50, 129, 200)]


@pytest.mark.parametrize("kv", KV)
@pytest.mark.parametrize("variant", ["plain", "rope_qkln_clip", "alibi"])
def test_gqa_decoder_follows_the_model(kv, variant):
    """Greedy tokens of the cached decoder against the fp32 model recomputed over the whole sequence at every step, and its
    cache holds only the kv heads."""
    ref, eng = _pair(_cfg(kv, **VARIANTS[variant]), kernels={"cuda_graph": True})
    prompts = _prompts()
    dec = eng.decoder(len(prompts))
    assert dec is not None
    seqs = [list(p) for p in prompts]
    follow = [True] * len(seqs)
    toks = dec.start(prompts, 16)
    assert dec.cache.shape[3] == kv
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


@pytest.mark.parametrize("kv", KV)
def test_gqa_score_matches_the_model(kv):
    from test_score_gpu import _fp32_stats, _pairs

    ref, eng = _pair(_cfg(kv, rope=True, learned_pos_emb=False))
    pairs = _pairs(eng.cfg)
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (i, lp, want_lp)
        if clear:
            assert hit == want_hit, i
