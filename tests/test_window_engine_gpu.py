"""B200Engine with ``attn_config.sliding_window_size`` (and ``softmax_scale``) against the fp32 PyTorch model: training alone,
with the document mask and in a Mistral-style combination, amp_fp8, ZeRO-3, activation checkpointing and CUDA graphs, the
library fallback, and the KV-cached decoder and scorer past the window."""
import pytest
import torch

from test_gqa_engine_gpu import LOGP_TOL, _ids, _match

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
MISTRAL = dict(rope=True, learned_pos_emb=False, kv_n_heads=2, norm_type="rmsnorm", ffn_type="mptglu", ffn_act="silu", no_bias=True,
               softmax_scale=0.1)


def _cfg(**kw):
    from photon_b200.models.mpt import MPTConfig

    base = dict(d_model=512, n_heads=8, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch", sliding_window_size=40)
    return MPTConfig(**{**base, **kw})


def _pair(cfg, precision="amp_bf16", kernels=None, **eng_kw):
    from photon_b200.models.engine import B200Engine
    from photon_b200.train.backend import TorchBackend

    ref = TorchBackend(cfg, DEV, "fp32", seed=3)
    eng = B200Engine(cfg, DEV, precision, dict(kernels or {"cuda_graph": False}), seed=5, **eng_kw)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return ref, eng


VARIANTS = {"plain": {}, "w0": dict(sliding_window_size=0), "w130": dict(sliding_window_size=130),
            "alibi": dict(alibi=True, learned_pos_emb=False), "d_head_128": dict(n_heads=4, sliding_window_size=129),
            "scale_only": dict(sliding_window_size=-1, softmax_scale=0.3), "mistral": MISTRAL}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_window_engine_matches_torch(variant):
    ref, eng = _pair(_cfg(**VARIANTS[variant]))
    assert eng.attn_mode == "b200"
    _match(ref, eng, _ids(4, 256, 1))
    a, b = ref.eval_stats(_ids(2, 256, 2)), eng.eval_stats(_ids(2, 256, 2))
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) / float(a["loss_sum"]) < 5e-3
    with torch.no_grad():
        la, lb = ref.logits(_ids(1, 256, 3)).float(), eng.logits(_ids(1, 256, 3)).float()
    assert ((la - lb).norm() / la.norm()).item() < 4e-2   # bf16 engine against fp32 model; 0.026 measured at softmax_scale 0.3


def test_window_changes_the_engine_loss():
    from photon_b200.models.engine import B200Engine

    ids = _ids(2, 256, 4)
    losses = [float(B200Engine(_cfg(sliding_window_size=w), DEV, "amp_bf16", {"cuda_graph": False}, seed=5).fwd_bwd(ids, 510.0)[0])
              for w in (-1, 255, 40)]
    assert losses[0] == losses[1] and losses[2] != losses[0], losses


@pytest.mark.parametrize("variant", ["plain", "mistral"])
def test_window_engine_document_mask(variant):
    from test_doc_engine_gpu import _batch

    ref, eng = _pair(_cfg(attn_uses_sequence_id=True, **({"rope": True, "learned_pos_emb": False} if variant == "plain" else MISTRAL)))
    ids, sid = _batch(4, 256, seed=1)
    _match(ref, eng, ids, sid)


def test_window_engine_amp_fp8_against_bf16():
    ref, eng = _pair(_cfg(), precision="amp_fp8")
    _, bf = _pair(_cfg())
    assert eng.fp8
    ids, denom = _ids(4, 256, 1), float(4 * 255)
    for e in (eng, bf):
        e.flat.zero_grad()
    l8, lb = float(eng.fwd_bwd(ids, denom)[0]), float(bf.fwd_bwd(ids, denom)[0])
    torch.cuda.synchronize()
    assert abs(l8 - lb) / lb < 2e-2, (l8, lb)
    cos = torch.nn.functional.cosine_similarity(eng.flat.grads, bf.flat.grads, dim=0).item()
    assert cos > 0.97, cos
    _match(ref, eng, ids, tol=(2e-2, 0.97, 0.25, 0.35))


def test_window_engine_full_sharding_equals_unsharded():
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import NvlZero3Comm

    cfg = _cfg(n_layers=3, kv_n_heads=2, softmax_scale=0.2)
    for precision in ("amp_bf16", "amp_fp8"):
        plain = B200Engine(cfg, DEV, precision, {"cuda_graph": False}, seed=5)
        comm = NvlZero3Comm(plain.flat.layout, cfg.n_layers, rank=0, world_size=1, device=DEV, fp8=precision == "amp_fp8")
        shard = B200Engine(cfg, DEV, precision, {}, seed=5, zero3=comm)
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


def test_window_engine_activation_checkpointing_graphs_and_launches():
    from photon_b200 import ops
    from photon_b200.models.engine import B200Engine

    cfg = _cfg(n_layers=3, qk_ln=True, rope=True, learned_pos_emb=False, softmax_scale=0.15)
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
    causal = B200Engine(_cfg(n_layers=3, qk_ln=True, rope=True, learned_pos_emb=False, sliding_window_size=-1), DEV, "amp_bf16",
                        {"cuda_graph": False}, seed=5)
    counts = []
    for e in (eager, causal):
        e.fwd_bwd(_ids(2, 256, 20), denom)
        torch.cuda.synchronize()
        ops.reset_launch_count()
        e.fwd_bwd(_ids(2, 256, 21), denom)
        torch.cuda.synchronize()
        counts.append(ops.launch_count())
    assert counts[0] == counts[1], counts


@pytest.mark.parametrize("how", ["kernels_torch", "seq_not_multiple_of_128"])
def test_window_engine_library_fallback(how):
    if how == "kernels_torch":
        ref, eng = _pair(_cfg(alibi=True, learned_pos_emb=False, softmax_scale=0.2), kernels={"cuda_graph": False, "attention": "torch"})
        assert eng.attn_mode == "torch"
        _match(ref, eng, _ids(4, 256, 1))
    else:
        ref, eng = _pair(_cfg(softmax_scale=0.2))
        _match(ref, eng, _ids(4, 200, 1))


# ------------------------------------------------------------------------------------------------ decoding and scoring
def _follow(ref, dec, prompts, n_new):
    seqs = [list(p) for p in prompts]
    follow = [True] * len(seqs)
    toks = dec.start(prompts, n_new)
    for t in range(n_new):
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
        if t < n_new - 1:
            toks = dec.step()


@pytest.mark.parametrize("variant", ["plain", "alibi", "mistral"])
def test_window_decoder_follows_the_model_past_the_window(variant):
    """Prompts shorter and longer than W = 300, 24 new tokens: positions past W, decode chunks wholly below the window."""
    kw = dict(VARIANTS[variant], max_seq_len=1024, sliding_window_size=300)
    ref, eng = _pair(_cfg(**kw), kernels={"cuda_graph": True})
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(0, 2048, (n,), generator=g).tolist() for n in (3, 290, 400, 700)]
    dec = eng.decoder(len(prompts))
    _follow(ref, dec, prompts, 24)


def test_window_score_matches_the_model():
    from test_score_gpu import _fp32_stats, _pairs

    ref, eng = _pair(_cfg(rope=True, learned_pos_emb=False, kv_n_heads=2, softmax_scale=0.1))
    pairs = _pairs(eng.cfg)
    assert max(len(c) + len(s) for c, s in pairs) > eng.cfg.sliding_window_size
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (i, lp, want_lp)
        if clear:
            assert hit == want_hit, i
