"""KV-cached greedy decoding on the engine: the skinny GEMM, decode attention, and the decoder against the fp32 model."""
import json
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
# bf16 tolerance on log-probabilities of the decoder vs the fp32 model (2-layer d_model 256 model): the bf16 weights and
# activations move each log-probability by a few 1e-2 at most
LOGP_TOL = 0.15


# ----------------------------------------------------------------------------------------------- skinny GEMM
SHAPES = [(768, 768), (768, 2304), (2048, 6144), (8192, 768), (768, 50368), (2048, 2304), (776, 1000)]


@pytest.mark.parametrize("M", [1, 3, 16, 64])
@pytest.mark.parametrize("K,N", SHAPES)
def test_skinny_gemm_matches_fp32_every_epilogue(M, K, N):
    from photon_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(M * 7 + K + N)
    x = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g)
    res = torch.randn(M, N, device=DEV, generator=g).bfloat16()
    ref = x.float() @ w.float().t()
    cases = {"plain": (None, None, False, ref), "bias": (bias, None, False, ref + bias),
             "residual": (bias, res, False, ref + bias + res.float()),
             "gelu": (bias, None, True, torch.nn.functional.gelu(ref + bias))}
    for name, (b, r, gelu, want) in cases.items():
        out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        ops.skinny_gemm(x, w, out, b, r, gelu)
        again = torch.empty_like(out)
        ops.skinny_gemm(x, w, again, b, r, gelu)
        torch.cuda.synchronize()
        torch.testing.assert_close(out.float(), want, rtol=2e-2, atol=3e-2, msg=lambda m: f"{name}: {m}")
        assert torch.equal(out, again), f"{name}: two runs differ"


def test_skinny_gemm_rejects_more_than_64_rows():
    from photon_b200 import ops

    x = torch.zeros(65, 768, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(768, 768, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="M <= 64"):
        ops.skinny_gemm(x, w, torch.empty(65, 768, dtype=torch.bfloat16, device=DEV))


# ------------------------------------------------------------------------------------------ decode attention
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
def test_decode_attention_ragged_matches_fp32(dh, alibi):
    """Each (sequence, head) row against the fp64 oracle, bounded by the bf16 baseline of the same row. The cache is one
    sequence per batch row, the query that sequence's row at position len - 1. Lengths 1000 and 2048 split into 4 and 8
    256-key partials, so the combine kernel merges several of them; peaked and rising inputs make one partial dominate."""
    import attention_oracle as A
    from photon_b200 import ops
    from photon_b200.models.mpt import alibi_slopes

    lens = [1, 2, 127, 128, 129, 1000, 2048]
    B, H, S = len(lens), 4, 2048
    slopes = alibi_slopes(H).to(DEV) if alibi else None
    scale = 1.0 / math.sqrt(dh)
    pos = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=DEV)
    for case in ("normal", "peaked", "rising"):
        seq, _ = A.make_inputs(case, B, S, H, dh, DEV, seed=dh + alibi)
        q, k, v = A.split_heads(seq, H)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = seq[torch.arange(B, device=DEV), pos.long()].contiguous()   # each sequence's row at its last position
        out = torch.empty(B, H * dh, dtype=torch.bfloat16, device=DEV)
        ops.decode_attention(qkv, kc, vc, pos, out, H, scale, slopes)
        again = torch.empty_like(out)
        ops.decode_attention(qkv, kc, vc, pos, again, H, scale, slopes)
        torch.cuda.synchronize()
        assert torch.equal(out, again)
        qr = qkv[:, : H * dh].view(B, H, 1, dh)
        kw = dict(causal=True, slopes=None if slopes is None else slopes.tolist(), q_pos=pos.long()[:, None], lengths=lens)
        ref, base = A.oracle(qr, kc, vc, scale, **kw), A.baseline(qr, kc, vc, scale, **kw)
        A.check("decode o", out.view(B, H, 1, dh), ref.o, base.o, rows=1, case=f"{case}, lens {lens}", whole_mean=True)


# ------------------------------------------------------------------------------------------------ engine
VARIANTS = {"default": {}, "alibi": dict(alibi=True, learned_pos_emb=False), "rope": dict(rope=True, learned_pos_emb=False),
            "qk_ln": dict(qk_ln=True), "clip_qkv": dict(clip_qkv=0.5), "no_bias": dict(no_bias=True), "d_head_128": dict(n_heads=2),
            "amp_fp8": {}}
PROMPT_LENS = [3, 50, 129, 200]
STEPS = 16


def _engine(variant="default", seed=5, cuda_graph=True):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    extra = dict(VARIANTS[variant])
    heads = extra.pop("n_heads", 4)
    cfg = MPTConfig(d_model=256, n_heads=heads, n_layers=2, max_seq_len=256, vocab_size=2048, attn_impl="torch", **extra)
    ref = TorchBackend(cfg, DEV, "fp32", seed=3)
    eng = B200Engine(cfg, DEV, "amp_fp8" if variant == "amp_fp8" else "amp_bf16", {"cuda_graph": cuda_graph}, seed=seed)
    eng.flat.params.copy_(ref.flat.params)
    eng.params_updated()
    return cfg, ref, eng


def _prompts(cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in PROMPT_LENS]


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_decoder_matches_fp32_model(variant):
    cfg, ref, eng = _engine(variant)
    dec = eng.decoder(len(PROMPT_LENS))
    assert dec is not None
    prompts = _prompts(cfg)
    seqs = [list(p) for p in prompts]
    follow = [True] * len(seqs)   # the row still is the fp32 model's own greedy path
    toks = dec.start(prompts, STEPS)
    for t in range(STEPS):
        got = torch.log_softmax(dec.logits.float(), -1)
        for i, s in enumerate(seqs):
            with torch.no_grad():
                want = torch.log_softmax(ref.logits(torch.tensor([s], device=DEV))[0, -1].float(), -1)
            err = (got[i] - want).abs().max().item()
            assert err < LOGP_TOL, (variant, t, i, err)
            top2 = want.topk(2).values
            if follow[i] and (top2[0] - top2[1]).item() < LOGP_TOL:
                follow[i] = False   # a near-tie: bf16 may pick the other token from here on
            if follow[i]:
                assert toks[i] == int(want.argmax()), (variant, t, i)
            s.append(toks[i])
        if t < STEPS - 1:
            toks = dec.step()


def test_decoder_graph_replay_equals_eager_and_repeats_bitwise():
    cfg, _, eng = _engine()
    prompts = _prompts(cfg, seed=1)

    def run(use_graph):
        from photon_b200.models.decode import KVDecoder

        dec = KVDecoder(eng, 4, use_graph=use_graph)
        out = [dec.start(prompts, STEPS)]
        out += [dec.step() for _ in range(STEPS - 1)]
        return out, dec.logits.clone()

    eager, l_eager = run(False)
    graph, l_graph = run(True)
    graph2, l_graph2 = run(True)
    assert eager == graph == graph2
    assert torch.equal(l_eager, l_graph) and torch.equal(l_graph, l_graph2)


def test_decoder_refuses_rows_past_the_cache():
    cfg, _, eng = _engine()
    dec = eng.decoder(2)
    with pytest.raises(ValueError, match="does not fit"):
        dec.start([[1] * 250], 16)


def test_generation_leaves_training_untouched():
    cfg, _, eng = _engine()
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device=DEV)
    denom = float(ids.numel())
    eng.flat.zero_grad()
    eng.fwd_bwd(ids, denom)
    before = eng.flat.grads.clone()
    params, shadow = eng.flat.params.clone(), eng.bf16_params.clone()
    graphs, ws = dict(eng._graphs), dict(eng._ws)
    dec = eng.decoder(4)
    dec.start(_prompts(cfg), 8)
    for _ in range(7):
        dec.step()
    torch.cuda.synchronize()
    assert torch.equal(params, eng.flat.params) and torch.equal(shadow, eng.bf16_params)
    assert graphs.keys() == eng._graphs.keys() and all(graphs[k] is eng._graphs[k] for k in graphs)
    assert ws.keys() == eng._ws.keys() and all(ws[k] is eng._ws[k] for k in ws)
    eng.flat.zero_grad()
    eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    # the training step itself is not bitwise reproducible (the embedding-gradient scatter and the attention dQ accumulate
    # with float atomics), so the replayed step is compared to the one before the generation at fp32-atomics noise level
    after = eng.flat.grads
    assert ((after - before).norm() / before.norm()).item() < 1e-3
    assert torch.nn.functional.cosine_similarity(after, before, dim=0).item() > 0.99999


def test_trainer_eval_generation_task_uses_decoder(tmp_path):
    from photon_b200.dataset.utils import ByteTokenizer
    from photon_b200.eval.icl import run_icl_suite
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.trainer import Trainer

    rows = [{"context": "ab", "answer": "c"}, {"context": "x" * 40, "answer": "y"}, {"context": "q", "answer": "r"}]
    (tmp_path / "gen.jsonl").write_text("\n".join(json.dumps(r) for r in rows))
    icl = {"icl_tasks_config": {"root_dir": str(tmp_path), "icl_tasks": [
        {"label": "gen", "dataset_uri": "gen.jsonl", "icl_task_type": "generation_task_with_answers", "max_new_tokens": 6,
         "batch_size": 2, "early_stopping_criteria": ["\n"]}]}}
    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=512)
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len))

    class Loader:
        def __iter__(self):
            while True:
                yield {"input_ids": ids, "labels": ids}

    tr = Trainer(cfg, optimizer_cfg=dict(name="adopt", lr=1e-3, betas=[0.9, 0.9999], eps=1e-6, weight_decay=0.0),
                 scheduler_cfg=dict(name="cosine_with_warmup", t_warmup="1ba", t_max="10ba", alpha_f=0.1), train_loader=Loader(),
                 global_train_batch_size=2, device_train_microbatch_size=2, precision="amp_bf16", max_duration="10ba", device=DEV)
    assert tr.state.backend.kind == "b200"
    starts = []

    def suite(logits_fn, decoder=None):
        assert decoder is not None
        orig = decoder.start

        def spy(prompts, n):
            starts.append(len(prompts))
            return orig(prompts, n)

        decoder.start = spy
        return run_icl_suite(logits_fn, ByteTokenizer(), icl, cfg.max_seq_len, decoder=decoder)

    tr.icl_suite = suite
    vals = tr.eval()
    assert starts == [2, 1]   # the task's batch_size
    recompute = run_icl_suite(tr.state.backend.logits, ByteTokenizer(), icl, cfg.max_seq_len)
    assert {k for k in vals if k.startswith("icl/")} == {f"icl/{k}" for k in recompute}
    tr.close()
