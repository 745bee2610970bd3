"""The whole sm_90a engine against the fp64 model (``model_oracle``), tensor by tensor, bounded by the pure-bf16 model.

Base shape: d_model 384 (6 heads of 64), 3 layers, max_seq_len 384 at S = 256 (``wpe`` rows 256.. must stay exactly zero),
B = 3, vocabulary 2008 (an N tail of 216 in the head GEMM, a K tail of 24 in its dgrad), FFN width 1352 and an LM-head chunk
of 320 rows, so T = 768 runs as chunks of 320, 320 and 128. Per model variant: a training step of two microbatches with
different loss scales (loss, token count, every gradient tensor), ``eval_stats`` (loss sum, correct predictions up to rows
the bf16 baseline itself cannot order) and ``engine.logits``; the KV decoder's logits after ``start`` and every ``step`` and
the scorer's log p for four variants; CUDA graphs with activation checkpointing, a freeze list and amp_fp8 as engine modes.
"""
import contextlib

import pytest
import torch

import model_oracle as MO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BASE = dict(d_model=384, n_heads=6, n_layers=3, max_seq_len=384, vocab_size=2008, ffn_hidden_size=1352)
B, S, CHUNK = 3, 256, 320
ROPE = dict(rope=True, learned_pos_emb=False)
VARIANTS = {
    "default": {},
    "no_bias": dict(no_bias=True),
    "alibi": dict(alibi=True, learned_pos_emb=False),
    "rope": ROPE,
    "qk_ln_clip": dict(qk_ln=True, clip_qkv=0.5),
    "d_head_128": dict(n_heads=3),
    "gqa": dict(kv_n_heads=2, qk_ln=True, **ROPE),
    "mqa": dict(kv_n_heads=1, qk_ln=True, **ROPE),
    "glu_silu": dict(ffn_type="mptglu", ffn_act="silu"),
    "mlp_silu_fractional": dict(ffn_act="silu", ffn_hidden_size=None, expansion_ratio=2.6875),   # width 1032
    "rmsnorm_qk_ln": dict(norm_type="rmsnorm", qk_ln=True),
    "doc": dict(attn_uses_sequence_id=True),
    "window_doc": dict(sliding_window_size=64, attn_uses_sequence_id=True),
    "softmax_scale": dict(softmax_scale=0.09),
    "tied_cap": dict(final_logit_softcapping=3.0),
    "untied_scale_cap": dict(tie_word_embeddings=False, logit_scale=1.7, final_logit_softcapping=4.0),
    "llama": dict(norm_type="rmsnorm", no_bias=True, ffn_type="mptglu", ffn_act="silu", ffn_hidden_size=1024,
                  tie_word_embeddings=False, kv_n_heads=2, **ROPE),
    "s200": {},
}
SEQ = {"s200": 200}
WORST: dict = {}   # part -> (worst ratio, where), over every check of the session


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\nworst ratios: " + "; ".join(f"{p} {r:.2f} ({w})" for p, (r, w) in sorted(WORST.items())))


@contextlib.contextmanager
def _exact_bf16_reduction():
    """The bf16 baseline's GEMMs accumulate in fp32 throughout, as the engine's do."""
    mm = torch.backends.cuda.matmul
    old = mm.allow_bf16_reduced_precision_reduction
    mm.allow_bf16_reduced_precision_reduction = False
    try:
        yield
    finally:
        mm.allow_bf16_reduced_precision_reduction = old


def _cfg(variant, **over):
    from photon_b200.models.mpt import MPTConfig

    return MPTConfig(**{**BASE, **VARIANTS[variant], **over})


def _engine(cfg, seed, precision="amp_bf16", kernels=None, **kw):
    """An engine whose weights (fp32 masters, bf16 shadow, frozen planes) are the bf16-exact test weights; returns it and them."""
    from photon_b200.models.engine import B200Engine

    eng = B200Engine(cfg, DEV, precision, {"cuda_graph": False, **(kernels or {})}, seed=seed, lm_head_chunk=CHUNK, **kw)
    w = MO.bf16_exact_weights(eng.model.named_parameters(), seed)
    with torch.no_grad():
        for n, p in eng.model.named_parameters():   # views of the flat fp32 masters and of the frozen plane
            p.copy_(w[n])
    eng.params_updated()
    return eng, w


def _batches(cfg, seq, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for scale in (1.0, 0.6):
        ids = torch.randint(0, cfg.vocab_size, (B, seq), generator=g)
        sid = None
        if cfg.attn_uses_sequence_id:   # documents of 1 .. ~120 tokens, boundaries anywhere (also inside 128-row tiles)
            sid = torch.cumsum((torch.rand(B, seq, generator=g) < 1 / 60).long(), 1)
        out.append(MO.Batch(ids, scale, 2.0 * B * (seq - 1), sid))
    return out


def _grads(eng):
    lay = eng.flat.layout
    return {n: lay.view(eng.flat.grads, n).clone() for n in lay.names}


def _train(eng, batches):
    """fwd_bwd of every microbatch into zeroed gradients; returns (loss sum, tokens, gradients after the first microbatch)."""
    eng.flat.zero_grad()
    loss, n, first = 0.0, 0, None
    for mb in batches:
        sid = None if mb.sequence_id is None else mb.sequence_id.to(DEV)
        l, t = eng.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale, sid)
        torch.cuda.synchronize()
        loss, n = loss + float(l), n + int(t)
        if first is None:
            first = _grads(eng)
    return loss, n, first


def _check_grads(chk, eng, ref, base):
    """Every gradient tensor. Without RoPE the QKV bias is checked as its q, k and v parts: the key part's exact gradient is
    zero or nearly so (see ``model_oracle.KNOWN``)."""
    c = eng.cfg
    for name in eng.flat.layout.names:
        g, o, b = eng.flat.layout.view(eng.flat.grads, name), ref.grads[name], base[name]
        if name.endswith("attn.Wqkv.bias") and not c.rope:
            d, kvd = c.d_model, c.kv_dim
            for part, sl in (("q", slice(0, d)), ("k", slice(d, d + kvd)), ("v", slice(d + kvd, d + 2 * kvd))):
                chk.tensor(f"{name}:{part}", g[sl], o[sl], b[sl])
        else:
            chk.tensor(name, g, o, b)


def _check_loss(chk, loss, ref, base):
    terr = torch.cat([(b - o).flatten() for b, o in zip(base.token_loss, ref.token_loss)])
    chk.sum("loss sum", loss, ref.loss_sum, MO.rms(terr), ref.n_tokens)


def _rows(x):
    return x.reshape(-1, x.shape[-1])


def _reference(cfg, w, batches, frozen=()):
    ref = MO.oracle(cfg, w, batches, frozen, device=DEV)
    with _exact_bf16_reduction():
        base = MO.baseline(cfg, w, batches, frozen, device=DEV)
    return ref, base


# ------------------------------------------------------------------------------------------------ training, eval, logits
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_engine_step_eval_and_logits_match_fp64(variant):
    from photon_b200.models.mpt import shift_labels

    cfg = _cfg(variant)
    seq = SEQ.get(variant, S)
    eng, w = _engine(cfg, seed=11)
    assert eng.attn_mode == "b200"
    batches = _batches(cfg, seq, seed=5)
    loss, n, first = _train(eng, batches)
    ref, base = _reference(cfg, w, batches)
    chk = MO.Checker(variant, worst=WORST)
    # ---- training step
    assert n == ref.n_tokens == 2 * B * (seq - 1)
    _check_loss(chk, loss, ref, base)
    _check_grads(chk, eng, ref, base.grads)
    if cfg.learned_pos_emb:
        chk.expect(bool((eng.flat.layout.view(eng.flat.grads, "transformer.wpe.weight")[seq:] == 0).all()),
                   "wpe rows past the sequence length are not zero")
    # ---- eval_stats on the first microbatch (same weights: no optimizer step ran)
    mb = batches[0]
    st = eng.eval_stats(mb.ids.to(DEV), None if mb.sequence_id is None else mb.sequence_id.to(DEV))
    terr = base.token_loss[0] - ref.token_loss[0]
    chk.sum("eval loss sum", float(st["loss_sum"]), float(ref.token_loss[0].sum()), MO.rms(terr), B * (seq - 1))
    assert int(st["n_tokens"]) == B * (seq - 1)
    lo, hi = MO.argmax_bounds(ref.logits[0], base.logits[0], shift_labels(mb.ids).to(DEV))
    print(f"[{variant}] n_correct {int(st['n_correct'])} in [{lo}, {hi}]")
    chk.expect(lo <= int(st["n_correct"]) <= hi, f"eval_stats n_correct {int(st['n_correct'])} outside [{lo}, {hi}]")
    # ---- engine.logits (the evaluator's path: no document ids, the head's transform applied)
    if mb.sequence_id is None:
        o_raw, b_raw = ref.logits[0], base.logits[0]
    else:
        one = [MO.Batch(mb.ids)]
        o_raw = MO.oracle(cfg, w, one, device=DEV, grad=False).logits[0]
        with _exact_bf16_reduction():
            b_raw = MO.baseline(cfg, w, one, device=DEV, grad=False).logits[0]
    got = eng.logits(mb.ids.to(DEV))
    o_log, b_log = _rows(MO.transformed(cfg, o_raw)), _rows(MO.transformed(cfg, b_raw.float()))
    chk.tensor("engine.logits", _rows(got), o_log, b_log)
    if variant in ("default", "untied_scale_cap"):
        _plants_flagged(cfg, seq, eng, ref, base, first, _rows(got), o_log, b_log)
    chk.finish()


def _plants_flagged(cfg, seq, eng, ref, base, first, logits, o_log, b_log):
    """The CPU plants applied to the engine's real gradients (and logits): the criterion measured on the H100 flags each."""
    planted = {label: (label.split(" ")[0], got) for label, got in MO.plants(cfg, seq, _grads(eng), first).items()}
    x = logits.double().clone()
    x[-MO.ROWS:] *= 1.02
    planted["engine.logits last 128 rows x1.02"] = ("engine.logits", x)
    missed = []
    for label, (name, got) in planted.items():
        r, b = (o_log, b_log) if name == "engine.logits" else (ref.grads[name], base.grads[name])
        rep = MO.tensor_report(name, got, r, b)
        print(f"plant {label}: flagged by {MO.failed_parts(rep)}: {rep['msg']}")
        if not MO.failed_parts(rep):
            missed.append(label)
    assert not missed, f"plants on the engine's output not flagged: {missed}"


# ------------------------------------------------------------------------------------------------ engine modes
def test_engine_graphs_and_checkpointing_match_fp64():
    cfg = _cfg("default")
    eng, w = _engine(cfg, seed=12, kernels={"cuda_graph": True}, activation_checkpointing=True)
    batches = _batches(cfg, S, seed=6)
    loss, n, _ = _train(eng, batches)
    assert len(eng._graphs) == 2   # one capture per loss scale  # noqa: SLF001
    ref, base = _reference(cfg, w, batches)
    chk = MO.Checker("graphs_ckpt", worst=WORST)
    _check_loss(chk, loss, ref, base)
    _check_grads(chk, eng, ref, base.grads)
    chk.finish()


FROZEN = ["transformer.blocks.0.attn.Wqkv.weight", "transformer.blocks.0.norm_1.bias", "transformer.blocks.1.ffn.up_proj.bias",
          "transformer.blocks.2.attn.out_proj.weight", "transformer.wpe.weight", "transformer.norm_f.weight"]


def test_engine_freeze_list_matches_fp64():
    cfg = _cfg("default")
    eng, w = _engine(cfg, seed=13, frozen_layers=FROZEN)
    assert not set(FROZEN) & set(eng.flat.layout.names)   # frozen tensors have no gradient slot at all
    before = eng.frozen_params.clone()
    batches = _batches(cfg, S, seed=7)
    loss, n, _ = _train(eng, batches)
    assert torch.equal(eng.frozen_params, before)
    ref, base = _reference(cfg, w, batches, FROZEN)
    for f in FROZEN:
        assert not ref.grads[f].any()
    chk = MO.Checker("frozen", worst=WORST)
    _check_loss(chk, loss, ref, base)
    _check_grads(chk, eng, ref, base.grads)
    chk.finish()


@pytest.mark.parametrize("variant", ["default", "rmsnorm_rope_gqa_untied"])
def test_engine_amp_fp8_matches_fp64(variant):
    """amp_fp8 (E4M3 / E5M2 block GEMMs) against the fp64 model, bounded by the TorchBackend("amp_fp8") emulation."""
    from photon_b200.train.backend import TorchBackend

    extra = {} if variant == "default" else dict(norm_type="rmsnorm", kv_n_heads=2, tie_word_embeddings=False, **ROPE)
    cfg = _cfg("default", ffn_hidden_size=1360, **extra)   # E4M3 rows of the FFN width must be 16-byte multiples
    eng, w = _engine(cfg, seed=14, precision="amp_fp8")
    batches = _batches(cfg, S, seed=8)
    loss, n, _ = _train(eng, batches)
    ref = MO.oracle(cfg, w, batches, device=DEV)
    emu = TorchBackend(cfg, DEV, "amp_fp8", seed=14)
    with torch.no_grad():
        for name, p in emu.model.named_parameters():
            p.copy_(w[name])
    emu.flat.zero_grad()
    eloss = 0.0
    with _exact_bf16_reduction():
        for mb in batches:
            eloss += float(emu.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale)[0])
    chk = MO.Checker(f"fp8:{variant}", MO.FP8, worst=WORST)
    # the emulation's loss is one number: its error stands for the per-token errors' sum
    chk.sum("loss sum", loss, ref.loss_sum, abs(eloss - ref.loss_sum), 1)
    _check_grads(chk, eng, ref, {name: emu.flat.layout.view(emu.flat.grads, name) for name in emu.flat.layout.names})
    chk.finish()


# ------------------------------------------------------------------------------------------------ decoder and scorer
SERVE = ["default", "gqa", "untied_scale_cap", "window_doc"]


@pytest.mark.parametrize("variant", SERVE)
def test_decoder_logits_match_fp64(variant):
    """``dec.logits`` after ``start`` and after every ``step`` against the oracle's logits of the same prefix: the prompt
    followed by the tokens the decoder chose."""
    cfg = _cfg(variant)
    eng, w = _engine(cfg, seed=15, kernels={"cuda_graph": True})
    dec = eng.decoder(3)
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in (37, 128, 201)]
    K = 5
    toks = [dec.start(prompts, K + 1)]
    got = [dec.logits.clone()]
    for _ in range(K):
        toks.append(dec.step())
        got.append(dec.logits.clone())
    refs, bases = [], []
    for i, p in enumerate(prompts):
        seq = [MO.Batch(torch.tensor(p + [t[i] for t in toks[:K]])[None])]
        rows = slice(len(p) - 1, len(p) + K)
        refs.append(MO.oracle(cfg, w, seq, device=DEV, grad=False).logits[0][0, rows])
        with _exact_bf16_reduction():
            bases.append(MO.baseline(cfg, w, seq, device=DEV, grad=False).logits[0][0, rows])
    got = torch.stack(got, 1).reshape(-1, cfg.vocab_size)          # rows: (prompt, step)
    ref, base = torch.stack(refs).reshape(-1, cfg.vocab_size), torch.stack(bases).reshape(-1, cfg.vocab_size)
    chk = MO.Checker(f"decoder:{variant}", worst=WORST)
    chk.tensor("decoder logits", got, ref, base)
    chk.finish()


@pytest.mark.parametrize("variant", SERVE)
def test_scorer_log_probs_match_fp64(variant):
    """Each pair's log p against the oracle's (bounded by the baseline's per-token log p errors pooled over the call), and
    its argmax flag wherever no scored row is ambiguous for bf16 arithmetic."""
    cfg = _cfg(variant)
    eng, w = _engine(cfg, seed=16)
    dec = eng.decoder(4)
    g = torch.Generator().manual_seed(10)
    r = lambda n: torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist()  # noqa: E731
    a, b, c = r(50), r(130), r(1)
    pairs = [(a, r(3)), (a, r(1)), (b, r(5)), (c, r(70))]
    got = dec.score(pairs)
    per_pair, errs = [], []
    for ctx, sc in pairs:
        seq = [MO.Batch(torch.tensor(ctx + sc)[None])]
        rows = slice(len(ctx) - 1, len(ctx) + len(sc) - 1)
        o_raw = MO.oracle(cfg, w, seq, device=DEV, grad=False).logits[0][0, rows]
        with _exact_bf16_reduction():
            b_raw = MO.baseline(cfg, w, seq, device=DEV, grad=False).logits[0][0, rows].float()
        tgt, at = torch.tensor(sc, device=DEV), torch.arange(len(sc), device=DEV)
        lp_o = MO.transformed(cfg, o_raw).log_softmax(-1)[at, tgt]
        lp_b = MO.transformed(cfg, b_raw).double().log_softmax(-1)[at, tgt]
        errs.append(lp_b - lp_o)
        per_pair.append((float(lp_o.sum()), bool((o_raw.argmax(-1) == tgt).all()), bool(MO.ambiguous_rows(o_raw, b_raw).any())))
    chk = MO.Checker(f"scorer:{variant}", worst=WORST)
    e = MO.rms(torch.cat(errs))
    for (ctx, sc), (lp, hit), (lp_o, hit_o, amb) in zip(pairs, got, per_pair):
        chk.sum(f"log p of {len(sc)} tokens after {len(ctx)}", lp, lp_o, e, len(sc))
        chk.expect(amb or hit == hit_o, f"argmax flag {hit} of {len(sc)} tokens after {len(ctx)}, oracle {hit_o}")
    chk.finish()


# ------------------------------------------------------------------------------------------------ clip_qkv on the clip
def test_clip_qkv_passes_gradient_on_the_clip():
    """Features whose Wqkv row is zero and whose bias is exactly +-clip_qkv sit on the clip for every token. torch.clamp (and
    llm-foundry's clamp_) pass the gradient there: the engine's bias gradients of those features must match the PyTorch
    model's and be nonzero."""
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048, clip_qkv=0.5)
    eng, w = _engine(cfg, seed=17)
    d, kvd = cfg.d_model, cfg.kv_dim
    # q and v features (a k feature that is the same for every key shifts whole score rows: its gradient is zero anyway)
    feats = [3, 70, d + kvd + 7, d + kvd + 200]
    for i in range(cfg.n_layers):
        w[f"transformer.blocks.{i}.attn.Wqkv.weight"][feats] = 0.0
        w[f"transformer.blocks.{i}.attn.Wqkv.bias"][feats] = torch.tensor([0.5, -0.5] * 2)
    with torch.no_grad():
        for n, p in eng.model.named_parameters():
            p.copy_(w[n])
    eng.params_updated()
    ref = TorchBackend(cfg, DEV, "fp32", seed=17)
    with torch.no_grad():
        for n, p in ref.model.named_parameters():
            p.copy_(w[n])
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=torch.Generator().manual_seed(3)).to(DEV)
    ref.flat.zero_grad(), eng.flat.zero_grad()
    ref.fwd_bwd(ids, 510.0)
    eng.fwd_bwd(ids, 510.0)
    torch.cuda.synchronize()
    for i in range(cfg.n_layers):
        name = f"transformer.blocks.{i}.attn.Wqkv.bias"
        a = ref.flat.layout.view(ref.flat.grads, name)[feats].double()
        b = eng.flat.layout.view(eng.flat.grads, name)[feats].double()
        print(name, a.tolist(), b.tolist())
        assert bool((a != 0).all()), a
        assert float((a - b).norm() / a.norm()) < 0.05, (a.tolist(), b.tolist())
