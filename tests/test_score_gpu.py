"""Log-likelihood scoring on the engine: cache attention, slotted cache appends, and ``KVDecoder.score`` against the fp32 model."""
import json
import math

import pytest
import torch

from test_decode_gpu import DEV, LOGP_TOL, VARIANTS, _engine

pytestmark = pytest.mark.gpu

SENTINEL = 7.0


# ------------------------------------------------------------------------------------------ cache attention
# (slot, n_rows, first_pos): prefixes 1, 127, 128, 129, 1000, 2047; tiles of 1, 2, 63 and 64 rows; runs of 65 and 200 rows that
# split into 64-row tiles; several runs on slots 0 and 1
RUNS = [(0, 1, 1), (0, 2, 300), (1, 64, 127), (1, 63, 1000), (2, 65, 128), (3, 200, 129), (4, 63, 1000), (5, 1, 2047), (0, 2, 1)]
GAP = 3   # untouched rows between runs


def _layout(runs):
    out, row = [], GAP
    for slot, n, p in runs:
        out.append((slot, row, n, p))
        row += n + GAP
    return out, row


@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
def test_cache_attention_matches_fp32(dh, alibi):
    """Every tile of the tile table against the fp64 oracle at its rows' own cache positions, bounded by the bf16 baseline of
    the same tile (the max part per tile and head, the mean part over all rows). The query rows of a run are the slot's own
    sequence at positions first_pos .. first_pos + n - 1."""
    import attention_oracle as A
    from photon_b200 import ops
    from photon_b200.models.mpt import alibi_slopes

    H, S, Bm = 3, 2048, 6
    runs, N = _layout(RUNS)
    slopes = alibi_slopes(H).to(DEV) if alibi else None
    scale = 1.0 / math.sqrt(dh)
    tiles = ops.cache_tiles(runs, DEV)
    assert tiles.shape[0] == 1 + 1 + 1 + 1 + 2 + 4 + 1 + 1 + 1
    for case in ("normal", "peaked", "rising"):
        seq, _ = A.make_inputs(case, Bm, S, H, dh, DEV, seed=dh * 2 + alibi)
        _, k, v = A.split_heads(seq, H)
        kc, vc = k.contiguous(), v.contiguous()
        qkv = torch.randn(N, 3 * H * dh, device=DEV).bfloat16()
        for slot, r0, n, p in runs:
            qkv[r0: r0 + n] = seq[slot, p: p + n]
        out = torch.full((N, H * dh), SENTINEL, dtype=torch.bfloat16, device=DEV)
        ops.cache_attention(qkv, kc, vc, tiles, out, H, scale, slopes)
        again = torch.full_like(out, SENTINEL)
        ops.cache_attention(qkv, kc, vc, tiles, again, H, scale, slopes)
        torch.cuda.synchronize()
        assert torch.equal(out, again), "two runs differ"
        covered = torch.zeros(N, dtype=torch.bool)
        got, refs, bases = [], [], []
        for slot, r0, n, p in tiles.tolist():
            covered[r0: r0 + n] = True
            q = qkv[r0: r0 + n, : H * dh].view(1, n, H, dh).transpose(1, 2)
            kw = dict(causal=True, slopes=None if slopes is None else slopes.tolist(), q_pos=(p + torch.arange(n, device=DEV))[None],
                      lengths=[p + n])
            ks, vs = kc[slot: slot + 1], vc[slot: slot + 1]
            refs.append(A.oracle(q, ks, vs, scale, **kw).o)
            bases.append(A.baseline(q, ks, vs, scale, **kw).o)
            got.append(out[r0: r0 + n].view(1, n, H, dh).transpose(1, 2))
        A.check_tiles("cache o", got, refs, bases, case=f"{case}, runs {RUNS}")
        assert bool((out[~covered.to(DEV)] == SENTINEL).all()), "a row outside the tiles was written"


@pytest.mark.parametrize("use_rope", [False, True])
def test_slotted_decode_append_matches_torch(use_rope):
    from photon_b200 import ops
    from photon_b200.models.mpt import rope_tables

    H, dh, S, Bm, N = 4, 64, 256, 3, 7
    d = H * dh
    g = torch.Generator(device=DEV).manual_seed(11 + use_rope)
    kc = torch.randn(Bm, H, S, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(Bm, H, S, dh, device=DEV, generator=g).bfloat16()
    qkv = torch.randn(N, 3 * d, device=DEV, generator=g).bfloat16()
    slot = torch.tensor([2, 2, 2, 0, 1, 1, 0], dtype=torch.int32, device=DEV)   # more rows than slots
    pos = torch.tensor([5, 6, 7, 0, 100, 255, 17], dtype=torch.int32, device=DEV)
    rope = tuple(t.contiguous() for t in rope_tables(S, dh, 10000.0, DEV)) if use_rope else None
    k_want, v_want, q_in = kc.clone(), vc.clone(), qkv.clone()
    ops.decode_append(qkv, pos, kc, vc, rope, H, slot=slot)
    torch.cuda.synchronize()
    x = q_in.float().view(N, 3, H, dh)
    q, k = x[:, 0], x[:, 1]
    if use_rope:
        c, s = rope[0][pos.long()][:, None], rope[1][pos.long()][:, None]

        def rot(t):
            t1, t2 = t[..., : dh // 2], t[..., dh // 2:]
            return torch.cat([t1 * c - t2 * s, t2 * c + t1 * s], -1)

        q, k = rot(q), rot(k)
    for r in range(N):
        k_want[slot[r], :, pos[r]] = k[r].bfloat16()
        v_want[slot[r], :, pos[r]] = q_in[r, 2 * d:].view(H, dh)
    torch.testing.assert_close(qkv[:, :d].float(), q.reshape(N, d), rtol=1e-2, atol=1e-2)
    assert torch.equal(qkv[:, d:], q_in[:, d:])
    torch.testing.assert_close(kc.float(), k_want.float(), rtol=1e-2, atol=1e-2)
    assert torch.equal(vc, v_want)
    untouched = torch.ones(Bm, S, dtype=torch.bool, device=DEV)
    untouched[slot.long(), pos.long()] = False
    assert torch.equal(kc.transpose(1, 2)[untouched], k_want.transpose(1, 2)[untouched])


# ------------------------------------------------------------------------------------------------ KVDecoder.score
def _pairs(cfg, seed=0):
    """A 4-choice question (scored lengths 1, 2, 17, 130 after one shared context), contexts of 1, 127, 128, 129 and 200 tokens,
    a pair truncated at max_seq_len as the evaluator truncates it, and schema-style pairs (contexts vary, one continuation)."""
    from photon_b200.eval.icl import ICLEvaluator

    g = torch.Generator().manual_seed(seed)
    rnd = lambda n: torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist()  # noqa: E731
    q = rnd(50)
    pairs = [(q, rnd(n)) for n in (1, 2, 17, 130)]
    pairs += [(rnd(n), rnd(3)) for n in (1, 127, 128, 129, 200)]
    ev = ICLEvaluator(None, None, cfg.max_seq_len)
    pairs.append(ev._truncate(rnd(250), rnd(10)))
    assert len(pairs[-1][0]) + len(pairs[-1][1]) == cfg.max_seq_len
    shared, cont = rnd(40), rnd(5)
    pairs += [(shared[:30], cont), (shared[:31], cont), (shared, cont)]
    return pairs


def _fp32_stats(ref, pairs):
    """(sum log p, all argmax, every top-2 margin > LOGP_TOL) of each pair under the fp32 model."""
    out = []
    for ctx, sc in pairs:
        ids = torch.tensor([ctx + sc], device=DEV)
        with torch.no_grad():
            lp = torch.log_softmax(ref.logits(ids)[0].float(), -1)[len(ctx) - 1: len(ctx) + len(sc) - 1]
        tgt = torch.tensor(sc, device=DEV)
        top2 = lp.topk(2, -1).values
        out.append((float(lp[torch.arange(len(sc)), tgt].sum()), bool((lp.argmax(-1) == tgt).all()),
                    bool(((top2[:, 0] - top2[:, 1]) > LOGP_TOL).all())))
    return out


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_score_matches_fp32_model(variant):
    cfg, ref, eng = _engine(variant)
    pairs = _pairs(cfg)
    dec = eng.decoder(len(pairs))
    got = dec.score(pairs)
    for i, ((lp, hit), (want_lp, want_hit, clear), (_, sc)) in enumerate(zip(got, _fp32_stats(ref, pairs), pairs)):
        assert abs(lp - want_lp) <= LOGP_TOL * len(sc), (variant, i, lp, want_lp)
        if clear:
            assert hit == want_hit, (variant, i)


def test_score_batch_equals_single_pairs_and_repeats_bitwise():
    cfg, _, eng = _engine()
    pairs = _pairs(cfg, seed=1)
    dec = eng.decoder(len(pairs))
    batch = dec.score(pairs)
    assert dec.score(pairs) == batch
    for (ctx, sc), (lp, _) in zip(pairs, batch):
        alone = dec.score([(ctx, sc)])[0][0]
        assert abs(alone - lp) <= LOGP_TOL * len(sc), (len(ctx), len(sc), alone, lp)
    for bad in ([([], [1])], [([1], [])], [([1] * 250, [2] * 7)], [([1], [2])] * (len(pairs) + 1)):
        with pytest.raises(ValueError):
            dec.score(bad)


def test_score_leaves_training_and_generation_untouched():
    cfg, _, eng = _engine()
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device=DEV)
    denom = float(ids.numel())
    eng.flat.zero_grad()
    eng.fwd_bwd(ids, denom)
    before = eng.flat.grads.clone()
    params, shadow = eng.flat.params.clone(), eng.bf16_params.clone()
    graphs, ws = dict(eng._graphs), dict(eng._ws)
    prompts = [torch.randint(0, cfg.vocab_size, (n,)).tolist() for n in (3, 50, 129, 200)]

    def generate(dec):
        out = [dec.start(prompts, 8)]
        out += [dec.step() for _ in range(7)]
        return out

    fresh = generate(eng.decoder(8))
    dec = eng.decoder(8)
    generate(dec)                      # captures the step graph of batch 4
    dec.score(_pairs(cfg)[:4])         # within the cache's capacity: the captured graph is kept and replayed
    assert generate(dec) == fresh      # the same decoder generates as before after scoring
    dec.score(_pairs(cfg)[4:12])       # grows the cache
    assert generate(dec) == fresh
    torch.cuda.synchronize()
    assert torch.equal(params, eng.flat.params) and torch.equal(shadow, eng.bf16_params)
    assert graphs.keys() == eng._graphs.keys() and all(graphs[k] is eng._graphs[k] for k in graphs)
    assert ws.keys() == eng._ws.keys() and all(ws[k] is eng._ws[k] for k in ws)
    eng.flat.zero_grad()
    eng.fwd_bwd(ids, denom)
    torch.cuda.synchronize()
    after = eng.flat.grads   # float-atomic noise only (see test_generation_leaves_training_untouched)
    assert ((after - before).norm() / before.norm()).item() < 1e-3
    assert torch.nn.functional.cosine_similarity(after, before, dim=0).item() > 0.99999


def test_trainer_eval_scoring_tasks_use_score(tmp_path):
    from photon_b200.dataset.utils import ByteTokenizer
    from photon_b200.eval.icl import run_icl_suite
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.trainer import Trainer

    mc = [{"query": "Q: 2+2", "choices": ["4", "5", "22", "four"], "gold": 0}, {"query": "sky", "choices": ["blue", "green"], "gold": 0},
          {"query": "x" * 30, "choices": ["y", "z", "yy"], "gold": 2}]
    lm = [{"context": "abc", "continuation": "def"}, {"context": "hello", "continuation": " world"}]
    schema = [{"context_options": ["The cat", "A dog"], "continuation": "ran", "gold": 1}]
    for name, rows in (("mc", mc), ("lm", lm), ("schema", schema)):
        (tmp_path / f"{name}.jsonl").write_text("\n".join(json.dumps(r) for r in rows))
    icl = {"icl_tasks_config": {"root_dir": str(tmp_path), "icl_tasks": [
        {"label": "mc", "dataset_uri": "mc.jsonl", "icl_task_type": "multiple_choice", "num_fewshot": [0, 1], "batch_size": 2},
        {"label": "lm", "dataset_uri": "lm.jsonl", "icl_task_type": "language_modeling", "batch_size": 4},
        {"label": "schema", "dataset_uri": "schema.jsonl", "icl_task_type": "schema", "batch_size": 4}]}}
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
    scored, logits_calls = [], []

    def suite(logits_fn, decoder=None):
        assert decoder is not None
        orig = decoder.score

        def spy(pairs):
            scored.append(len(pairs))
            return orig(pairs)

        decoder.score = spy
        return run_icl_suite(lambda x: logits_calls.append(x.shape) or logits_fn(x), ByteTokenizer(), icl, cfg.max_seq_len,
                             decoder=decoder)

    tr.icl_suite = suite
    vals = tr.eval()
    assert sum(scored) == 2 * (4 + 2 + 3) + 2 + 2 and not logits_calls   # every pair through score, none through logits
    assert scored[:3] == [6, 3, 6]   # two whole questions per call (batch_size 2), then one
    pairwise = run_icl_suite(tr.state.backend.logits, ByteTokenizer(), icl, cfg.max_seq_len)
    assert {k for k in vals if k.startswith("icl/")} == {f"icl/{k}" for k in pairwise}
    tr.close()
