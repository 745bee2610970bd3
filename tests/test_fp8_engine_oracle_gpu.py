"""The amp_fp8 engine call by call against fp64 on its own E4M3 / E5M2 operands (``fp8_oracle``), and its delayed scaling
against the recipe of ``photon_b200.train.fp8``.

A recorder wraps the engine's fp8 ops on ``photon_b200.ops`` (``gemm_fp8``, the quantising producers, ``transpose_u8`` and
``fp8_update_scales``). Each call's inputs and the scales it reads are cloned before it runs and its outputs after, on the
engine's stream, and checked at once:

* every GEMM output against the fp64 product of the bytes it read, de-scaled by the scales those bytes were quantised with;
* every operand against the producer write it came from (role, scale, bytes);
* producer bytes bitwise against ``bf16 · scale`` cast with saturation (norms: within one step at rounding boundaries), and
  the amax each records;
* after every training prologue, the delayed scales bitwise against :class:`fp8_oracle.Recipe` fed the engine's own amaxes.

Shapes: the engine of ``test_engine_oracle_gpu.py`` (d_model 384, 3 layers, T = 768, FFN 1360, LM-head chunk 320), and one
step of two mpt-125m-wide layers at B·S = 16384 for the split-K weight gradients over long K.
"""
import re

import pytest
import torch

import fp8_oracle as FO
import model_oracle as MO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BASE = dict(d_model=384, n_heads=6, n_layers=3, max_seq_len=384, vocab_size=2008, ffn_hidden_size=1360)
ROPE = dict(rope=True, learned_pos_emb=False)
B, S, CHUNK = 3, 256, 320
WORST: dict = {}          # check -> (worst ratio, where)
EXCESS: dict = {}         # K -> largest accumulation error seen, in 2^-24 · Σ|a·b|


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("\nworst ratio to the bound: " + "; ".join(f"{k} {r:.3g} ({w})" for k, (r, w) in sorted(WORST.items())))
    print("accumulation error / (2^-24 · Σ|a·b|) by K, epilogue: " +
          ", ".join(f"K={k} epi {e}: {v:.3g} ({v / k:.3g} K, {w})" for (k, e), (v, w) in sorted(EXCESS.items())))


def _note(what, ratio):
    kind = re.sub(r"gemm\[\d+,\d+\]|role \d+|\(\d+, \d+\)", "", what).strip()
    if ratio > WORST.get(kind, (-1.0, ""))[0]:
        WORST[kind] = (ratio, what)


class Recorder:
    """Wraps the fp8 ops, checks every call as it happens and keeps the failures (``errors``), the scale updates and, with
    ``keep``, the GEMM calls (for the plants)."""

    def __init__(self, eng, monkeypatch, keep=False):
        from photon_b200 import ops

        self.eng, self.keep, self.active = eng, keep, True
        self.prod = FO.Producers()
        self.errors: list[str] = []
        self.gemms: list[FO.GemmCall] = []
        self.norm_calls: list[tuple] = []        # (bytes, y · scale, bound) of the norm producers, with keep
        self.wiring: list[tuple] = []            # (what, role, meta column, source), with keep
        self.updates: list[tuple] = []           # (training amax fed to the recipe, scales after)
        self.f32: list[tuple] = []               # (pass, prev was zero, output view, output after)
        self.saturated = self.nonfinite = self.n_gemm = 0
        self.pass_id, self.pass_open, self.train_amax = -1, False, None
        self.forward_bytes: dict = {}            # (pass, producer, role) -> bytes: a recompute must write them again
        self.n = eng._n_dyn
        for name in ("gemm_fp8", "colsum_quant", "layernorm_fwd_q8", "rmsnorm_fwd_q8", "fp8_quantize_segments", "transpose_u8",
                     "fp8_update_scales"):
            real = getattr(ops, name)
            monkeypatch.setattr(ops, name, self._wrap(name, real))

    def _wrap(self, name, real):
        mine = getattr(self, "_" + name)

        def call(*a, **k):
            if not self.active:
                return real(*a, **k)
            return mine(real, *a, **k)
        return call

    def _fail(self, msg):
        self.errors.append(msg)

    def _reports(self, reps):
        for r in reps:
            _note(r.what, r.worst)
            if not r.ok:
                self._fail(f"{r.what}: {r.bad_tiles} tile(s) over the bound, worst {r.worst:.3g} at tile {r.where}")

    def _produced(self, t, producer, role, scale, data):
        key = (self.pass_id, producer, role)
        if key in self.forward_bytes and not torch.equal(self.forward_bytes[key], data):
            self._fail(f"{producer} role {role}: the recompute wrote other bytes than the forward")
        self.forward_bytes.setdefault(key, data)
        self.prod.wrote(t, producer, role, scale, data)

    def _amax(self, what, before, after, call_amax):
        """The running amax after a call is max(before, the call's amax), exactly."""
        want = max(before, call_amax)
        if after != want:
            self._fail(f"{what}: amax {after!r} recorded, max(before {before!r}, max|x| {call_amax!r}) = {want!r}")

    def _bytes_stats(self, y8, fmt):
        self.saturated += int(FO.saturated(y8, fmt).sum())
        self.nonfinite += int(FO.nonfinite(y8, fmt).sum())

    # ------------------------------------------------------------------------------------------ the ops
    def _gemm_fp8(self, real, a, b, out, meta, role_a, role_b, *, a_mn=False, b_mn=False, epi=0, a_fmt=0, b_fmt=0, bias=None,
                  aux=None, out2=None, accumulate=False, alpha=1.0, cluster=0, out8=None, role_out=-1):
        m = meta.clone()
        ac, bc = a.clone(), b.clone()
        prev = out.clone() if epi == FO.EPI_F32 and accumulate else None
        auxc, biasc = (aux.clone() if aux is not None else None), (bias.clone() if bias is not None else None)
        real(a, b, out, meta, role_a, role_b, a_mn=a_mn, b_mn=b_mn, epi=epi, a_fmt=a_fmt, b_fmt=b_fmt, bias=bias, aux=aux, out2=out2,
             accumulate=accumulate, alpha=alpha, cluster=cluster, out8=out8, role_out=role_out)
        name = f"gemm[{role_a},{role_b}] epi {epi} {tuple(out.shape)}"
        scales = []
        for what, t, c, role in (("A", a, ac, role_a), ("B", b, bc, role_b)):
            src = self.prod.source(t)
            errs = FO.wiring_errors(f"{name} {what}", role, m[:, role], src)
            if src is not None and not torch.equal(src[3].view(-1), c.view(-1)):
                errs.append(f"{name} {what}: the operand's bytes are not the ones its producer wrote")
            self.errors += errs
            if self.keep:
                self.wiring.append((f"{name} {what}", role, m[:, role].cpu(), src))
            scales.append(src[2] if src is not None else float(m[0, role]))
        A = ac.t().contiguous() if a_mn else ac
        Bm = bc.t().contiguous() if b_mn else bc
        call = FO.GemmCall(A, Bm, a_fmt, b_fmt, scales[0], scales[1], epi, None if epi == FO.EPI_GELU_GRAD_Q8 else out.clone(),
                           alpha, biasc, auxc, prev, out2.clone() if out2 is not None else None,
                           out8.clone() if out8 is not None else None, name=name)
        if out8 is not None:
            call.q8_scale = float(m[0, role_out])
            call.amax_before, call.amax_after = float(m[2, role_out]), float(meta[2, role_out])
            self._bytes_stats(call.out8, FO.E4M3)
            self._produced(out8, "gemm_fp8 gelu", role_out, call.q8_scale, call.out8)
        self._reports(FO.gemm_check(call))
        if epi != FO.EPI_GELU_GRAD_Q8:
            K = A.shape[1]
            ex = FO.accumulation_excess(call)
            if ex > EXCESS.get((K, epi), (0.0, ""))[0]:
                EXCESS[(K, epi)] = (ex, name)
        if epi == FO.EPI_F32:
            self.f32.append((self.pass_id, prev is None or not bool(prev.any()), out, call.out))
        self.n_gemm += 1
        if self.keep:
            self.gemms.append(call)

    def _colsum_quant(self, real, dy, out_sum, y8, fmt=1, meta=None, role=-1):
        dyc = dy.clone()
        prev = out_sum.clone() if out_sum is not None else None
        m = meta[:, role].clone() if y8 is not None else None
        real(dy, out_sum, y8, fmt, meta, role)
        if out_sum is not None:
            ref, err = FO.colsum_bound(dyc, prev)
            self._reports([FO.tile_report(f"colsum[{role}] column sums", (out_sum.double() - ref).abs(), err)])
            self.f32.append((self.pass_id, not bool(prev.any()), out_sum, out_sum.clone()))
        if y8 is not None:
            got, s = y8.clone(), float(m[0])
            want = FO.quantize(dyc, s, fmt)
            if not torch.equal(got, want):
                self._fail(f"colsum_quant role {role}: {int((got != want).sum())} bytes differ from the saturating cast")
            self._amax(f"colsum_quant role {role}", float(m[2]), float(meta[2, role]), float(dyc.float().abs().max()))
            self._bytes_stats(got, fmt)
            self._produced(y8, "colsum_quant", role, s, got)

    def _norm(self, real, args, x, gamma, beta, y8, rstd, eps, meta, role, rms):
        xc, m = x.clone(), meta[:, role].clone()
        real(*args)
        s = float(m[0])
        y, err, rs = FO.norm_reference(xc, gamma, beta, eps, rms)
        got = y8.clone()
        ys, es = y * s, err * s + 2 * FO.EPS32 * (y * s).abs()
        bad = FO.byte_errors(got.view_as(y), ys, es, FO.E4M3)
        what = f"{'rmsnorm' if rms else 'layernorm'}_fwd_q8 role {role}"
        self._reports([FO.tile_report(f"{what} E4M3", bad.double(), torch.full_like(ys, 0.5)),
                       FO.tile_report(f"{what} rstd", (rstd.double() - rs).abs(), 2.0 ** -19 * rs)])
        am, am_err = float(y.abs().max()), float(err.max())
        before, after = float(m[2]), float(meta[2, role])
        miss = abs(after - am) / am_err if after > before else max(0.0, am - before) / am_err
        self._reports([FO.Report(f"{what} amax", miss, (0, 0), int(miss > 1))])
        self._bytes_stats(got, FO.E4M3)
        if self.keep:
            self.norm_calls.append((got.view_as(y), ys, es))
        self._produced(y8, "norm", role, s, got)

    def _layernorm_fwd_q8(self, real, x, gamma, beta, y8, mean, rstd, eps, meta, role):
        self._norm(real, (x, gamma, beta, y8, mean, rstd, eps, meta, role), x, gamma, beta, y8, rstd, eps, meta, role, False)

    def _rmsnorm_fwd_q8(self, real, x, gamma, y8, rstd, eps, meta, role):
        self._norm(real, (x, gamma, y8, rstd, eps, meta, role), x, gamma, None, y8, rstd, eps, meta, role, True)

    def _fp8_quantize_segments(self, real, src, dst8, seg, meta, role0):
        srcc = src.clone()
        real(src, dst8, seg, meta, role0)
        for i, (off, n) in enumerate(seg.tolist()):
            r = role0 + i
            w = srcc[off:off + n]
            amax = w.float().abs().max()
            s = torch.tensor(448.0, dtype=torch.float32, device=DEV) / amax
            got = meta[:, r]
            if not (torch.equal(got[0], s) and torch.equal(got[1], 1 / s) and torch.equal(got[2], amax)):
                self._fail(f"weight role {r}: (scale, 1/scale, amax) {got.tolist()} != 448/amax of the shadow "
                           f"({float(s)!r}, {float(1 / s)!r}, {float(amax)!r})")
            q = dst8[off:off + n]
            if not torch.equal(q, FO.quantize(w, float(s), FO.E4M3)):
                self._fail(f"weight role {r}: E4M3 bytes differ from the saturating cast of the shadow")
            self.prod.wrote(q, "fp8_quantize_segments", r, float(s), q.clone())

    def _transpose_u8(self, real, src, dst):
        real(src, dst)
        if not torch.equal(dst, src.t()):
            self._fail(f"transpose_u8 {tuple(src.shape)}: not src.t()")
        s = self.prod.source(src)
        if s is None:
            self._fail("transpose_u8: its source has no producer")
        else:
            self.prod.wrote(dst, "transpose_u8 of " + s[0], s[1], s[2], dst.clone())

    def _fp8_update_scales(self, real, meta, hist, fmax, pos, n, margin_mult=1.0):
        before = meta[2, :n].clone()
        if self.pass_open:          # the calibration pass ends at the real pass's prologue
            self.train_amax = before
        fed = self.train_amax if self.train_amax is not None else torch.zeros_like(before)
        real(meta, hist, fmax, pos, n, margin_mult)
        if bool(meta[2, :n].any()):
            self._fail("fp8_update_scales left an amax unreset")
        self.updates.append((fed.cpu(), meta[:2, :n].cpu()))
        self.pass_id += 1
        self.pass_open = True

    # ------------------------------------------------------------------------------------------ the engine
    def fwd_bwd(self, mb, **kw):
        sid = None if mb.sequence_id is None else mb.sequence_id.to(DEV)
        out = self.eng.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale, sid, **kw)
        torch.cuda.synchronize()
        self.train_amax, self.pass_open = self.eng.fp8_meta[2, :self.n].clone(), False
        return out

    def eval_stats(self, ids):
        self.pass_id += 1           # its forward writes other bytes than the training pass before it
        out = self.eng.eval_stats(ids)
        torch.cuda.synchronize()
        return out

    def assert_clean(self):
        kinds: dict = {}   # failures grouped by what failed (roles, shapes and numbers stripped): count, first example
        for e in self.errors:
            k = re.sub(r"gemm\[\d+,\d+\]|role \d+|\(\d+, \d+\)|[-+]?\d[\d.e+-]*", "#", e)
            n, first = kinds.get(k, (0, e))
            kinds[k] = (n + 1, first)
        assert not self.errors, f"{len(self.errors)} failure(s):\n" + "\n".join(f"{n}x {first}" for n, first in kinds.values())


def _cfg(**over):
    from photon_b200.models.mpt import MPTConfig

    return MPTConfig(**{**BASE, **over})


def _engine(cfg, seed=21, kernels=None, **kw):
    from photon_b200.models.engine import B200Engine

    eng = B200Engine(cfg, DEV, "amp_fp8", {"cuda_graph": False, **(kernels or {})}, seed=seed, lm_head_chunk=CHUNK, **kw)
    w = MO.bf16_exact_weights(eng.model.named_parameters(), seed)
    with torch.no_grad():
        for n, p in eng.model.named_parameters():
            p.copy_(w[n])
    eng.params_updated()
    return eng


def _batches(cfg, n, seed, b=B, s=S, scales=None):
    g = torch.Generator().manual_seed(seed)
    return [MO.Batch(torch.randint(0, cfg.vocab_size, (b, s), generator=g), (scales or {}).get(i, 1.0), 2.0 * b * (s - 1))
            for i in range(n)]


def _check_recipe(rec, history_len=16, margin=0):
    recipe = FO.Recipe(FO.role_formats(rec.eng.cfg.n_layers), history_len, margin)
    scales = []
    for k, (fed, after) in enumerate(rec.updates):
        want = recipe.observe(fed)
        bad = FO.scale_mismatches(after, want)
        assert not bad, (f"prologue {k}: roles {bad[:8]} differ from the recipe: engine {after[:, bad[:4]].tolist()}, "
                         f"recipe {want[:, bad[:4]].tolist()}")
        scales.append(after[0])
    return scales


# ------------------------------------------------------------------------------------------------ variants
FROZEN = ["transformer.blocks.0.attn.Wqkv.weight", "transformer.blocks.1.ffn.up_proj.weight", "transformer.blocks.1.ffn.down_proj.weight",
          "transformer.blocks.2.attn.out_proj.weight", "transformer.blocks.1.ffn.up_proj.bias"]
VARIANTS = {
    "default": (dict(), {}),
    "no_bias": (dict(no_bias=True), {}),
    "rmsnorm_rope_gqa_untied": (dict(norm_type="rmsnorm", kv_n_heads=2, tie_word_embeddings=False, **ROPE), {}),
    "frozen": (dict(), dict(frozen_layers=FROZEN)),
    "checkpointing": (dict(), dict(activation_checkpointing=True)),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_fp8_calls_match_fp64(variant, monkeypatch):
    """Two microbatches (the first with its calibration pass) and one evaluation: every fp8 call checked."""
    over, kw = VARIANTS[variant]
    cfg = _cfg(**over)
    eng = _engine(cfg, **kw)
    rec = Recorder(eng, monkeypatch)
    if variant == "frozen":
        eng.params_updated()       # the frozen E4M3 plane and its K-major copies, quantised under the recorder
    eng.flat.zero_grad()
    for mb in _batches(cfg, 2, seed=3, scales={1: 0.6}):
        rec.fwd_bwd(mb)
    rec.eval_stats(_batches(cfg, 1, seed=4)[0].ids.to(DEV))
    rec.assert_clean()
    assert rec.nonfinite == 0
    # per pass and block: 4 forward GEMMs and, for every trainable weight, its wgrad, and the dgrads down to the lowest one
    assert rec.n_gemm >= 3 * 4 * cfg.n_layers + 4
    _check_recipe(rec)


def test_fp8_calls_match_fp64_at_training_token_count(monkeypatch):
    """One microbatch of B·S = 16384 tokens at mpt-125m widths, two layers: the weight gradients split K = 16384 across CTAs."""
    cfg = _cfg(d_model=768, n_heads=12, n_layers=2, max_seq_len=2048, vocab_size=50368, ffn_hidden_size=3072)
    from photon_b200.models.engine import B200Engine

    eng = B200Engine(cfg, DEV, "amp_fp8", {"cuda_graph": False}, seed=5)
    rec = Recorder(eng, monkeypatch)
    eng.flat.zero_grad()
    rec.fwd_bwd(_batches(cfg, 1, seed=6, b=8, s=2048)[0])
    rec.assert_clean()
    _check_recipe(rec)
    assert (16384, FO.EPI_F32) in EXCESS


def test_calibration_leaves_one_pass_of_gradients(monkeypatch):
    """The first fwd_bwd runs a discarded calibration pass: the real pass accumulates into zeroed gradients, the gradients it
    leaves are exactly the real pass's, and the calibration amaxes seed the history (the recipe check)."""
    cfg = _cfg()
    eng = _engine(cfg)
    rec = Recorder(eng, monkeypatch)
    eng.flat.zero_grad()
    rec.fwd_bwd(_batches(cfg, 1, seed=7)[0])
    rec.assert_clean()
    assert len(rec.updates) == 2 and bool(rec.updates[1][0].gt(0).all()), "the calibration pass must record every role's amax"
    real = [f for f in rec.f32 if f[0] == 1]
    assert real and all(zero for _, zero, _, _ in real), "the real pass must accumulate into zeroed gradients"
    for _, _, view, after in real:
        assert torch.equal(view, after), "a gradient changed after the real pass wrote it"
    _check_recipe(rec)


def _run_schedule(rec, batches, evals, spike_at):
    cfg = rec.eng.cfg
    ev = _batches(cfg, 1, seed=99)[0].ids.to(DEV)
    states, metas = {}, []
    rec.eng.flat.zero_grad()
    for k, mb in enumerate(batches):
        sat0 = rec.saturated
        rec.fwd_bwd(mb)
        metas.append(rec.eng.fp8_meta[:2].clone())
        if k == spike_at:
            assert rec.saturated > sat0, "a 50x gradient spike against delayed scales must saturate"
        if k in evals:
            rec.eval_stats(ev)
            rec.eng.logits(ev[:1, :64])
            torch.cuda.synchronize()
        states[k] = rec.eng.fp8_state_dict()
    return states, metas


@pytest.mark.parametrize("history_len,margin,n_mb", [(16, 0, 21), (4, 1, 9)])
def test_delayed_scaling_follows_recipe(history_len, margin, n_mb, monkeypatch):
    """``n_mb`` microbatches with a 50x gradient spike, evaluations in between and a resume mid-history: after every prologue
    the engine's delayed scales are the recipe's, bitwise. The spike holds the gradient scales for exactly ``history_len``
    prologues. Evaluation casts with the training scales and leaves the scaling state alone, so an engine resumed from a
    checkpoint and run without evaluations continues the same scale sequence bitwise."""
    cfg = _cfg()
    kernels = {"fp8_amax_history_len": history_len, "fp8_margin": margin}
    eng = _engine(cfg, kernels=kernels)
    rec = Recorder(eng, monkeypatch)
    spike = 3
    batches = _batches(cfg, n_mb, seed=11, scales={spike: 50.0})
    states, metas = _run_schedule(rec, batches, evals={1, spike, spike + 2, n_mb - 3}, spike_at=spike)
    rec.assert_clean()
    assert rec.nonfinite == 0
    scales = _check_recipe(rec, history_len, margin)
    # prologue j + 1 (the first fwd_bwd has two) is the one of microbatch j; the spike's amax enters at microbatch spike + 1
    grad_roles = [r for r, f in enumerate(FO.role_formats(cfg.n_layers)) if f == FO.E5M2]
    first = spike + 2
    held = torch.stack(scales[first:first + history_len])[:, grad_roles]
    assert torch.equal(held, held[:1].expand_as(held)), "the spike must set every gradient scale for history_len prologues"
    if first + history_len < len(scales):
        after = scales[first + history_len][grad_roles]
        assert bool((after > held[0]).all()), "the spike must leave the history after exactly history_len prologues"

    # resume: a fresh engine loads the state of microbatch `cut` and runs the rest without evaluations
    rec.active = False
    cut = spike + 1
    eng2 = _engine(cfg, kernels=kernels)
    eng2.load_fp8_state_dict(states[cut])
    eng2.flat.zero_grad()
    for k in range(cut + 1, n_mb):
        mb = batches[k]
        eng2.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale)
        assert torch.equal(eng2.fp8_meta[:2], metas[k]), f"the resumed scales differ at microbatch {k}"


def test_evaluation_leaves_training_scales(monkeypatch):
    """eval_stats / logits between training microbatches change no scale, history or amax the next prologue reads."""
    cfg = _cfg()
    eng = _engine(cfg)
    batches = _batches(cfg, 3, seed=13)
    eng.flat.zero_grad()
    for mb in batches[:2]:
        eng.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale)
    before = {k: v.clone() for k, v in eng.fp8_state_dict().items() if torch.is_tensor(v)}
    big = _batches(cfg, 1, seed=14)[0].ids.to(DEV)
    eng.eval_stats(big)
    eng.logits(big[:1, :64])
    after = eng.fp8_state_dict()
    n = eng._n_dyn
    assert torch.equal(after["hist"], before["hist"]) and torch.equal(after["pos"], before["pos"])
    assert torch.equal(after["meta"][:, :n], before["meta"][:, :n])


# ------------------------------------------------------------------------------------------------ plants
def test_plants_are_flagged(monkeypatch):
    """Errors planted in real captured calls: each must be flagged."""
    cfg = _cfg()
    eng = _engine(cfg)
    rec = Recorder(eng, monkeypatch, keep=True)
    eng.flat.zero_grad()
    for mb in _batches(cfg, 2, seed=17):
        rec.fwd_bwd(mb)
    rec.assert_clean()
    last = rec.gemms[::-1]     # the second microbatch's calls (the calibration pass casts with unit scales)
    fwd = next(c for c in last if c.epi == FO.EPI_RESIDUAL)
    wgrad = next(c for c in last if c.epi == FO.EPI_F32)
    dgrad = next(c for c in last if c.epi == FO.EPI_MUL)
    q8 = next(c for c in last if c.epi == FO.EPI_GELU_GRAD_Q8)
    flagged = lambda call: not all(r.ok for r in FO.gemm_check(call))  # noqa: E731
    for c in (fwd, wgrad, dgrad, q8):
        assert not flagged(c)
    for c in (fwd, dgrad):   # the weight gradients' bound (2^-6 of Σ|a·b|) is wider than 1 % of their largest elements
        assert flagged(FO.plant_tile_scale(c, 1.01)), f"{c.name}: tile x1.01"
    for c in (fwd, wgrad, dgrad):
        assert flagged(FO.plant_dropped_kblock(c, kb=1)), f"{c.name}: K block dropped"
    assert flagged(FO.plant_dropped_kblock(q8, kb=1)), "E4M3 epilogue: K block dropped"
    # an operand de-scaled with the neighbouring role's scale (the next role in the meta the GEMM read)
    what, role, col, src = next(w for w in reversed(rec.wiring) if w[0] == fwd.name + " A")
    assert not FO.wiring_errors(what, role, col, src)
    neighbour = eng.fp8_meta[:, role + 1].cpu()
    assert float(neighbour[0]) != fwd.sa
    assert FO.wiring_errors(what, role, neighbour, src), "neighbouring role's scale"
    assert flagged(FO.GemmCall(**{**fwd.__dict__, "sa": float(neighbour[0])})), "GEMM de-scaled with the neighbouring role's scale"
    # one E4M3 byte two steps off: in the GELU epilogue's output and in a norm's output
    z, _ = FO.accumulation_bound(q8)
    assert flagged(FO.GemmCall(**{**q8.__dict__, "out8": FO.plant_two_steps(q8.out8, z * FO.gelu_parts(z)[0])})), "E4M3 byte two steps off"
    got, ys, es = rec.norm_calls[-1]
    assert bool(FO.byte_errors(FO.plant_two_steps(got, ys), ys, es, FO.E4M3).any()), "norm E4M3 byte two steps off"
    # a recipe whose history is one entry short
    spike = [torch.full((eng._n_dyn,), 1.0 if k != 2 else 50.0) for k in range(20)]
    full, short = FO.Recipe(FO.role_formats(cfg.n_layers), 16), FO.Recipe(FO.role_formats(cfg.n_layers), 15)
    assert any(not torch.equal(full.observe(a), short.observe(a)) for a in spike), "history one entry short"
