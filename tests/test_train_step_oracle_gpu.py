"""Every optimizer step of ``Trainer`` on the sm_90a engine against an fp64 step (``step_oracle``) from the state it started in.

Model: the engine oracle's base (d_model 384, 6 heads, 3 layers, vocabulary 2008, FFN width 1352; 1360 under amp_fp8, whose E4M3
rows must be 16-byte multiples) at S = 256, global batch 4 in microbatches of 2, bf16-exact starting weights with nonzero
biases. Four steps through ``Trainer.fit``, one batch per call, on a warmup + cosine schedule (learning-rate factors 0, 1/2,
1, 3/4), with a clip that binds on every step unless the variant has none. An ``after_backward`` callback takes the state the
optimizer is about to step from: p_t, m_t, v_t, the bf16 shadow and the accumulated gradient. Per step t:

(a) the shadow equals ``bf16(p_t)`` bitwise;
(b) the gradient against ``model_oracle.oracle`` at the weights the engine computes with, ``bf16(p_t)`` for the matrices and
    ``p_t`` for biases and norm weights (read from the fp32 masters), per tensor with ``model_oracle.Checker``,
    bounded by the pure-bf16 model (amp_fp8: by the ``TorchBackend("amp_fp8")`` emulation at the same weights), at twice
    the whole-engine test's slack (``SLACK``). The key part of the QKV bias is left out: its exact gradient is zero and both sides are
    rounding noise there (``model_oracle.KNOWN``). For t >= 1 this is what sees a stale shadow, CUDA graph or E4M3 weight;
(c) the logged ``l2_norm/grad/clipped_from`` within ``step_oracle.NORM_REL`` of the fp64 norm of that gradient;
(d) p, m and v after the step against ``step_oracle.step`` from (p_t, m_t, v_t) with the engine's own gradient: the
    bounds of ``fused_oracle.optim_step``, widened by the reference's change when the clip coefficient moves by
    ``step_oracle.COEF_REL`` either way (the fp32 coefficient the trainer forms may differ that much from the fp64 one);
(e) the shadow after the step equals ``bf16(p_{t+1})`` bitwise; a frozen plane stays bitwise unchanged.

Matrix: ADOPT (decoupled and ``decouple: false``), DecoupledAdamW and SGD, all with weight decay 0.1; AdamW without a clip;
ADOPT under CUDA graphs, activation checkpointing, amp_fp8, the engine oracle's freeze list, ``kernels.optimizer: torch``
and ZeRO-3 at a world of one. ``test_ddp_zero_step_matches_fp64_step`` drives the fused ZeRO-1 kernel (reduce, norm, clip,
optimizer, broadcast in one launch) at a world of one. Plants: a reference with the previous step's learning rate, without
the clip, with AdamW's bias correction at t, with AdamW's decay scaled by lr instead of lr / lr_0, without ADOPT's coupled
decay, and the gradient oracle at the weights of step t - 1: each must be flagged, and the test prints by which check.

Runtime of this file on an NVIDIA H100 80GB HBM3: 27 s of tests, 32 s with pytest's start-up.
"""
import dataclasses

import pytest
import torch

import fused_oracle as fo
import model_oracle as MO
import step_oracle as SO
from photon_b200.train.callbacks import Callback
from test_engine_oracle_gpu import BASE, FROZEN, _exact_bf16_reduction

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
B, MB, S, STEPS = 4, 2, 256, 4
MAX_NORM = 0.05
PLANT_STEP = 3
VARIANTS = {
    "adopt": dict(setup="adopt"),
    "adopt_coupled": dict(setup="adopt_coupled"),
    "decoupled_adamw": dict(setup="decoupled_adamw"),
    "sgd": dict(setup="sgd"),
    "decoupled_adamw_noclip": dict(setup="decoupled_adamw", clip=None),
    "adopt_cuda_graph": dict(setup="adopt", kernels={"cuda_graph": True}),
    "adopt_checkpointing": dict(setup="adopt", activation_checkpointing=True),
    "adopt_fp8": dict(setup="adopt", precision="amp_fp8"),
    "adopt_frozen": dict(setup="adopt", frozen_layers=FROZEN),
    "adopt_torch_optimizer": dict(setup="adopt", kernels={"optimizer": "torch"}),
    "adopt_zero3": dict(setup="adopt", zero3=True),
}
# Twice the whole-engine slack (``model_oracle.BF16`` / ``FP8``): after a few steps the weights have left the point that slack
# was measured at, and the attention backward's delta residual (``model_oracle.KNOWN``) reaches 1.1-1.2x of it on some
# attention tensors by step 3 (q part of the last block's QKV bias, whole; an out_proj weight under amp_fp8, scale; key rows of
# a Wqkv weight, block; H100). A stale shadow, graph or E4M3 weight is far outside either: see the gradient plant.
SLACK = dataclasses.replace(MO.BF16, whole=2 * MO.BF16.whole, scale=2 * MO.BF16.scale, block=2 * MO.BF16.block)
SLACK_FP8 = dataclasses.replace(MO.FP8, whole=2 * MO.FP8.whole, scale=2 * MO.FP8.scale)
PLANTED = {"adopt", "adopt_coupled", "decoupled_adamw"}   # where the plants of each optimizer are shown to be flagged


class _StepState(Callback):
    """``after_backward``: the state the optimizer is about to step from (in the optimizer's layout: a shard under ZeRO-3)."""

    def __init__(self):
        self.before = []

    def after_backward(self, tr):
        self.before.append(_state(tr))


@pytest.fixture
def step_state():
    return _StepState()


def _state(tr):
    st, be = tr.state, tr.state.backend
    torch.cuda.synchronize()
    return dict(p=st.flat.params.clone(), g=st.flat.grads.clone(), m=st.optimizer.exp_avg.clone(),
                v=st.optimizer.exp_avg_sq.clone(), shadow=be.bf16_params.clone(),
                frozen=None if be.frozen_params is None else (be.frozen_params.clone(), be.frozen_bf16.clone()))


def _cfg(precision):
    from photon_b200.models.mpt import MPTConfig

    return MPTConfig(**{**BASE, **({"ffn_hidden_size": 1360} if precision == "amp_fp8" else {})})


def _full(tr, x):
    """``x`` in the full flat layout (ZeRO-3: this rank's shard scattered into it; with one rank that is everything)."""
    comm = tr.grad_comm
    if not getattr(comm, "zero3", False):
        return x
    return comm.plan.shard_to_full(x, 0, torch.zeros(tr.state.flat.layout.total, dtype=x.dtype, device=x.device))


def _set_weights(tr, seed):
    """bf16-exact starting weights (``model_oracle.bf16_exact_weights``) in the masters, the shadow and the frozen plane."""
    be, flat = tr.state.backend, tr.state.flat
    lay, flay = flat.layout, be.frozen_layout
    full = flat.full_params().clone()
    named = {n: lay.view(full, n) for n in lay.names}
    if flay is not None:
        named.update({n: flay.view(be.frozen_params, n) for n in flay.names})
    w = MO.bf16_exact_weights(named, seed)
    for n in lay.names:
        lay.view(full, n).copy_(w[n])
    flat.load_full_params(full)
    if flay is not None:
        for n in flay.names:
            flay.view(be.frozen_params, n).copy_(w[n])
    be.params_updated()


def _weights(tr, state):
    """name -> the weights the engine computes with: the bf16 shadow for the matrices (the GEMMs and embeddings read it), the
    fp32 masters for the 1-D tensors (biases and norm weights are read in fp32), the frozen plane for frozen tensors."""
    be, lay, flay = tr.state.backend, tr.state.flat.layout, tr.state.backend.frozen_layout
    w16, w32 = _full(tr, state["shadow"]).float(), _full(tr, state["p"])
    w = {n: lay.view(w16 if len(shp) > 1 else w32, n) for n, shp in zip(lay.names, lay.shapes)}
    if flay is not None:
        w.update({n: flay.view(be.frozen_params, n) for n in flay.names})
    return w


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


def _grad_references(cfg, w, mbs, frozen, emu):
    """(fp64 oracle result, name -> bounding gradient): the bf16 model's, or under amp_fp8 the emulation's."""
    ref = MO.oracle(cfg, w, mbs, frozen, device=DEV)
    if emu is None:
        with _exact_bf16_reduction():
            return ref, MO.baseline(cfg, w, mbs, frozen, device=DEV).grads
    with torch.no_grad():
        for name, p in emu.model.named_parameters():
            p.copy_(w[name])
    emu.flat.zero_grad()
    with _exact_bf16_reduction():
        for mb in mbs:
            emu.fwd_bwd(mb.ids.to(DEV), mb.denom, mb.scale)
    return ref, {n: emu.flat.layout.view(emu.flat.grads, n).clone() for n in emu.flat.layout.names}


def _grad_tensors(cfg, lay, g):
    """(label, engine gradient slice, slice of a full tensor) of every checked gradient; without RoPE the QKV bias as its q and
    v parts (the key part's exact gradient is zero: rounding noise on both sides, see ``model_oracle.KNOWN``)."""
    out = []
    for name in lay.names:
        if name.endswith("attn.Wqkv.bias") and not cfg.rope:
            d, kvd = cfg.d_model, cfg.kv_dim
            out += [(f"{name}:q", name, slice(0, d)), (f"{name}:v", name, slice(d + kvd, d + 2 * kvd))]
        else:
            out.append((name, name, slice(None)))
    return [(label, lay.view(g, name)[sl], name, sl) for label, name, sl in out]


def _trainer(variant, cb):
    from photon_b200.parallel.zero3 import NvlZero3Comm
    from photon_b200.train.trainer import Trainer
    from photon_b200.utils.flat import layout_for_model_cfg

    v = VARIANTS[variant]
    precision = v.get("precision", "amp_bf16")
    cfg = _cfg(precision)
    comm = NvlZero3Comm(layout_for_model_cfg(cfg), cfg.n_layers, rank=0, world_size=1, device=DEV) if v.get("zero3") else None
    gen = torch.Generator().manual_seed(21)
    batches = [{"input_ids": torch.randint(0, cfg.vocab_size, (B, S), generator=gen)} for _ in range(STEPS)]
    tr = Trainer(cfg, optimizer_cfg=SO.SETUPS[v["setup"]], scheduler_cfg=SO.SCHEDULE, train_loader=batches,
                 global_train_batch_size=B, device_train_microbatch_size=MB, precision=precision, max_duration=f"{STEPS}ba",
                 grad_clip_norm=v.get("clip", MAX_NORM), device=DEV, kernels={"cuda_graph": False, **v.get("kernels", {})},
                 frozen_layers=v.get("frozen_layers"), activation_checkpointing=v.get("activation_checkpointing", False),
                 grad_comm=comm, callbacks=[cb], seed=23)
    assert tr.state.backend.kind == "b200"
    _set_weights(tr, seed=23)
    return tr, cfg, batches


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_train_steps_match_fp64_step(variant, step_state):
    from photon_b200.train.backend import TorchBackend

    v = VARIANTS[variant]
    opt_cfg = SO.SETUPS[v["setup"]]
    clip = v.get("clip", MAX_NORM)
    tr, cfg, batches = _trainer(variant, step_state)
    be, lay = tr.state.backend, tr.state.flat.layout
    frozen = v.get("frozen_layers") or ()
    emu = TorchBackend(cfg, DEV, "amp_fp8", seed=23) if v.get("precision") == "amp_fp8" else None
    chk = MO.Checker(variant, SLACK_FP8 if emu is not None else SLACK)
    frozen0 = _state(tr)["frozen"]
    n_tok = float(B * (S - 1))
    after, prev_w = [], None
    for t in range(STEPS):
        tr.fit("1ba")
        after.append(_state(tr))
        pre, post = step_state.before[t], after[t]
        tag = f"step {t}"
        # (a) the shadow the step's forward read
        chk.expect(torch.equal(_bits(pre["shadow"]), _bits(pre["p"].bfloat16())), f"{tag}: shadow != bf16(p_t) before the step")
        # (b) the engine's gradient at the weights it computed with
        w = _weights(tr, pre)
        ids = batches[t]["input_ids"]
        mbs = [MO.Batch(ids[i:i + MB], 1.0, n_tok) for i in range(0, B, MB)]
        ref, base = _grad_references(cfg, w, mbs, frozen, emu)
        g_full = _full(tr, pre["g"])
        for label, g, name, sl in _grad_tensors(cfg, lay, g_full):
            chk.tensor(f"{tag} {label}", g, ref.grads[name][sl], base[name][sl])
        # (c) the logged norm and the clip coefficient
        norm, coef = SO.clip(pre["g"], clip)
        if clip is not None:
            logged = tr.loggers[0].data["l2_norm/grad/clipped_from"][-1][1]
            print(f"[{variant}] {tag}: norm {logged:.9g} (fp64 {norm:.9g}), coefficient {coef:.4g}")
            chk.expect(abs(logged - norm) <= SO.NORM_REL * norm, f"{tag}: logged norm {logged!r}, fp64 {norm!r}")
            chk.expect(coef < 1.0, f"{tag}: the clip does not bind (coefficient {coef})")
        else:
            chk.expect("l2_norm/grad/clipped_from" not in tr.loggers[0].data, f"{tag}: a norm was logged without a clip")
        # (d) the update
        lr = opt_cfg["lr"] * SO.lr_factor(SO.SCHEDULE, t)
        P, M, V, tol = SO.step(opt_cfg, t, lr, pre["p"], pre["g"], pre["m"], pre["v"], coef)
        for k, got, want in (("p", post["p"], P), ("m", post["m"], M), ("v", post["v"], V)):
            bad, msg = fo.worst(got, want, tol[k])
            chk.expect(bad == 0, f"{tag}: {k} after the step: {bad} elements out of bounds; {msg}")
        # (e) the shadow the next step reads, the frozen plane
        chk.expect(torch.equal(_bits(post["shadow"]), _bits(post["p"].bfloat16())), f"{tag}: shadow != bf16(p_t+1) after the step")
        if frozen0 is not None:
            chk.expect(all(torch.equal(_bits(a), _bits(b)) for a, b in zip(post["frozen"], frozen0)), f"{tag}: frozen plane changed")
        if t == PLANT_STEP and variant in PLANTED:
            _plants_flagged(variant, opt_cfg, t, pre, post, coef, cfg, lay, prev_w, mbs, frozen, g_full, chk.slack)
        prev_w = w
    if v.get("kernels", {}).get("cuda_graph"):
        assert be.use_graph and len(be._graphs) == 1   # captured at step 0, replayed since  # noqa: SLF001
    tr.close()
    if tr.grad_comm is not None:
        tr.grad_comm.close()
    chk.finish()


def _plants_flagged(variant, opt_cfg, t, pre, post, coef, cfg, lay, prev_w, mbs, frozen, g_full, slack):
    """Each planted mistake, checked as the test checks the real thing, must fail; prints which check caught it."""
    lr = lambda s: opt_cfg["lr"] * SO.lr_factor(SO.SCHEDULE, s)  # noqa: E731
    args = (pre["p"], pre["g"], pre["m"], pre["v"])
    planted = {"reference with the lr of step t-1": SO.step(opt_cfg, t, lr(t - 1), *args, coef),
               "reference without the clip": SO.step(opt_cfg, t, lr(t), *args, 1.0)}
    for p in SO.plants_for(opt_cfg):
        planted[f"reference with {p}"] = SO.step(opt_cfg, t, lr(t), *args, coef, plant=p)
    missed = []
    for label, (P, M, V, tol) in planted.items():
        caught = [k for k, got, want in (("p", post["p"], P), ("m", post["m"], M), ("v", post["v"], V))
                  if fo.worst(got, want, tol[k])[0]]
        print(f"[{variant}] plant {label}: flagged by the {caught} update checks")
        if not caught:
            missed.append(label)
    if variant == "adopt":
        ref, base = _grad_references(cfg, prev_w, mbs, frozen, None)
        caught = []
        for label, g, name, sl in _grad_tensors(cfg, lay, g_full):
            parts = MO.failed_parts(MO.tensor_report(label, g, ref.grads[name][sl], base[name][sl], slack), slack)
            if parts:
                caught.append(f"{label} ({', '.join(parts)})")
        print(f"[{variant}] plant gradient oracle at the weights of step t-1: flagged by {len(caught)} tensors: {caught[:6]}")
        if not caught:
            missed.append("gradient oracle at the weights of step t-1")
    assert not missed, f"plants not flagged: {missed}"


# ------------------------------------------------------------------------------------------------ fused ZeRO-1 step
@pytest.mark.parametrize("setup", ["adopt", "decoupled_adamw", "sgd"])
def test_ddp_zero_step_matches_fp64_step(setup):
    """``NvlZeroComm.step`` (one ``ddp_zero_step`` launch: reduce with the 1 / loss-scale folded in, norm, clip coefficient,
    optimizer, broadcast of masters and shadow) at a world of one, four steps with ``inv_scale`` 0.5 and a binding clip:
    the returned norm, p, m, v and the shadow bits against ``step_oracle`` with the gradient halved."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.ddp import NvlZeroComm
    from photon_b200.train.optim import build_optimizer
    from photon_b200.utils.flat import layout_for_model_cfg

    cfg = _cfg("amp_bf16")
    opt_cfg = SO.SETUPS[setup]
    comm = NvlZeroComm(layout_for_model_cfg(cfg).total, rank=0, world_size=1, device=DEV)
    eng = B200Engine(cfg, DEV, "amp_bf16", {"cuda_graph": False}, seed=29, params_storage=comm.params, grads_storage=comm.grads,
                     shadow_storage=comm.shadow)
    opt = build_optimizer(opt_cfg, eng.flat, use_kernel=True, bf16_shadow=eng.bf16_params, shard=comm.shard(),
                          shard_bounds=comm.shard_bounds())
    gen = torch.Generator().manual_seed(31)
    fails = []
    for t in range(STEPS):
        ids = torch.randint(0, cfg.vocab_size, (B, S), generator=gen).to(DEV)
        eng.flat.zero_grad()
        for i in range(0, B, MB):
            eng.fwd_bwd(ids[i:i + MB], float(B * (S - 1)))
        torch.cuda.synchronize()
        p, g, m, v = (x.clone() for x in (eng.flat.params, eng.flat.grads, opt.exp_avg, opt.exp_avg_sq))
        lr = opt_cfg["lr"] * SO.lr_factor(SO.SCHEDULE, t)
        got_norm = float(comm.step(opt, lr, MAX_NORM, 0.5))
        g = g.double() * 0.5
        norm, coef = SO.clip(g, MAX_NORM)
        print(f"[ddp_zero_step {setup}] step {t}: norm {got_norm:.9g} (fp64 {norm:.9g}), coefficient {coef:.4g}")
        if not (abs(got_norm - norm) <= SO.NORM_REL * norm and coef < 1.0):
            fails.append(f"step {t}: norm {got_norm!r} vs fp64 {norm!r}, coefficient {coef}")
        P, M, V, tol = SO.step(opt_cfg, t, lr, p, g, m, v, coef)
        for k, got, want in (("p", eng.flat.params, P), ("m", opt.exp_avg, M), ("v", opt.exp_avg_sq, V)):
            bad, msg = fo.worst(got, want, tol[k])
            if bad:
                fails.append(f"step {t}: {k}: {bad} elements out of bounds; {msg}")
        if not torch.equal(_bits(eng.bf16_params), _bits(eng.flat.params.bfloat16())):
            fails.append(f"step {t}: shadow != bf16(p)")
    comm.close()
    assert not fails, "\n".join(fails)
