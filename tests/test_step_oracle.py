"""The fp64 step reference (``step_oracle``) against the optimizers' fp32 torch path and against ``fused_oracle``'s mirror of
the optimizer kernel fed with ``ops.optimizer_hyper``'s scalars, on the CPU: five steps of a warmup + cosine schedule with a
binding clip, for every optimizer setup the GPU step test trains with."""
import pytest
import torch

import fused_oracle as fo
import step_oracle as SO

N = 4100


class _Flat:
    """The two planes of a FlatParams, which is all FlatOptimizer touches."""

    def __init__(self, n):
        self.params = torch.randn(n) * 0.5
        self.grads = torch.zeros(n)


def _flagged(got, ref):
    """Names of the planes of ``got`` (p, m, v) outside ``ref``'s bounds."""
    P, M, V, tol = ref
    return [k for k, a, b in zip("pmv", got, (P, M, V)) if fo.worst(a, b, tol[k])[0]]


@pytest.mark.parametrize("setup", list(SO.SETUPS))
def test_step_reference_matches_torch_path_and_kernel_mirror(setup):
    from photon_b200 import ops
    from photon_b200.train.optim import build_optimizer, clip_coefficient
    from photon_b200.train.schedulers import build_scheduler

    cfg = SO.SETUPS[setup]
    kind = SO.KIND[cfg["name"]]
    torch.manual_seed(kind)
    flat = _Flat(N)
    opt = build_optimizer(cfg, flat, use_kernel=False)
    sched = build_scheduler(SO.SCHEDULE)
    max_norm = 1.0
    lrs = [cfg["lr"] * SO.lr_factor(SO.SCHEDULE, t) for t in range(5)]
    for t in range(5):
        assert abs(sched(t) - SO.lr_factor(SO.SCHEDULE, t)) <= 1e-15
        g = torch.randn(N) * 0.1 * (1 + t)
        g[::5] = 0.0
        flat.grads.copy_(g)
        norm, coef = SO.clip(g, max_norm)
        assert coef < 0.5
        coef32 = clip_coefficient(g.norm(), max_norm)          # what the trainer hands the optimizer
        p0, m0, v0 = flat.params.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
        ref = SO.step(cfg, t, lrs[t], p0, g, m0, v0, coef)
        P, M, V, tol = ref
        tag = f"{setup} step {t}"
        # the kernel's arithmetic (fused_oracle's transcription) with the scalars the kernel is given
        h = ops.optimizer_hyper(opt, opt.initial_lr * sched(t))
        Pk, Mk, Vk, _ = fo.optim_step(kind, p0, g, m0, v0, h, grad_mult=float(coef32))
        fo.assert_within(Pk, P, tol["p"], tag + " kernel mirror p")
        if kind != 2:
            fo.assert_within(Mk, M, tol["m"], tag + " kernel mirror m")
            fo.assert_within(Vk, V, tol["v"], tag + " kernel mirror v")
        opt.step(sched(t), coef32)
        got = (flat.params, opt.exp_avg, opt.exp_avg_sq)
        fo.assert_within(got[0], P, tol["p"], tag + " torch path p")
        if kind != 2:
            fo.assert_within(got[1], M, tol["m"], tag + " torch path m")
            fo.assert_within(got[2], V, tol["v"], tag + " torch path v")
        if t == 3:
            # the mistakes the step test must see, computed by the reference and held to its true bounds
            plants = {"lr of step t-1": SO.step(cfg, t, lrs[t - 1], p0, g, m0, v0, coef),
                      "clip not applied": SO.step(cfg, t, lrs[t], p0, g, m0, v0, 1.0)}
            for p in SO.plants_for(cfg):
                plants[p] = SO.step(cfg, t, lrs[t], p0, g, m0, v0, coef, plant=p)
            for label, (Pp, Mp, Vp, _) in plants.items():
                caught = _flagged((Pp, Mp, Vp), ref)
                print(f"{setup} plant {label}: flagged on {caught}")
                assert caught, f"{setup}: plant '{label}' is within the reference's bounds"
