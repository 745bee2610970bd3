"""The fp64 references of ``fused_oracle`` against independent derivations on the CPU: LayerNorm and cross-entropy against
float64 ``torch.autograd``, the optimizer transcription against the torch path of ``photon_b200.train.optim``."""
import math

import pytest
import torch
import torch.nn.functional as F

import fused_oracle as fo

F64 = torch.float64


def test_ulp_helpers():
    one = torch.tensor([1.0, 1.5, -3.0, 0.0])
    assert fo.bf16_ulp(one).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -133]
    assert fo.e4m3_ulp(one).tolist() == [0.125, 0.125, 0.25, 2.0 ** -9]
    assert fo.e5m2_ulp(one).tolist() == [0.25, 0.25, 0.5, 2.0 ** -16]
    assert fo.fp32_ulp(torch.tensor([1.0])).item() == 2.0 ** -23
    x = torch.tensor([1.0625, 1.1875, 500.0, -1000.0, 2.0 ** -10, 0.3])
    assert fo.fp8_round(x, "e4m3").tolist() == [1.0, 1.25, 448.0, -448.0, 0.0, 0.3125]   # ties to even; saturation; subnormal
    torch.testing.assert_close(fo.fp8_round(x.float(), "e4m3").float(),
                               x.float().clamp(-448, 448).to(torch.float8_e4m3fn).float(), rtol=0, atol=0)


@pytest.mark.parametrize("d", [64, 200, 1032])
def test_layernorm_reference_matches_autograd(d):
    torch.manual_seed(d)
    T = 9
    x = (torch.randn(T, d) * 0.5 + 30.0).bfloat16()
    g, b = torch.rand(d) + 0.5, torch.randn(d) * 0.1
    dy, dres = torch.randn(T, d).bfloat16(), torch.randn(T, d).bfloat16()
    y, mu, rs = fo.layernorm_fwd(x, g, b, 1e-5)
    xd = x.to(F64).requires_grad_(True)
    gd, bd = g.to(F64).requires_grad_(True), b.to(F64).requires_grad_(True)
    ref = F.layer_norm(xd, (d,), gd, bd, 1e-5)
    torch.testing.assert_close(y, ref.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mu, x.to(F64).mean(-1), rtol=1e-14, atol=0)
    torch.testing.assert_close(rs, 1.0 / torch.sqrt(x.to(F64).var(-1, unbiased=False) + 1e-5), rtol=1e-12, atol=0)
    ref.backward(dy.to(F64))
    dx, dgamma, dbeta, floor, ag, ab = fo.layernorm_bwd(dy, x, g, mu, rs, dres)
    torch.testing.assert_close(dx, xd.grad + dres.to(F64), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dgamma, gd.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dbeta, bd.grad, rtol=1e-10, atol=1e-10)
    assert (floor > 0).all() and (ag >= dgamma.abs() - 1e-9).all() and (ab >= dbeta.abs() - 1e-9).all()
    # the one-pass variance the large offset is there to catch is far outside the rstd bound
    xf = x.float()
    one_pass = torch.rsqrt((xf * xf).mean(-1) - xf.mean(-1) ** 2 + 1e-5).to(F64)
    assert ((one_pass / rs - 1).abs() > fo.ln_rstd_rel_tol(x, rs)).any()


@pytest.mark.parametrize("V,scale", [(16, 1.0), (2048, 30.0)])
def test_cross_entropy_reference_matches_autograd(V, scale):
    torch.manual_seed(V)
    R = 12
    logits = (torch.randn(R, V) * scale).bfloat16()
    logits[3] = 0.5                                  # constant row: every index ties, argmax is 0
    tgt = torch.randint(0, V, (R,))
    tgt[0], tgt[1], tgt[2], tgt[3] = -100, V, 0, V - 1
    uni = torch.log_softmax(torch.randn(V), -1)
    gs = 1.0 / 7.0
    out = fo.cross_entropy(logits, tgt, gs, uni)
    xd = logits.to(F64).requires_grad_(True)
    t = torch.where((tgt >= 0) & (tgt < V), tgt, torch.full_like(tgt, -100))
    loss = F.cross_entropy(xd, t, ignore_index=-100, reduction="none")
    (loss.sum() * gs).backward()
    torch.testing.assert_close(out["loss"], loss.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(out["lse"], torch.logsumexp(logits.to(F64), -1), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(out["dlogits"], xd.grad, rtol=1e-12, atol=1e-15)
    assert out["argmax"][3].item() == 0
    valid = t != -100
    assert out["stats"][1].item() == valid.sum().item()
    assert out["stats"][2].item() == ((logits.to(F64).argmax(-1) == t) & valid).sum().item()
    assert math.isclose(out["stats"][3].item(), -uni.to(F64)[t[valid]].sum().item(), rel_tol=1e-13)
    assert out["dlogits"][:2].abs().max().item() == 0.0


class _Flat:
    """The two planes of a FlatParams, which is all FlatOptimizer touches."""

    def __init__(self, n):
        self.params = torch.randn(n)
        self.grads = torch.zeros(n)


@pytest.mark.parametrize("name,kind,decouple", [("adopt", 0, True), ("decoupled_adamw", 1, True), ("sgd", 2, True), ("adopt", 0, False)],
                         ids=["adopt-0", "decoupled_adamw-1", "sgd-2", "adopt_coupled_decay-0"])
def test_optim_step_matches_torch_path(name, kind, decouple):
    """``optim_step`` (fp64, the kernel's line order) and the fp32 torch path of FlatOptimizer take the same steps; ADOPT also
    with ``decouple: false``, where the weight decay is added to the gradient."""
    from photon_b200 import ops
    from photon_b200.train.optim import build_optimizer

    torch.manual_seed(kind)
    n = 4100
    flat = _Flat(n)
    # betas exact in fp32: the kernel forms 1 - beta in fp32 from the rounded beta, the torch path in double, and with
    # beta2 = 0.99 those two differ by 8 fp32 ulps of 1 - beta2 before any arithmetic happens
    cfg = dict(name=name, lr=3e-2, betas=[0.875, 0.9921875], eps=1e-6, weight_decay=0.1)
    if name == "adopt":
        cfg.update(clip_exp=0.25, decouple=decouple)
    opt = build_optimizer(cfg, flat, use_kernel=False)
    for step in range(5):
        g = torch.randn(n) * (10.0 if step == 1 else 1.0)
        g[::5] = 0.0
        flat.grads.copy_(g)
        lr_factor = 0.9
        h = ops.optimizer_hyper(opt, opt.initial_lr * lr_factor)
        gm = 0.5
        p0, m0, v0 = flat.params.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
        P, M, V, tol = fo.optim_step(kind, p0, g, m0, v0, h, grad_mult=gm)
        opt.step(lr_factor, gm)
        fo.assert_within(flat.params, P, tol["p"], f"{name} step {step} p")
        if kind != 2:
            fo.assert_within(opt.exp_avg, M, tol["m"], f"{name} step {step} m")
            fo.assert_within(opt.exp_avg_sq, V, tol["v"], f"{name} step {step} v")
        if kind == 0 and step == 1:     # clip = 1 ** 0.25 and the 10x gradient pushes |g| / sqrt(v) past it: the clamp binds
            assert h["clip"] == 1.0 and (g.abs() * gm / v0.sqrt().clamp(min=1e-6) > 1.0).any()
