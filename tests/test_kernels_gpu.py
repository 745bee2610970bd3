"""Numerics of every hand-written sm_90a kernel vs a plain PyTorch fp32 reference of the same op."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _rand(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device=_dev(), dtype=torch.float32) * scale).to(dtype)


def _close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = int((err > tol).sum().item())     # every element, no "fraction may be wrong" allowance
    assert bad == 0, f"{what}: {bad} of {err.numel()} elements out of tolerance, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 768), (384, 768, 3072), (1024, 2304, 768), (200, 328, 136)])
def test_gemm_kk_bias(M, N, K):
    from photon_b200 import ops

    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    bias = torch.randn(N, device=_dev())
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    ops.gemm(a, b, out, bias=bias)
    ref = a.float() @ b.float().t() + bias
    _close(out, ref, 2e-2, 2e-2, "gemm K/K + bias")


@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("layout", ["kk", "kmn", "mnmn"])
def test_gemm_cta_pair_matches_single_cta(cluster, layout):
    """cta_group::2 (CTA pair, 256-row UMMA) and cta_group::1 produce the same numbers for every operand layout,
    including odd tile counts (the pair's second CTA then runs out of range) and split-K accumulation."""
    from photon_b200 import ops

    M, N, K = 640, 520, 1088          # 5 M-tiles (odd), N tail, K tail
    if layout == "kk":
        a, b = _rand(M, K), _rand(N, K, scale=0.05)
        out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
        ops.gemm(a, b, out, cluster=cluster)
        _close(out, a.float() @ b.float().t(), 2e-2, 3e-2, f"K/K cluster={cluster}")
    elif layout == "kmn":
        a, b = _rand(M, K), _rand(K, N, scale=0.05)
        out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
        ops.gemm(a, b, out, b_mn=True, cluster=cluster)
        _close(out, a.float() @ b.float(), 2e-2, 3e-2, f"K/MN cluster={cluster}")
    else:
        a, b = _rand(K * 4, M), _rand(K * 4, N)     # long K -> split-K path
        out = torch.zeros(M, N, device=_dev(), dtype=torch.float32)
        ops.gemm(a, b, out, a_mn=True, b_mn=True, epi=ops.EPI_F32, accumulate=True, cluster=cluster)
        _close(out, a.float().t() @ b.float(), 1e-2, 0.2, f"MN/MN cluster={cluster}")


def test_gemm_residual_and_gelu_dual():
    from photon_b200 import ops

    M, N, K = 512, 768, 768
    a, b, r = _rand(M, K), _rand(N, K, scale=0.05), _rand(M, N)
    bias = torch.randn(N, device=_dev()) * 0.1
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    ops.linear_fwd(a, b, bias, out, residual=r)
    _close(out, a.float() @ b.float().t() + bias + r.float(), 2e-2, 2e-2, "residual epilogue")
    pre, act = torch.empty_like(out), torch.empty_like(out)
    ops.linear_gelu_fwd(a, b, bias, pre, act)
    z = a.float() @ b.float().t() + bias
    _close(pre, z, 2e-2, 2e-2, "gelu-dual pre")
    _close(act, F.gelu(z), 2e-2, 2e-2, "gelu-dual act")


def test_gemm_dgrad_mn_major_b():
    from photon_b200 import ops

    T, N, K = 512, 1024, 768  # dy [T,N], w [N,K] -> dx [T,K]
    dy, w = _rand(T, N), _rand(N, K, scale=0.05)
    dx = torch.empty(T, K, device=_dev(), dtype=torch.bfloat16)
    ops.linear_dgrad(dy, w, dx)
    _close(dx, dy.float() @ w.float(), 2e-2, 3e-2, "dgrad (B MN-major)")
    z = _rand(T, K)
    ops.linear_dgrad(dy, w, dx, gelu_pre=z)
    zf = z.float().requires_grad_(True)
    (F.gelu(zf)).sum().backward()
    _close(dx, (dy.float() @ w.float()) * zf.grad, 2e-2, 3e-2, "dgrad * gelu'")


def test_gemm_wgrad_mn_major_both_accumulate():
    from photon_b200 import ops

    T, N, K = 1024, 768, 512  # dy [T,N], x [T,K] -> dw [N,K]
    dy, x = _rand(T, N), _rand(T, K)
    dw = torch.zeros(N, K, device=_dev(), dtype=torch.float32)
    ops.linear_wgrad(dy, x, dw, accumulate=False)
    ref = dy.float().t() @ x.float()
    _close(dw, ref, 1e-2, 5e-2, "wgrad store")
    ops.linear_wgrad(dy, x, dw, accumulate=True)
    _close(dw, 2 * ref, 1e-2, 1e-1, "wgrad TMA reduce-add")


def test_gemm_lm_head_tail_tile():
    from photon_b200 import ops

    T, V, d = 256, 50368, 768
    h, wte = _rand(T, d), _rand(V, d, scale=0.02)
    logits = torch.empty(T, V, device=_dev(), dtype=torch.bfloat16)
    ops.gemm(h, wte, logits)
    _close(logits, h.float() @ wte.float().t(), 2e-2, 2e-2, "lm head (N tail)")


def test_layernorm_fwd_bwd():
    from photon_b200 import ops

    for T, d in [(512, 768), (96, 2048), (40, 4096)]:
        x, dy, dres = _rand(T, d), _rand(T, d), _rand(T, d)
        g = torch.rand(d, device=_dev()) + 0.5
        b = torch.randn(d, device=_dev()) * 0.1
        y = torch.empty_like(x)
        mean, rstd = torch.empty(T, device=_dev()), torch.empty(T, device=_dev())
        ops.layernorm_fwd(x, g, b, y, mean, rstd)
        xf = x.float().requires_grad_(True)
        gf, bf = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        ref = F.layer_norm(xf, (d,), gf, bf, 1e-5)
        _close(y, ref, 2e-2, 2e-2, f"ln fwd d={d}")
        ref.backward(dy.float())
        dx = torch.empty_like(x)
        dg, db = torch.zeros(d, device=_dev()), torch.zeros(d, device=_dev())
        ops.layernorm_bwd(dy, x, g, mean, rstd, dres, dx, dg, db)
        _close(dx, xf.grad + dres.float(), 2e-2, 3e-2, f"ln bwd dx d={d}")
        _close(dg, gf.grad, 2e-3, 2e-2, f"ln dgamma d={d}")     # fp32 column sums of the same bf16 inputs: only mean / rstd rounding differs
        _close(db, bf.grad, 2e-3, 2e-2, f"ln dbeta d={d}")


def test_cross_entropy_loss_and_grad():
    from photon_b200 import ops

    T, V = 300, 50368
    logits = _rand(T, V, scale=2.0)
    tg = torch.randint(0, V, (T,), device=_dev())
    tg[::7] = -100
    lf = logits.float().requires_grad_(True)
    ref = F.cross_entropy(lf, tg, ignore_index=-100, reduction="sum")
    scale = 1.0 / 123.0
    (ref * scale).backward()
    stats = torch.zeros(4, dtype=torch.float64, device=_dev())
    work = logits.clone()
    ops.cross_entropy(work, tg, scale, True, stats)
    assert abs(stats[0].item() - ref.item()) / ref.item() < 2e-3
    assert stats[1].item() == (tg != -100).sum().item()
    nc = ((logits.float().argmax(-1) == tg) & (tg != -100)).sum().item()
    assert abs(stats[2].item() - nc) <= 2
    _close(work, lf.grad, 3e-2, 1e-5, "dlogits")


def test_embedding_fwd_bwd():
    from photon_b200 import ops

    B, S, d, V = 3, 64, 768, 1000
    ids = torch.randint(0, V, (B * S,), device=_dev())
    wte, wpe = _rand(V, d), _rand(S, d)
    out = torch.empty(B * S, d, device=_dev(), dtype=torch.bfloat16)
    ops.embed_fwd(ids, wte, wpe, out, S)
    ref = wte.float()[ids] + wpe.float().repeat(B, 1)
    _close(out, ref, 1e-2, 1e-2, "embed fwd")
    dh = _rand(B * S, d)
    dwte, dwpe = torch.zeros(V, d, device=_dev()), torch.zeros(S, d, device=_dev())
    ops.embed_bwd(ids, dh, dwte, dwpe, S)
    rwte = torch.zeros(V, d, device=_dev()).index_add_(0, ids, dh.float())
    _close(dwte, rwte, 1e-3, 1e-3, "embed bwd wte")
    _close(dwpe, dh.float().view(B, S, d).sum(0), 1e-3, 1e-3, "embed bwd wpe")


def test_colsum_norm_axpby_cast():
    from photon_b200 import ops

    dy = _rand(1000, 3072)
    out = torch.zeros(3072, device=_dev())
    ops.col_sum(dy, out)
    _close(out, dy.float().sum(0), 1e-3, 5e-2, "col_sum")
    x = torch.randn(1 << 20, device=_dev())
    assert abs(ops.flat_l2_norm(x).item() - x.double().norm().item()) / x.norm().item() < 1e-5
    acc, y = torch.randn(4096, device=_dev()), torch.randn(4096, device=_dev())
    ref = 0.25 * acc + 0.75 * y
    ops.axpby_(acc, y, 0.25, 0.75)
    _close(acc, ref, 1e-6, 1e-6, "axpby")
    dst = torch.empty(4096, device=_dev(), dtype=torch.bfloat16)
    ops.cast_bf16(y, dst)
    assert torch.equal(dst, y.to(torch.bfloat16))


@pytest.mark.parametrize("name", ["adopt", "decoupled_adamw"])
def test_fused_optimizer_matches_torch_path(name):
    import torch.nn as nn

    from photon_b200.train.optim import build_optimizer
    from photon_b200.utils.flat import FlatParams

    torch.manual_seed(0)
    mk = lambda: nn.Sequential(nn.Linear(64, 64), nn.Linear(64, 32)).to(_dev())  # noqa: E731
    ma, mb = mk(), mk()
    mb.load_state_dict(ma.state_dict())
    fa, fb = FlatParams(ma), FlatParams(mb)
    cfg = dict(name=name, lr=1e-2, betas=[0.9, 0.99], eps=1e-6, weight_decay=0.01)
    shadow = torch.zeros(fa.layout.total, device=_dev(), dtype=torch.bfloat16)
    oa = build_optimizer(cfg, fa, use_kernel=True, bf16_shadow=shadow)
    ob = build_optimizer(cfg, fb, use_kernel=False)
    for step in range(4):
        g = torch.randn(fa.layout.total, device=_dev())
        fa.grads.copy_(g), fb.grads.copy_(g)
        gm = torch.tensor(0.5, device=_dev())
        oa.step(0.9, gm), ob.step(0.9, gm)
    _close(fa.params, fb.params, 1e-5, 1e-6, f"{name} params")
    _close(oa.exp_avg_sq, ob.exp_avg_sq, 1e-5, 1e-8, f"{name} v")
    assert torch.equal(shadow, fa.params.to(torch.bfloat16))


def test_gemm_gelu_with_saved_derivative_and_mul_epilogue():
    """EPI_GELU_GRAD (act + gelu'(z) from one CDF/PDF evaluation) and EPI_MUL (dgrad * saved derivative) reproduce the
    exact-erf GELU forward / backward."""
    from photon_b200 import ops

    torch.manual_seed(0)
    T, K, N = 512, 256, 768
    x = (torch.randn(T, K, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)
    b = torch.randn(N, device="cuda") * 0.1
    act = torch.empty(T, N, device="cuda", dtype=torch.bfloat16)
    dact = torch.empty_like(act)
    ops.linear_gelu_grad_fwd(x, w, b, dact, act)
    z = (x.float() @ w.float().t() + b).requires_grad_(True)
    ref = torch.nn.functional.gelu(z)
    (gref,) = torch.autograd.grad(ref.sum(), z)
    assert (act.float() - ref).abs().max().item() < 3e-2
    assert (dact.float() - gref).abs().max().item() < 1.5e-2
    dy = (torch.randn(T, N, device="cuda") * 0.3).to(torch.bfloat16)
    w2 = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)          # [N_out, K_in] of the next layer
    mul = torch.rand(T, K, device="cuda").to(torch.bfloat16)
    dx = torch.empty(T, K, device="cuda", dtype=torch.bfloat16)
    ops.linear_dgrad(dy, w2, dx, mul=mul)
    rdx = (dy.float() @ w2.float()) * mul.float()
    assert ((dx.float() - rdx).norm() / rdx.norm()).item() < 1e-2
