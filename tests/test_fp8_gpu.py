"""fp8 (wgmma e4m3 / e5m2) path: GEMMs, quantising producers and the amp_fp8 engine vs PyTorch fp32 references.

The oracle is the recipe of ``photon_b200/train/fp8.py``: operands are the fp8 values (E4M3 forward, E5M2 gradients) times
per-tensor scales, products exact, accumulation fp32, de-scale in the epilogue."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FMAX = {E4M3: 448.0, E5M2: 57344.0}


def _dev():
    return torch.device("cuda", 0)


def _q(x, dtype, scale):
    """(bits as uint8, de-quantised fp32 values) of the saturating cast of ``x * scale``."""
    q = (x.float() * scale).clamp(-FMAX[dtype], FMAX[dtype]).to(dtype)
    return q.view(torch.uint8), q.float() / scale


def _meta(scales):
    m = torch.zeros(3, len(scales), device=_dev())
    m[0] = torch.tensor(scales, device=_dev())
    m[1] = 1.0 / m[0]
    return m


def _close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).float().mean().item()
    assert bad == 0.0, f"{what}: {bad * 100:.4f}% elements out of tolerance, max err {err.max().item():.4g}, ref max {ref.abs().max().item():.4g}"


@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("M,N,K", [(128, 256, 128), (640, 520, 1088), (1024, 2304, 768), (200, 328, 272)])
def test_gemm_fp8_forward_bias_residual(M, N, K, cluster):
    from photon_b200 import ops

    x, w = torch.randn(M, K, device=_dev()), torch.randn(N, K, device=_dev()) * 0.05
    sx, sw = 448.0 / x.abs().max().item(), 448.0 / w.abs().max().item()
    x8, xd = _q(x, E4M3, sx)
    w8, wd = _q(w, E4M3, sw)
    bias = torch.randn(N, device=_dev())
    res = torch.randn(M, N, device=_dev()).bfloat16()
    meta = _meta([sx, sw])
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    ops.gemm_fp8(x8, w8, out, meta, 0, 1, bias=bias, cluster=cluster)
    ref = xd @ wd.t() + bias
    _close(out, ref, 1e-2, 1e-2, "fp8 K/K + bias")           # bf16 output rounding only: products and sums are exact / fp32
    ops.gemm_fp8(x8, w8, out, meta, 0, 1, epi=ops.EPI_RESIDUAL, bias=bias, aux=res, cluster=cluster)
    _close(out, ref + res.float(), 1e-2, 2e-2, "fp8 K/K + bias + residual")


@pytest.mark.parametrize("cluster", [1, 2])
def test_gemm_fp8_dgrad_mn_major_weight(cluster):
    """dX = dY(E5M2, K-major) · W(E4M3, stored [N,K], consumed MN-major) — the 8-bit formats allow MN-major operands."""
    from photon_b200 import ops

    T, N, K = 640, 1088, 528
    dy, w = torch.randn(T, N, device=_dev()) * 1e-3, torch.randn(N, K, device=_dev()) * 0.05
    sg, sw = 57344.0 / dy.abs().max().item(), 448.0 / w.abs().max().item()
    dy8, dyd = _q(dy, E5M2, sg)
    w8, wd = _q(w, E4M3, sw)
    meta = _meta([sg, sw])
    dx = torch.empty(T, K, device=_dev(), dtype=torch.bfloat16)
    ops.gemm_fp8(dy8, w8, dx, meta, 0, 1, b_mn=True, a_fmt=ops.E5M2, b_fmt=ops.E4M3, cluster=cluster)
    ref = dyd @ wd
    _close(dx, ref, 1e-2, 1e-2 * ref.abs().max().item(), "fp8 dgrad")
    mul = torch.rand(T, K, device=_dev()).bfloat16()
    ops.gemm_fp8(dy8, w8, dx, meta, 0, 1, b_mn=True, epi=ops.EPI_MUL, a_fmt=ops.E5M2, b_fmt=ops.E4M3, aux=mul, cluster=cluster)
    _close(dx, ref * mul.float(), 1e-2, 1e-2 * ref.abs().max().item(), "fp8 dgrad * mul")


@pytest.mark.parametrize("cluster", [1, 2])
def test_gemm_fp8_wgrad_both_mn_major_splitk(cluster):
    """dW += dY^T(E5M2) · X(E4M3): both operands consumed MN-major from their [T, ·] storage, fp32 TMA reduce-add, split-K."""
    from photon_b200 import ops

    T, N, K = 4352, 640, 528
    dy, x = torch.randn(T, N, device=_dev()) * 1e-3, torch.randn(T, K, device=_dev())
    sg, sx = 57344.0 / dy.abs().max().item(), 448.0 / x.abs().max().item()
    dy8, dyd = _q(dy, E5M2, sg)
    x8, xd = _q(x, E4M3, sx)
    meta = _meta([sg, sx])
    dw0 = torch.randn(N, K, device=_dev())
    dw = dw0.clone()
    ops.gemm_fp8(dy8, x8, dw, meta, 0, 1, a_mn=True, b_mn=True, epi=ops.EPI_F32, a_fmt=ops.E5M2, b_fmt=ops.E4M3, accumulate=True,
                 cluster=cluster)
    ref = dw0 + dyd.t() @ xd
    _close(dw, ref, 1e-4, 1e-4 * ref.abs().max().item(), "fp8 wgrad")


def test_gemm_fp8_gelu_epilogue_emits_e4m3_and_amax():
    from photon_b200 import ops

    M, N, K = 512, 1024, 768
    x, w = torch.randn(M, K, device=_dev()), torch.randn(N, K, device=_dev()) * 0.05
    sx, sw = 448.0 / x.abs().max().item(), 448.0 / w.abs().max().item()
    x8, xd = _q(x, E4M3, sx)
    w8, wd = _q(w, E4M3, sw)
    bias = torch.randn(N, device=_dev())
    z = xd @ wd.t() + bias
    act = F.gelu(z)
    su = 448.0 / act.abs().max().item()
    meta = _meta([sx, sw, su])
    dact = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    u8 = torch.zeros(M, N, device=_dev(), dtype=torch.uint8)
    ops.gemm_fp8(x8, w8, dact, meta, 0, 1, epi=ops.EPI_GELU_GRAD_Q8, bias=bias, out2=dact, out8=u8, role_out=2)
    zz = z.clone().requires_grad_(True)
    (gref,) = torch.autograd.grad(F.gelu(zz).sum(), zz)
    _close(dact, gref, 1e-2, 1e-2, "gelu'")
    got = u8.view(E4M3).float() / su
    _close(got, act, 0.07, 2e-3 * act.abs().max().item(), "gelu as E4M3")      # one E4M3 ulp = 2^-3 relative
    assert abs(meta[2, 2].item() - act.abs().max().item()) <= 2e-2 * act.abs().max().item()


@pytest.mark.parametrize("d", [768, 2048])
def test_layernorm_fwd_q8(d):
    from photon_b200 import ops

    T = 1000
    x = (torch.randn(T, d, device=_dev()) * 2 + 0.3).bfloat16()
    g, b = torch.rand(d, device=_dev()) + 0.5, torch.randn(d, device=_dev()) * 0.1
    ref = F.layer_norm(x.float(), (d,), g, b, 1e-5)
    s = 448.0 / ref.abs().max().item() * 0.9
    meta = _meta([1.0, s])
    y8 = torch.zeros(T, d, device=_dev(), dtype=torch.uint8)
    mean, rstd = torch.empty(T, device=_dev()), torch.empty(T, device=_dev())
    ops.layernorm_fwd_q8(x, g, b, y8, mean, rstd, 1e-5, meta, 1)
    _, want = _q(ref, E4M3, s)
    got = y8.view(E4M3).float() / s
    assert ((got - want).abs() > 0.13 * want.abs() + 1e-3).float().mean().item() < 1e-4     # rounding-boundary flips only
    assert abs(meta[2, 1].item() - ref.abs().max().item()) < 1e-2 * ref.abs().max().item()
    torch.testing.assert_close(mean, x.float().mean(-1), rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_colsum_quant_one_pass(fmt):
    from photon_b200 import ops

    T, N = 3000, 2304
    dt = E4M3 if fmt == "e4m3" else E5M2
    dy = (torch.randn(T, N, device=_dev()) * 3e-4).bfloat16()
    s = FMAX[dt] / dy.float().abs().max().item()
    meta = _meta([s])
    db0 = torch.randn(N, device=_dev())
    db = db0.clone()
    y8 = torch.zeros(T, N, device=_dev(), dtype=torch.uint8)
    ops.colsum_quant(dy, db, y8, ops.E4M3 if fmt == "e4m3" else ops.E5M2, meta, 0)
    torch.testing.assert_close(db, db0 + dy.float().sum(0), rtol=1e-4, atol=1e-5)
    bits, _ = _q(dy, dt, s)
    assert (y8 != bits).float().mean().item() < 1e-4
    assert abs(meta[2, 0].item() - dy.float().abs().max().item()) < 1e-6
    # pure column sum / pure quantise
    db2 = torch.zeros(N, device=_dev())
    ops.colsum_quant(dy, db2, None)
    torch.testing.assert_close(db2, dy.float().sum(0), rtol=1e-4, atol=1e-5)


def test_weight_segments_current_scaling_and_delayed_scale_update():
    from photon_b200 import ops

    n = 3
    sizes = [768 * 2304, 768 * 768, 3072 * 768]
    offs, total = [], 0
    for s in sizes:
        offs.append(total)
        total += s + 256
    src = torch.zeros(total, device=_dev(), dtype=torch.bfloat16)
    for o, s, k in zip(offs, sizes, (0.02, 0.5, 3.0)):
        src[o:o + s] = (torch.randn(s, device=_dev()) * k).bfloat16()
    seg = torch.tensor(list(zip(offs, sizes)), dtype=torch.int64, device=_dev())
    meta = torch.zeros(3, 2 + n, device=_dev())
    meta[:2] = 1.0
    dst = torch.zeros(total, device=_dev(), dtype=torch.uint8)
    ops.fp8_quantize_segments(src, dst, seg, meta, 2)
    for i, (o, s) in enumerate(zip(offs, sizes)):
        amax = src[o:o + s].float().abs().max().item()
        assert abs(meta[2, 2 + i].item() - amax) < 1e-6
        assert abs(meta[0, 2 + i].item() - 448.0 / amax) < 1e-3 * 448.0 / amax
        bits, _ = _q(src[o:o + s], E4M3, meta[0, 2 + i].item())
        assert (dst[o:o + s] != bits).float().mean().item() < 1e-4
    # delayed scaling over a 4-deep history for the two dynamic roles
    hist = torch.zeros(2, 4, device=_dev())
    fmax = torch.tensor([448.0, 57344.0], device=_dev())
    pos = torch.zeros(1, dtype=torch.int32, device=_dev())
    for step, (a0, a1) in enumerate([(2.0, 1e-3), (8.0, 5e-4), (1.0, 1e-4), (1.0, 1e-4), (1.0, 1e-4), (1.0, 1e-4)]):
        meta[2, 0], meta[2, 1] = a0, a1
        ops.fp8_update_scales(meta, hist, fmax, pos, 2, 1.0)
        window0 = [2.0, 8.0, 1.0, 1.0, 1.0, 1.0][max(0, step - 3): step + 1]
        assert abs(meta[0, 0].item() - 448.0 / max(window0)) < 1e-3
        assert meta[2, 0].item() == 0.0 and abs(meta[0, 0].item() * meta[1, 0].item() - 1.0) < 1e-6
    assert int(pos.item()) == 6
    assert abs(meta[0, 1].item() - 57344.0 / 1e-4) / (57344.0 / 1e-4) < 1e-5


def _make(precision, graph):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048)
    return B200Engine(cfg, device=_dev(), precision=precision, kernels={"cuda_graph": graph}, seed=3)


def _torch_grads(precision, params, ids):
    """Gradients of the stock-PyTorch backend (``amp_fp8`` = the quantise/de-quantise emulation of train/fp8.py: the recipe oracle)."""
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.backend import TorchBackend

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048)
    be = TorchBackend(cfg, device=_dev(), precision=precision, seed=3)
    be.flat.params.copy_(params)
    be.flat.zero_grad()
    be.fwd_bwd(ids, 4.0 * 255)
    return be.flat.grads.clone()


@pytest.mark.parametrize("graph", [False, True])
def test_engine_amp_fp8_tracks_bf16(graph):
    """Same weights, same batch: the fp8 engine's loss follows the bf16 engine's and its gradients are as close to the bf16
    gradients as the recipe allows — per large tensor, cosine(ours fp8, ours bf16) is no worse than what the PyTorch emulation of
    the same recipe achieves against PyTorch bf16 (minus a small margin) — through eager launches and CUDA-graph replay."""
    e8, e16 = _make("amp_fp8", graph), _make("amp_bf16", graph)
    assert e8.fp8 and not e16.fp8
    e8.flat.params.copy_(e16.flat.params)
    e8.params_updated()
    ids = torch.randint(0, 2048, (4, 256), device=_dev())
    o8, o16 = _torch_grads("amp_fp8", e16.flat.params, ids), _torch_grads("amp_bf16", e16.flat.params, ids)
    for _ in range(2):           # second call replays the graph (when enabled) and uses rolled scales
        for e in (e8, e16):
            e.flat.zero_grad()
        l8, n8 = e8.fwd_bwd(ids, 4.0 * 255)
        l16, n16 = e16.fwd_bwd(ids, 4.0 * 255)
    assert float(n8) == float(n16)
    assert abs(float(l8) - float(l16)) / float(l16) < 2e-2
    lay = e8.flat.layout

    def cos(x, y, i):
        a, b = lay.view(x, i).flatten().double(), lay.view(y, i).flatten().double()
        return float((a @ b) / (a.norm() * b.norm()))

    for i, name in enumerate(lay.names):
        if lay.numels[i] < 256 * 256:
            continue
        assert cos(e16.flat.grads, o16, i) > 0.99, (name, "bf16 engine vs torch bf16")
        ours, oracle = cos(e8.flat.grads, e16.flat.grads, i), cos(o8, o16, i)
        assert ours > 0.95 and ours > oracle - 0.015, (name, ours, oracle)
    assert float((e8.fp8_meta[0, : e8._n_dyn] != 1.0).float().mean()) == 1.0     # every activation / gradient role got a scale
    sd = e8.fp8_state_dict()
    e8.load_fp8_state_dict(sd)
    st = e8.eval_stats(ids)
    assert torch.isfinite(st["loss_sum"])


def test_trainer_amp_fp8_loss_goes_down():
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.train.trainer import Trainer

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=1024)
    ids = torch.randint(0, cfg.vocab_size, (8, cfg.max_seq_len))

    class Loader:
        def __iter__(self):
            while True:
                yield {"input_ids": ids, "labels": ids}

    tr = Trainer(cfg, optimizer_cfg=dict(name="decoupled_adamw", lr=2e-3, betas=[0.9, 0.95], eps=1e-8, weight_decay=0.0),
                 scheduler_cfg=dict(name="cosine_with_warmup", t_warmup="2ba", t_max="40ba", alpha_f=0.1), train_loader=Loader(),
                 global_train_batch_size=8, device_train_microbatch_size=4, precision="amp_fp8", max_duration="40ba",
                 grad_clip_norm=1.0, device=_dev())
    assert tr.state.backend.kind == "b200" and tr.state.backend.fp8
    tr.fit("30ba")
    loss = [v for _, v in tr.loggers[0].data["loss/train/total"]]
    assert loss[-1] < 0.6 * loss[0], loss
    assert tr.state_dict()["state"]["fp8"]["meta"].shape[0] == 3
    tr.close()


def _mx_dequant(q, sf, R):
    """E4M3 data x E8M0 scale atoms [K/128][rblk][512] -> fp32 (the layout ops.mx_quantize documents)."""
    G = q.shape[1] // 32
    r = torch.arange(R, device=q.device)[:, None].expand(R, G)
    g = torch.arange(G, device=q.device)[None, :].expand(R, G)
    s = sf[g // 4, r // 128, (r % 32) * 16 + ((r // 32) % 4) * 4 + (g % 4)]
    return q.view(E4M3).float() * torch.exp2(s.float() - 127).repeat_interleave(32, dim=1)


@pytest.mark.parametrize("M,N,K", [(128, 256, 128), (640, 776, 1152), (2048, 2304, 768)])
def test_gemm_mxfp8_block_scaled(M, N, K):
    """OCP MXFP8 (one E8M0 scale per 32 K-elements of every row of A and B, applied to the fp32 wgmma partial sum of each K group):
    quantiser and GEMM against the de-quantise-then-multiply oracle; rows of wildly different magnitude keep their precision."""
    from photon_b200 import ops

    x = (torch.randn(M, K, device=_dev()) * torch.exp(2 * torch.randn(M, 1, device=_dev()))).bfloat16()   # per-row magnitudes over ~4 decades
    w = (torch.randn(N, K, device=_dev()) * 0.05).bfloat16()
    xq, xsf = ops.mx_quantize(x)
    wq, wsf = ops.mx_quantize(w, 2 * ((N + 255) // 256))
    # the quantiser itself: power-of-two scale = 2^(floor(log2 amax) - 8) per 32-block, saturating E4M3 cast
    blocks = x.float().view(M, K // 32, 32)
    amax = blocks.abs().amax(-1)
    e = torch.where(amax > 0, torch.floor(torch.log2(amax)) - 8, torch.full_like(amax, -127.0))
    want_q = (blocks * torch.exp2(-e)[..., None]).clamp(-448, 448).to(E4M3).view(M, K)
    assert (xq.view(E4M3).float() != want_q.float()).float().mean().item() < 1e-4
    bias = torch.randn(N, device=_dev())
    out = torch.empty(M, N, device=_dev(), dtype=torch.bfloat16)
    ops.gemm_mxfp8(xq, wq, out, xsf, wsf, bias)
    ref = _mx_dequant(xq, xsf, M) @ _mx_dequant(wq, wsf, N).t() + bias
    _close(out, ref, 1e-2, 1e-2 * ref.abs().max().item() / 8, "mxfp8 gemm")
    full = x.float() @ w.float().t() + bias
    assert ((out.float() - full).norm() / full.norm()).item() < 0.06       # MXFP8 quantisation noise, not kernel error
