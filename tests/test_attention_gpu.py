"""wgmma flash attention (fwd + bwd) vs an fp32 PyTorch reference of the same op."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv, H, causal=True):
    B, S, D3 = qkv.shape
    d = D3 // 3
    dh = d // H
    q, k, v = qkv.float().view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    att = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
    if causal:
        att = att.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=qkv.device).tril(), float("-inf"))
    lse = torch.logsumexp(att, dim=-1)
    o = torch.softmax(att, dim=-1) @ v
    return o.transpose(1, 2).reshape(B, S, d), lse


@pytest.mark.parametrize("B,S,H,dh", [(1, 128, 1, 64), (2, 256, 4, 64), (1, 512, 2, 64), (2, 256, 2, 128), (1, 2048, 2, 64)])
def test_attention_fwd(B, S, H, dh):
    from photon_b200 import ops

    d = H * dh
    qkv = (torch.randn(B, S, 3 * d, device="cuda:0") * 1.0).to(torch.bfloat16)
    out = torch.empty(B, S, d, device="cuda:0", dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda:0", dtype=torch.float32)
    ops.attention_fwd(qkv, out, lse, H, 1.0 / math.sqrt(dh), True)
    torch.cuda.synchronize()
    ro, rl = _ref(qkv, H)
    err = (out.float() - ro).abs().max().item()
    assert err < 3e-2, f"attention fwd max err {err}"
    assert (lse - rl).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,S,H,dh", [(1, 128, 1, 64), (1, 256, 2, 64), (2, 512, 4, 64), (1, 2048, 2, 64),
                                      (1, 128, 1, 128), (2, 512, 3, 128), (1, 1024, 2, 128)])
def test_attention_bwd(B, S, H, dh):
    from photon_b200 import ops

    d = H * dh
    qkv = (torch.randn(B, S, 3 * d, device="cuda:0")).to(torch.bfloat16)
    dout = (torch.randn(B, S, d, device="cuda:0")).to(torch.bfloat16)
    out = torch.empty(B, S, d, device="cuda:0", dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda:0", dtype=torch.float32)
    scale = 1.0 / math.sqrt(dh)
    ops.attention_fwd(qkv, out, lse, H, scale, True)
    dqkv = torch.zeros_like(qkv)
    delta = torch.empty_like(lse)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True)
    torch.cuda.synchronize()
    x = qkv.float().requires_grad_(True)
    ro, _ = _ref(x, H)
    ro.backward(dout.float())
    g = x.grad
    for name, sl in (("dq", slice(0, d)), ("dk", slice(d, 2 * d)), ("dv", slice(2 * d, 3 * d))):
        a, b = dqkv[..., sl].float(), g[..., sl]
        rel = ((a - b).norm() / b.norm()).item()
        assert rel < 3e-2, f"{name} rel err {rel}"


def _sdpa_ref(qkv, H, causal, dout=None):
    """Library reference for shapes where the explicit S x S fp32 oracle is too large."""
    B, S, D3 = qkv.shape
    d = D3 // 3
    dh = d // H
    x = qkv.float().requires_grad_(dout is not None)
    q, k, v = x.view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal).transpose(1, 2).reshape(B, S, d)
    if dout is None:
        return o, None
    o.backward(dout.float())
    return o.detach(), x.grad


@pytest.mark.parametrize("B,S,H,causal,dh", [(4, 1024, 12, True, 64), (8, 512, 12, True, 64), (3, 768, 5, True, 64), (4, 512, 12, False, 64),
                                             (2, 1024, 3, False, 64), (4, 1024, 16, True, 128), (2, 512, 8, False, 128)])
def test_attention_persistent_many_items(B, S, H, causal, dh):
    """More work items than SMs: every CTA walks several (batch*head, tile) items, so the cross-item pipelines
    (barrier parities, double-buffered O / K-V, deferred epilogues) and the non-causal path are exercised."""
    from photon_b200 import ops

    d = H * dh
    qkv = torch.randn(B, S, 3 * d, device="cuda:0").to(torch.bfloat16)
    dout = torch.randn(B, S, d, device="cuda:0").to(torch.bfloat16)
    out = torch.empty(B, S, d, device="cuda:0", dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda:0", dtype=torch.float32)
    scale = 1.0 / math.sqrt(dh)
    ops.attention_fwd(qkv, out, lse, H, scale, causal)
    dqkv = torch.zeros_like(qkv)
    delta = torch.empty_like(lse)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, causal)
    torch.cuda.synchronize()
    ro, g = _sdpa_ref(qkv, H, causal, dout)
    assert (out.float() - ro).abs().max().item() < 3e-2
    for name, sl in (("dq", slice(0, d)), ("dk", slice(d, 2 * d)), ("dv", slice(2 * d, 3 * d))):
        a, b = dqkv[..., sl].float(), g[..., sl]
        rel = ((a - b).norm() / b.norm()).item()
        assert rel < 3e-2, f"{name} rel err {rel}"
    # second call on the same buffers must give the same answer (no state leaks between launches)
    out2 = torch.empty_like(out)
    ops.attention_fwd(qkv, out2, lse, H, scale, causal)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("B,S,H,dh", [(2, 512, 4, 64), (1, 1024, 3, 128)])
def test_attention_alibi_fwd_bwd(B, S, H, dh):
    """attn_config.alibi: score += slope_h * (key - query) inside both kernels, vs an explicit fp32 oracle."""
    from photon_b200 import ops
    from photon_b200.models.mpt import alibi_slopes

    d = H * dh
    qkv = torch.randn(B, S, 3 * d, device="cuda:0").to(torch.bfloat16)
    dout = torch.randn(B, S, d, device="cuda:0").to(torch.bfloat16)
    slopes = alibi_slopes(H, 8).to("cuda:0")
    out = torch.empty(B, S, d, device="cuda:0", dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda:0", dtype=torch.float32)
    scale = 1.0 / math.sqrt(dh)
    ops.attention_fwd(qkv, out, lse, H, scale, True, slopes)
    dqkv = torch.zeros_like(qkv)
    delta = torch.empty_like(lse)
    ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, slopes)
    torch.cuda.synchronize()
    x = qkv.float().requires_grad_(True)
    q, k, v = x.view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    pos = torch.arange(S, device="cuda:0")
    bias = slopes[:, None, None] * (pos[None, :] - pos[:, None]).clamp(max=0).float()[None]
    att = (q @ k.transpose(-1, -2)) * scale + bias[None]
    att = att.masked_fill(~torch.ones(S, S, dtype=torch.bool, device="cuda:0").tril(), float("-inf"))
    ro = (torch.softmax(att, dim=-1) @ v).transpose(1, 2).reshape(B, S, d)
    assert (out.float() - ro).abs().max().item() < 3e-2
    assert (lse - torch.logsumexp(att, dim=-1)).abs().max().item() < 2e-2
    ro.backward(dout.float())
    for name, sl in (("dq", slice(0, d)), ("dk", slice(d, 2 * d)), ("dv", slice(2 * d, 3 * d))):
        a, b = dqkv[..., sl].float(), x.grad[..., sl]
        assert ((a - b).norm() / b.norm()).item() < 3e-2, name


def test_rope_kernel_matches_oracle_and_inverts():
    from photon_b200 import ops
    from photon_b200.models.mpt import apply_rope, rope_tables

    B, S, H, dh = 2, 256, 4, 64
    d = H * dh
    qkv = torch.randn(B, S, 3 * d, device="cuda:0").to(torch.bfloat16)
    cos, sin = rope_tables(S, dh, 10000.0, "cuda:0")
    ref = qkv.float().view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)            # [3, B, H, S, dh]
    rq, rk = apply_rope(ref[0], cos, sin), apply_rope(ref[1], cos, sin)
    work = qkv.clone()
    ops.rope_(work, cos.contiguous(), sin.contiguous(), H)
    got = work.float().view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    assert (got[0] - rq).abs().max().item() < 3e-2 and (got[1] - rk).abs().max().item() < 3e-2
    assert torch.equal(got[2], ref[2])                                        # v untouched
    ops.rope_(work, cos.contiguous(), sin.contiguous(), H, inverse=True)      # rotation is orthogonal
    assert (work.float() - qkv.float()).abs().max().item() < 6e-2
