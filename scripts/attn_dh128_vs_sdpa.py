"""d_head = 128 attention (MPT-1B geometry): our wgmma forward / backward vs torch SDPA (library) on the same tensors."""
import math
import sys

import torch

sys.path.insert(0, ".")
from photon_b200 import ops  # noqa: E402

B, S, H, dh = 8, 2048, 16, 128
d = H * dh
dev = "cuda"
qkv = torch.randn(B, S, 3 * d, device=dev).to(torch.bfloat16)
dout = torch.randn(B, S, d, device=dev).to(torch.bfloat16)
out = torch.empty(B, S, d, device=dev, dtype=torch.bfloat16)
lse = torch.empty(B, H, S, device=dev)
dqkv = torch.empty_like(qkv)
delta = torch.empty_like(lse)
scale = 1 / math.sqrt(dh)


def timed(fn, it=10):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(it):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / it


f_ours = timed(lambda: ops.attention_fwd(qkv, out, lse, H, scale, True))
b_ours = timed(lambda: ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True))
x = qkv.detach().requires_grad_(True)


def sdpa_fwd():
    q, k, v = x.view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
    return torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)


f_lib = timed(lambda: sdpa_fwd())
o = sdpa_fwd()
g = dout.view(B, S, H, dh).transpose(1, 2)
b_lib = timed(lambda: torch.autograd.grad(o, x, g, retain_graph=True))
flops_f = 4 * B * H * S * S * dh / 2
print({"shape": [B, S, H, dh], "fwd_ms": {"ours": f_ours, "sdpa": f_lib}, "bwd_ms": {"ours": b_ours, "sdpa": b_lib},
       "fwd_tflops_ours": flops_f / f_ours / 1e9, "bwd_tflops_ours": 2.5 * flops_f / b_ours / 1e9})
