"""Our wgmma attention forward / backward vs the library kernels on the same tensors, at both flagship geometries:
(b32, H12, S2048, d64) = MPT-125M and (b8, H16, S2048, d128) = MPT-1B. Libraries: torch SDPA restricted to each backend
(cuDNN, flash) and flash-attn 2.8 (the package the reference calls, here its build for the installed GPU). CUDA-event timed, L2 flushed."""
import json
import math
import sys

import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

sys.path.insert(0, ".")
from photon_b200 import ops  # noqa: E402

dev = "cuda"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timed(fn, it=8):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(it):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


rows = []
for B, S, H, dh in [(32, 2048, 12, 64), (8, 2048, 16, 128)]:
    d = H * dh
    qkv = torch.randn(B, S, 3 * d, device=dev).to(torch.bfloat16)
    dout = torch.randn(B, S, d, device=dev).to(torch.bfloat16)
    out = torch.empty(B, S, d, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device=dev)
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    scale = 1 / math.sqrt(dh)
    row = {"shape": {"B": B, "S": S, "H": H, "d_head": dh}, "fwd_ms": {}, "bwd_ms": {}}
    row["fwd_ms"]["ours"] = timed(lambda: ops.attention_fwd(qkv, out, lse, H, scale, True))
    row["bwd_ms"]["ours"] = timed(lambda: ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True))
    x = qkv.detach().requires_grad_(True)
    g = dout.view(B, S, H, dh).transpose(1, 2)
    for name, be in (("sdpa_cudnn", SDPBackend.CUDNN_ATTENTION), ("sdpa_flash", SDPBackend.FLASH_ATTENTION)):
        try:
            with sdpa_kernel(be):
                def fwd():
                    q, k, v = x.view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
                    return torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)

                row["fwd_ms"][name] = timed(fwd)
                o = fwd()
                row["bwd_ms"][name] = timed(lambda: torch.autograd.grad(o, x, g, retain_graph=True))
        except Exception as e:  # noqa: BLE001
            row["fwd_ms"][name] = row["bwd_ms"][name] = f"unavailable: {type(e).__name__}"
    try:
        from flash_attn import flash_attn_qkvpacked_func

        xp = qkv.view(B, S, 3, H, dh).detach().requires_grad_(True)
        row["fwd_ms"]["flash_attn_2.8"] = timed(lambda: flash_attn_qkvpacked_func(xp, causal=True))
        o2 = flash_attn_qkvpacked_func(xp, causal=True)
        g2 = dout.view(B, S, H, dh)
        row["bwd_ms"]["flash_attn_2.8"] = timed(lambda: torch.autograd.grad(o2, xp, g2, retain_graph=True))
    except Exception as e:  # noqa: BLE001
        row["fwd_ms"]["flash_attn_2.8"] = row["bwd_ms"]["flash_attn_2.8"] = f"unavailable: {type(e).__name__}"
    fl = 4 * B * H * S * S * dh / 2
    row["fwd_tflops_ours"] = fl / row["fwd_ms"]["ours"] / 1e9
    row["bwd_tflops_ours"] = 2.5 * fl / row["bwd_ms"]["ours"] / 1e9
    best_f = min(v for k, v in row["fwd_ms"].items() if k != "ours" and isinstance(v, float))
    best_b = min(v for k, v in row["bwd_ms"].items() if k != "ours" and isinstance(v, float))
    row["ours_vs_best_library"] = {"fwd": best_f / row["fwd_ms"]["ours"], "bwd": best_b / row["bwd_ms"]["ours"]}
    rows.append(row)
    print(json.dumps(row), flush=True)
open("gpurun_out/attn_vs_library.json", "w").write(json.dumps(rows, indent=1))
