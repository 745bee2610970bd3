"""Fit attention-forward time = CTAs/SMs * (F + n_kv * t): fixed per-CTA cost F vs per-KV-tile cost t.

Non-causal runs with the same number of CTAs (b*H*S/128 fixed) but different n_kv = S/128 separate the two.
Run on a GPU:  python scripts/attn_scaling.py
"""
import json
import sys

import torch

sys.path.insert(0, ".")
from photon_b200 import ops  # noqa: E402


def timed(fn, iters=10):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    global SMS
    SMS = torch.cuda.get_device_properties(0).multi_processor_count
    H, dh = 12, 64
    rows = []
    for causal in (False, True):
        for S in (256, 512, 1024, 2048, 4096):
            b = max(1, (32 * 2048) // S)           # b*S constant -> same number of CTAs
            qkv = torch.randn(b, S, 3 * H * dh, device="cuda", dtype=torch.bfloat16)
            out = torch.empty(b, S, H * dh, device="cuda", dtype=torch.bfloat16)
            lse = torch.empty(b, H, S, device="cuda", dtype=torch.float32)
            ms = timed(lambda: ops.attention_fwd(qkv, out, lse, H, dh ** -0.5, causal))
            ctas = b * H * S // 128
            n_kv = (S // 128 + 1) / 2 if causal else S // 128
            us_per_cta = ms * 1e3 * SMS / ctas
            rows.append(dict(causal=causal, S=S, b=b, ms=ms, ctas=ctas, avg_kv_tiles=n_kv, us_per_cta=us_per_cta))
            print(rows[-1], flush=True)
    # backward: same fit (one CTA per (b, h, kv tile) walking the query tiles)
    brow = []
    for causal in (False, True):
        for S in (256, 512, 1024, 2048, 4096):
            b = max(1, (32 * 2048) // S)
            qkv = torch.randn(b, S, 3 * H * dh, device="cuda", dtype=torch.bfloat16)
            out = torch.empty(b, S, H * dh, device="cuda", dtype=torch.bfloat16)
            lse = torch.empty(b, H, S, device="cuda", dtype=torch.float32)
            ops.attention_fwd(qkv, out, lse, H, dh ** -0.5, causal)
            dout = torch.randn_like(out)
            dqkv = torch.empty_like(qkv)
            delta = torch.empty(b, H, S, device="cuda", dtype=torch.float32)
            ms = timed(lambda: ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, dh ** -0.5, causal))
            ctas = b * H * S // 128
            n_q = (S // 128 + 1) / 2 if causal else S // 128
            brow.append(dict(bwd=True, causal=causal, S=S, ms=ms, avg_q_tiles=n_q, us_per_cta=ms * 1e3 * SMS / ctas))
            print(brow[-1], flush=True)
    bn = [r for r in brow if not r["causal"]]
    tb = (bn[-1]["us_per_cta"] - bn[0]["us_per_cta"]) / (bn[-1]["avg_q_tiles"] - bn[0]["avg_q_tiles"])
    print(json.dumps({"bwd_per_q_tile_us": tb, "bwd_fixed_per_cta_us": bn[0]["us_per_cta"] - tb * bn[0]["avg_q_tiles"],
                      "note": "includes the delta / dq-convert helper kernels"}))
    nc = [r for r in rows if not r["causal"]]
    x0, x1 = nc[0], nc[-1]
    t = (x1["us_per_cta"] - x0["us_per_cta"]) / (x1["avg_kv_tiles"] - x0["avg_kv_tiles"])
    F = x0["us_per_cta"] - t * x0["avg_kv_tiles"]
    print(json.dumps({"per_kv_tile_us": t, "fixed_per_cta_us": F}))


if __name__ == "__main__":
    main()
