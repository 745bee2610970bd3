"""Grouped-query attention on MPT-1B shapes (16 heads of 128, S = 2048) at kv_n_heads 16 (multi-head), 4 and 1 (multi-query):

* attention forward + backward (``ops.attention_fwd`` + ``ops.attention_bwd``) at microbatch 8;
* one decode step's attention for one layer (``decode_append`` + ``decode_attention``) at batch 32 with 2048 cached positions,
  with the cache bytes it reads per step and the whole 24-layer cache size;
* one training microbatch (forward + backward, ``B200Engine.fwd_bwd``) of MPT-1B at microbatch 4 (the three engines stay
  resident so that the variants alternate, and only one workspace is alive at a time).

Variants are alternated inside every repeat (the spread of the repeats is printed), and the card's name and power limit are read
in the same run. Prints one JSON document.

    python scripts/gqa_bench.py [--repeats 3] [--quick] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

H, DH, S, L, D = 16, 128, 2048, 24, 2048
KV = (16, 4, 1)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().splitlines() or ["?, ?, ?"])[0].split(", ")
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def time_fn(fn, iters: int, warmup: int = 3) -> float:
    """Mean seconds per call by CUDA events over ``iters`` calls after ``warmup``."""
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def attention_case(kv: int, dev, B: int = 8):
    from photon_b200 import ops

    g = torch.Generator(device=dev).manual_seed(kv)
    qkv = torch.randn(B, S, (H + 2 * kv) * DH, device=dev, generator=g).bfloat16()
    dout = torch.randn(B, S, H * DH, device=dev, generator=g).bfloat16()
    out = torch.empty(B, S, H * DH, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(B, H, S, dtype=torch.float32, device=dev)
    dqkv, delta = torch.empty_like(qkv), torch.empty_like(lse)
    scale = 1.0 / math.sqrt(DH)

    def run():
        ops.attention_fwd(qkv, out, lse, H, scale, True, n_kv_heads=kv)
        ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, n_kv_heads=kv)
    return run


def decode_case(kv: int, dev, B: int = 32):
    from photon_b200 import ops

    g = torch.Generator(device=dev).manual_seed(kv)
    kc = torch.randn(B, kv, S, DH, device=dev, generator=g).bfloat16()
    vc = torch.randn_like(kc)
    qkv = torch.randn(B, (H + 2 * kv) * DH, device=dev, generator=g).bfloat16()
    pos = torch.full((B,), S - 1, dtype=torch.int32, device=dev)   # the last position: 2047 cached keys plus the new one
    out = torch.empty(B, H * DH, dtype=torch.bfloat16, device=dev)

    def run():
        ops.decode_append(qkv, pos, kc, vc, None, H, n_kv_heads=kv)
        ops.decode_attention(qkv, kc, vc, pos, out, H, 1.0 / math.sqrt(DH), n_kv_heads=kv)
    return run


def train_engine(kv: int, dev):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=D, n_heads=H, n_layers=L, max_seq_len=S, vocab_size=50368, kv_n_heads=kv)
    return B200Engine(cfg, dev, "amp_bf16", {}, seed=0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="attention and decode only (no MPT-1B training microbatch)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gqa_bench.py measures on the GPU; there is none here")
    dev = torch.device("cuda", 0)
    res: dict = {"card": card(), "shapes": dict(n_heads=H, d_head=DH, seq=S, n_layers=L, d_model=D), "kv_n_heads": list(KV)}
    attn = {kv: attention_case(kv, dev) for kv in KV}
    dec = {kv: decode_case(kv, dev) for kv in KV}
    times: dict = {k: {kv: [] for kv in KV} for k in ("attn_fwd_bwd_ms", "decode_attn_us")}
    for _ in range(a.repeats):
        for kv in KV:   # alternated inside every repeat
            times["attn_fwd_bwd_ms"][kv].append(time_fn(attn[kv], 10) * 1e3)
            times["decode_attn_us"][kv].append(time_fn(dec[kv], 100) * 1e6)
    del attn, dec
    if not a.quick:
        times["train_microbatch_ms"] = {kv: [] for kv in KV}
        engines = {kv: train_engine(kv, dev) for kv in KV}
        ids = torch.randint(0, 50368, (4, S), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        denom = float(ids.numel())
        for _ in range(a.repeats):
            for kv, eng in engines.items():
                times["train_microbatch_ms"][kv].append(time_fn(lambda e=eng: e.fwd_bwd(ids, denom), 5, warmup=2) * 1e3)
                eng.close()   # one workspace at a time (the three engines' parameters stay resident)
        res["num_params"] = {kv: e.cfg.num_params() for kv, e in engines.items()}
        del engines
    for k, per in times.items():
        res[k] = {kv: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for kv, v in per.items()}
    res["decode_cache_bytes_read_per_layer_step"] = {kv: 2 * 32 * kv * S * DH * 2 for kv in KV}
    res["decode_cache_gb_24_layers"] = {kv: L * 2 * 32 * kv * S * DH * 2 / 1e9 for kv in KV}
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
