"""Decode measurements on the GPU: cached-decoder tokens/s against the recompute path, and kernel times of the skinny GEMM
(against the training GEMM, ``ops.linear_fwd``) and of decode attention, with achieved bytes/s as a share of the H100 SXM's
3.35 TB/s. Prints one JSON document (card name and power limit read in the same run).

    python scripts/decode_bench.py [--quick] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

HBM_BYTES_S = 3.35e12
MODELS = {"mpt-125m": dict(d_model=768, n_heads=12, n_layers=12), "mpt-1b": dict(d_model=2048, n_heads=16, n_layers=24)}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().splitlines() or ["?, ?, ?"])[0].split(", ")
    return {"name": name, "power_limit": power, "max_sm_clock": clk, "torch_device": torch.cuda.get_device_name(0)}


def time_kernel(fn, iters: int = 50, warmup: int = 5) -> float:
    """Mean seconds per call by CUDA events over ``iters`` launches after ``warmup``."""
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


def gemm_rows(dev, quick: bool) -> list[dict]:
    from photon_b200 import ops

    out = []
    for model, m in MODELS.items():
        d = m["d_model"]
        shapes = {"qkv": (3 * d, d), "out_proj": (d, d), "up": (4 * d, d), "down": (d, 4 * d), "lm_head": (50368, d)}
        for name, (N, K) in shapes.items():
            w = torch.randn(N, K, device=dev).bfloat16()
            for M in ((1, 16, 128) if quick else (1, 4, 16, 64, 128)):
                x = torch.randn(M, K, device=dev).bfloat16()
                y = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
                nbytes = 2 * (N * K + M * K + M * N)
                row = {"model": model, "gemm": name, "M": M, "N": N, "K": K, "bytes": nbytes}
                t_ref = time_kernel(lambda: ops.linear_fwd(x, w, None, y))
                row.update(linear_fwd_us=t_ref * 1e6, linear_fwd_hbm_share=nbytes / t_ref / HBM_BYTES_S)
                if M <= 64:
                    t = time_kernel(lambda: ops.skinny_gemm(x, w, y))
                    row.update(skinny_us=t * 1e6, skinny_hbm_share=nbytes / t / HBM_BYTES_S, skinny_speedup=t_ref / t)
                out.append(row)
    return out


def attention_rows(dev) -> list[dict]:
    from photon_b200 import ops

    out = []
    for model, m in MODELS.items():
        H, dh = m["n_heads"], m["d_model"] // m["n_heads"]
        for B in (1, 16, 64):
            for n in (512, 2048):
                kc = torch.randn(B, H, 2048, dh, device=dev).bfloat16()
                vc = torch.randn_like(kc)
                q = torch.randn(B, 3 * H * dh, device=dev).bfloat16()
                pos = torch.full((B,), n - 1, dtype=torch.int32, device=dev)
                o = torch.empty(B, H * dh, dtype=torch.bfloat16, device=dev)
                t = time_kernel(lambda: ops.decode_attention(q, kc, vc, pos, o, H, 1.0 / math.sqrt(dh)))
                nbytes = 2 * B * H * n * dh * 2
                out.append({"model": model, "batch": B, "kv_len": n, "d_head": dh, "us": t * 1e6, "bytes": nbytes,
                            "hbm_share": nbytes / t / HBM_BYTES_S})
                del kc, vc
    return out


def decode_rows(dev, quick: bool, new_tokens: int = 64) -> list[dict]:
    from photon_b200.eval.icl import _RecomputeDecoder
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    out = []
    for model, m in MODELS.items():
        cfg = MPTConfig(max_seq_len=2048, vocab_size=50368, **m)
        eng = B200Engine(cfg, dev, "amp_bf16", seed=1)
        g = torch.Generator().manual_seed(0)
        for plen in ((512,) if quick else (512, 1800)):
            rec = _RecomputeDecoder(eng.logits, cfg.max_seq_len)
            prompt = torch.randint(0, cfg.vocab_size, (plen,), generator=g).tolist()
            rec.start([prompt], new_tokens)   # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rec.start([prompt], new_tokens)
            for _ in range(new_tokens - 1):
                rec.step()
            torch.cuda.synchronize()
            t_rec = time.perf_counter() - t0
            for B in ((1, 16) if quick else (1, 4, 16, 64)):
                prompts = [torch.randint(0, cfg.vocab_size, (plen,), generator=g).tolist() for _ in range(B)]
                dec = eng.decoder(B)
                dec.start(prompts, new_tokens)   # warm-up: buffers, kernel attributes, graph capture
                for _ in range(3):
                    dec.step()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dec.start(prompts, new_tokens)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                for _ in range(new_tokens - 1):
                    dec.step()
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                out.append({"model": model, "prompt": plen, "batch": B, "new_tokens": new_tokens,
                            "cached_tokens_per_s": B * new_tokens / (t2 - t0), "cached_prefill_s": t1 - t0,
                            "cached_step_ms": (t2 - t1) / (new_tokens - 1) * 1e3,
                            "recompute_tokens_per_s": new_tokens / t_rec, "recompute_batch": 1})
                dec.close()
                del dec
                torch.cuda.empty_cache()
        eng.close()
        del eng
        torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="fewer shapes")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "gemm": gemm_rows(dev, a.quick), "attention": attention_rows(dev), "decode": decode_rows(dev, a.quick)}
    text = json.dumps(res)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))
    print(text)


if __name__ == "__main__":
    main()
