"""Sliding-window attention (``attn_config.sliding_window_size``) against plain causal attention on one GPU.

1. Attention forward + backward kernel time at S = 2048 (d_head 64 with 12 heads, d_head 128 with 16 heads) for
   W = 256, 512 and 1024, and at S = 8192 for W = 1024, each beside the share of (query tile, key tile) pairs the window
   leaves the forward (128 x 128 tiles, computed from the shapes): the bound on the kernel speedup.
2. The MPT-125M and MPT-1B training microbatch (forward + backward on the engine, CUDA graph), W = 512 against off.
3. Decoding at a context of about 2000 tokens, W = 256 against off: the decode-attention kernels alone (MPT-1B heads, 8
   sequences), and one whole greedy step of MPT-125M (8 sequences, CUDA graph).

The two arms of every comparison alternate inside one run (other work shares the host). Prints one JSON line per row and
writes them, with the card's name and power limit, to ``--out``.

    python scripts/window_attention_bench.py --out /tmp/window_attention_bench.json
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from doc_attention_bench import card, time_ms  # noqa: E402

from photon_b200 import ops  # noqa: E402

DEV = torch.device("cuda", 0)
MODELS = {"mpt-125m": dict(d_model=768, n_heads=12, n_layers=12), "mpt-1b": dict(d_model=2048, n_heads=16, n_layers=24)}


def tile_pairs(S: int, W: int, tile: int = 128) -> int:
    """(query tile, key tile) pairs the causal forward visits per head; W < 0: no window."""
    n = S // tile
    return sum(qt + 1 - (max(0, qt * tile - W) // tile if W >= 0 else 0) for qt in range(n))


def _alternate(fns: dict, reps: int, iters: int) -> dict:
    for f in fns.values():   # warm-up: module load, smem attributes, graph capture
        time_ms(f, 3)
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            t[k].append(time_ms(f, iters))
    return {k: (statistics.median(v), max(v) - min(v)) for k, v in t.items()}


def kernel_rows(args) -> list[dict]:
    rows = []
    for S, B, windows in ((2048, args.batch, (256, 512, 1024)), (8192, max(1, args.batch // 4), (1024,))):
        for dh, H in ((64, 12), (128, 16)):
            d = H * dh
            g = torch.Generator(device="cpu").manual_seed(0)
            qkv = torch.randn(B, S, 3 * d, generator=g).to(DEV).bfloat16()
            dout = torch.randn(B, S, d, generator=g).to(DEV).bfloat16()
            out, lse = torch.empty(B, S, d, dtype=torch.bfloat16, device=DEV), torch.empty(B, H, S, device=DEV)
            dqkv, delta = torch.empty_like(qkv), torch.empty_like(lse)
            scale = 1.0 / math.sqrt(dh)

            def step(W: int) -> None:
                ops.attention_fwd(qkv, out, lse, H, scale, True, window=W)
                ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, window=W)

            res = _alternate({W: (lambda W=W: step(W)) for W in (-1, *windows)}, args.reps, args.iters)
            causal, spread = res[-1]
            for W in windows:
                ms, sp = res[W]
                rows.append({"table": "kernel", "d_head": dh, "heads": H, "batch": B, "seq": S, "window": W,
                             "tile_pairs": tile_pairs(S, W), "tile_pairs_causal": tile_pairs(S, -1),
                             "tile_bound": round(tile_pairs(S, -1) / tile_pairs(S, W), 3), "causal_ms": round(causal, 4),
                             "window_ms": round(ms, 4), "speedup": round(causal / ms, 3), "spread_causal_ms": round(spread, 4),
                             "spread_window_ms": round(sp, 4)})
                print(json.dumps(rows[-1]), flush=True)
            del qkv, dout, out, lse, dqkv, delta
            torch.cuda.empty_cache()
    return rows


def step_rows(args) -> list[dict]:
    from photon_b200.data.synthetic import synthetic_batch
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    rows, S, W = [], 2048, 512
    for name in args.models:
        b = args.step_batch[name]
        ids = torch.from_numpy(synthetic_batch(b, S, seed=1)).to(DEV)
        engines = {w: B200Engine(MPTConfig(**MODELS[name], max_seq_len=S, vocab_size=50368, attn_impl="flash", sliding_window_size=w),
                                 DEV, "amp_bf16", {}, seed=5) for w in (-1, W)}
        denom = float(b * (S - 1))
        res = _alternate({w: (lambda e=e: e.fwd_bwd(ids, denom)) for w, e in engines.items()}, args.reps, args.step_iters)
        (off, sp_off), (on, sp_on) = res[-1], res[W]
        rows.append({"table": "step", "model": name, "microbatch": b, "seq": S, "window": W, "off_ms": round(off, 3),
                     "window_ms": round(on, 3), "speedup": round(off / on, 3), "spread_off_ms": round(sp_off, 3),
                     "spread_window_ms": round(sp_on, 3), "launches_off": engines[-1].launches_per_microbatch,
                     "launches_window": engines[W].launches_per_microbatch})
        print(json.dumps(rows[-1]), flush=True)
        for w in list(engines):
            engines.pop(w).close()
        torch.cuda.empty_cache()
    return rows


def decode_rows(args) -> list[dict]:
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    rows, W, B, ctx = [], 256, 8, 2000
    # the decode-attention kernels alone: MPT-1B heads, one layer of an S_max = 2048 cache, every sequence at position ctx
    H, dh, S = 16, 128, 2048
    g = torch.Generator(device="cpu").manual_seed(0)
    kc, vc = (torch.randn(B, H, S, dh, generator=g).to(DEV).bfloat16() for _ in range(2))
    q = torch.randn(B, 3 * H * dh, generator=g).to(DEV).bfloat16()
    o = torch.empty(B, H * dh, dtype=torch.bfloat16, device=DEV)
    pos = torch.full((B,), ctx, dtype=torch.int32, device=DEV)
    res = _alternate({w: (lambda w=w: ops.decode_attention(q, kc, vc, pos, o, H, 1.0 / math.sqrt(dh), window=w)) for w in (-1, W)},
                     args.reps, 200)
    rows.append({"table": "decode_attention", "heads": H, "d_head": dh, "batch": B, "context": ctx + 1, "window": W,
                 "off_us": round(res[-1][0] * 1e3, 2), "window_us": round(res[W][0] * 1e3, 2),
                 "speedup": round(res[-1][0] / res[W][0], 3), "spread_off_us": round(res[-1][1] * 1e3, 2),
                 "spread_window_us": round(res[W][1] * 1e3, 2)})
    print(json.dumps(rows[-1]), flush=True)
    # one greedy step of MPT-125M with 8 prompts of ctx tokens (the cache and the step graph are the decoder's own)
    n_steps = 40
    decs = {}
    for w in (-1, W):
        cfg = MPTConfig(**MODELS["mpt-125m"], max_seq_len=S, vocab_size=50368, attn_impl="flash", sliding_window_size=w)
        eng = B200Engine(cfg, DEV, "amp_bf16", {}, seed=5)
        dec = eng.decoder(B)
        prompts = [torch.randint(0, 50368, (ctx,), generator=torch.Generator().manual_seed(i)).tolist() for i in range(B)]
        dec.start(prompts, n_steps + 2)
        dec.step()   # captures the step graph
        decs[w] = (eng, dec)
    t = {w: [] for w in decs}
    for _ in range(args.reps):   # alternating blocks of steps; every step extends the same sequences
        for w, (_, dec) in decs.items():
            t[w].append(time_ms(dec.step, n_steps // args.reps))
    (off, on) = (statistics.median(t[-1]), statistics.median(t[W]))
    rows.append({"table": "decode_step", "model": "mpt-125m", "batch": B, "context": ctx, "window": W, "off_ms": round(off, 4),
                 "window_ms": round(on, 4), "speedup": round(off / on, 3), "spread_off_ms": round(max(t[-1]) - min(t[-1]), 4),
                 "spread_window_ms": round(max(t[W]) - min(t[W]), 4)})
    print(json.dumps(rows[-1]), flush=True)
    for w in list(decs):
        decs.pop(w)[0].close()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8, help="rows of the S = 2048 kernel comparison (S = 8192 uses a quarter)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--step-iters", type=int, default=5)
    ap.add_argument("--models", nargs="*", default=["mpt-125m", "mpt-1b"])
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.step_batch = {"mpt-125m": 16, "mpt-1b": 4}   # two engines (window on / off) live at once
    if not torch.cuda.is_available():
        raise SystemExit("window_attention_bench.py measures on the GPU; no CUDA device here")
    info = card()
    print(json.dumps(info), flush=True)
    rows = kernel_rows(args)
    if not args.skip_steps:
        rows += step_rows(args)
    if not args.skip_decode:
        rows += decode_rows(args)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps({"card": info, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
