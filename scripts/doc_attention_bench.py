"""Document-masked attention (``attn_config.attn_uses_sequence_id``) against plain causal attention on one GPU.

1. Attention forward + backward kernel time at S = 2048 (d_head 64 with 12 heads, d_head 128 with 16 heads) for three
   document layouts: the EOS positions of the synthetic C4 stream (log-normal lengths, median ~400 tokens), one document per
   row (the cost of the mask path itself) and 128-token documents (the most tiles skipped).
2. The MPT-125M and MPT-1B training microbatch (forward + backward on the engine, CUDA graph) on synthetic C4 batches with
   ``eos_token_id = 0``, flag on and off.

The two arms of every comparison alternate inside one run (other work shares the host). Prints one JSON line per row and
writes them, with the card's name and power limit, to ``--out``.

    python scripts/doc_attention_bench.py --out /tmp/doc_attention_bench.json
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

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from photon_b200 import ops  # noqa: E402
from photon_b200.data.streaming import sequence_ids  # noqa: E402
from photon_b200.data.synthetic import EOS_ID, synthetic_batch  # noqa: E402

DEV = torch.device("cuda", 0)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = ([s.strip() for s in q.stdout.strip().split(",")] + ["?", "?", "?"])[:3] if q.returncode == 0 else ("?", "?", "?")
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit": power, "max_sm_clock": clock}


def layout_ids(name: str, B: int, S: int) -> torch.Tensor:
    if name == "c4":
        ids = torch.from_numpy(synthetic_batch(B, S, seed=0))
        return sequence_ids(ids, eos_token_id=EOS_ID)
    if name == "one":
        return torch.zeros(B, S, dtype=torch.int64)
    if name == "doc128":
        return (torch.arange(S) // 128).repeat(B, 1)
    raise ValueError(name)


def live_tile_fraction(sid: torch.Tensor, tile: int = 128) -> float:
    """Key tiles the masked forward loads over those the causal forward loads (128 x 128 tiles)."""
    B, S = sid.shape
    n = S // tile
    causal = B * n * (n + 1) // 2
    live = 0
    for b in range(B):
        row = sid[b]
        for qt in range(n):
            first = int((row == row[qt * tile]).nonzero()[0])      # ids are runs: the document's first row
            live += qt + 1 - first // tile
    return live / causal


def time_ms(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def kernel_rows(args) -> list[dict]:
    rows = []
    B, S = args.batch, 2048
    for dh, H in ((64, 12), (128, 16)):
        d = H * dh
        g = torch.Generator(device="cpu").manual_seed(0)
        qkv = torch.randn(B, S, 3 * d, generator=g).to(DEV).bfloat16()
        dout = torch.randn(B, S, d, generator=g).to(DEV).bfloat16()
        out, lse = torch.empty(B, S, d, dtype=torch.bfloat16, device=DEV), torch.empty(B, H, S, device=DEV)
        dqkv, delta = torch.empty_like(qkv), torch.empty_like(lse)
        ds, de = torch.empty(B * S, dtype=torch.int32, device=DEV), torch.empty(B * S, dtype=torch.int32, device=DEV)
        scale = 1.0 / math.sqrt(dh)
        for lay in ("c4", "one", "doc128"):
            sid = layout_ids(lay, B, S)
            ops.doc_bounds(sid.to(DEV), ds, de)

            def step(doc: bool) -> None:
                ops.attention_fwd(qkv, out, lse, H, scale, True, None, ds if doc else None)
                ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, scale, True, None, ds if doc else None, de if doc else None)

            for doc in (False, True):   # warm-up: module load, smem attributes
                time_ms(lambda: step(doc), 3)
            t = {False: [], True: []}
            for _ in range(args.reps):
                for doc in (False, True):
                    t[doc].append(time_ms(lambda: step(doc), args.iters))
            causal, masked = statistics.median(t[False]), statistics.median(t[True])
            rows.append({"table": "kernel", "d_head": dh, "heads": H, "batch": B, "seq": S, "layout": lay,
                         "live_tiles": round(live_tile_fraction(sid), 4), "causal_ms": round(causal, 4), "doc_ms": round(masked, 4),
                         "speedup": round(causal / masked, 3), "spread_causal_ms": round(max(t[False]) - min(t[False]), 4),
                         "spread_doc_ms": round(max(t[True]) - min(t[True]), 4)})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def step_rows(args) -> list[dict]:
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    models = {"mpt-125m": dict(d_model=768, n_heads=12, n_layers=12), "mpt-1b": dict(d_model=2048, n_heads=16, n_layers=24)}
    rows = []
    S = 2048
    for name in args.models:
        b = args.step_batch[name]
        ids_host = torch.from_numpy(synthetic_batch(b, S, seed=1))
        sid = sequence_ids(ids_host, eos_token_id=EOS_ID).to(DEV)
        ids = ids_host.to(DEV)
        engines = {}
        for on in (False, True):
            cfg = MPTConfig(**models[name], max_seq_len=S, vocab_size=50368, attn_impl="flash", attn_uses_sequence_id=on)
            engines[on] = B200Engine(cfg, DEV, "amp_bf16", {}, seed=5)
        denom = float(b * (S - 1))
        kw = {False: {}, True: {"sequence_id": sid}}
        for on in (False, True):   # capture + warm-up
            for _ in range(2):
                engines[on].fwd_bwd(ids, denom, **kw[on])
        torch.cuda.synchronize()
        t = {False: [], True: []}
        for _ in range(args.reps):
            for on in (False, True):
                t[on].append(time_ms(lambda: engines[on].fwd_bwd(ids, denom, **kw[on]), args.step_iters))
        off, on_ = statistics.median(t[False]), statistics.median(t[True])
        rows.append({"table": "step", "model": name, "microbatch": b, "seq": S, "live_tiles": round(live_tile_fraction(sid.cpu()), 4),
                     "flag_off_ms": round(off, 3), "flag_on_ms": round(on_, 3), "speedup": round(off / on_, 3),
                     "spread_off_ms": round(max(t[False]) - min(t[False]), 3), "spread_on_ms": round(max(t[True]) - min(t[True]), 3),
                     "launches_off": engines[False].launches_per_microbatch, "launches_on": engines[True].launches_per_microbatch})
        print(json.dumps(rows[-1]), flush=True)
        for on in list(engines):
            engines.pop(on).close()
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8, help="rows of the kernel comparison")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--step-iters", type=int, default=5)
    ap.add_argument("--models", nargs="*", default=["mpt-125m", "mpt-1b"])
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.step_batch = {"mpt-125m": 16, "mpt-1b": 4}   # two engines (flag on / off) live at once
    if not torch.cuda.is_available():
        raise SystemExit("doc_attention_bench.py measures on the GPU; no CUDA device here")
    info = card()
    print(json.dumps(info), flush=True)
    rows = kernel_rows(args)
    if not args.skip_steps:
        rows += step_rows(args)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps({"card": info, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
