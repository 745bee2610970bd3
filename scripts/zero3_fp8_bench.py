"""Full parameter sharding (``kernels.param_sharding=zero3``): amp_bf16 against amp_fp8 on the same model, in one invocation,
alternating the two arms after warm-up. One optimizer step = one microbatch of ``mb`` × 2048 tokens through ``Trainer.fit``, timed
with CUDA events. Also reported: the requantisation kernel's time (CUDA events around ``NvlZero3Comm.requantize``, which runs once
per optimizer step), the bytes one block pull moves (from the sharding plan: E4M3 = one byte per element) and peak memory (the
torch allocator's peak plus the symmetric arena, which is allocated outside it). Prints one JSON document; the card name and
power limit are read in the same run.

    python scripts/zero3_fp8_bench.py [--models mpt-1b,mpt-3b] [--steps 4] [--warmup 2] [--rounds 2] [--out FILE]
    torchrun --nproc-per-node N scripts/zero3_fp8_bench.py --models mpt-7b      # N ranks, one GPU each
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

SEQ = 2048
MODELS = {"mpt-1b": (dict(d_model=2048, n_heads=16, n_layers=24), 8), "mpt-3b": (dict(d_model=2560, n_heads=20, n_layers=32), 2),
          "mpt-7b": (dict(d_model=4096, n_heads=32, n_layers=32), 2)}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().splitlines() or ["?, ?, ?"])[0].split(", ")
    return {"name": name, "power_limit": power, "max_sm_clock": clk, "torch_device": torch.cuda.get_device_name(0)}


def gather_bytes(plan) -> dict:
    """Bytes one rank pulls per block unit (bf16 vs E4M3) and per microbatch (every block twice: forward and backward)."""
    blocks = [u.per * plan.world_size for u in plan.units[:-1]]
    return {"block_params": blocks[0], "per_block_pull_bf16": 2 * blocks[0], "per_block_pull_e4m3": blocks[0],
            "per_microbatch_bf16": 2 * 2 * sum(blocks), "per_microbatch_e4m3": 2 * sum(blocks)}


def time_arm(cfg, mb: int, precision: str, steps: int, warmup: int, rank: int, world: int, dev: torch.device) -> dict:
    from photon_b200.parallel.zero3 import NvlZero3Comm
    from photon_b200.train.trainer import Trainer
    from photon_b200.utils.flat import layout_for_model_cfg

    mc = {"name": "mpt_causal_lm", "d_model": cfg.d_model, "n_heads": cfg.n_heads, "n_layers": cfg.n_layers, "expansion_ratio": 4,
          "max_seq_len": SEQ, "vocab_size": cfg.vocab_size}
    torch.cuda.reset_peak_memory_stats(dev)
    comm = NvlZero3Comm(layout_for_model_cfg(mc), cfg.n_layers, rank=rank, world_size=world, device=dev, fp8=precision == "amp_fp8")
    g = torch.Generator().manual_seed(rank)
    ids = torch.randint(0, cfg.vocab_size, (mb, SEQ), generator=g).pin_memory()

    class Loader:
        def __iter__(self):
            while True:
                yield {"input_ids": ids, "labels": ids}

    tr = Trainer(cfg, optimizer_cfg=dict(name="decoupled_adamw", lr=6e-4, betas=[0.9, 0.95], eps=1e-8, weight_decay=0.0),
                 scheduler_cfg=dict(name="constant_with_warmup", t_warmup="1ba"), train_loader=Loader(), global_train_batch_size=mb * world,
                 device_train_microbatch_size=mb, precision=precision, max_duration=f"{warmup + steps + 1}ba", grad_clip_norm=1.0,
                 device=dev, seed=17, grad_comm=comm, rank=rank, world_size=world)
    tr.fit(f"{warmup}ba")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    a.record()
    tr.fit(f"{warmup + steps}ba")
    b.record()
    torch.cuda.synchronize(dev)
    ms = a.elapsed_time(b) / steps
    row = {"precision": precision, "step_ms": round(ms, 2), "tokens_per_s": round(world * mb * SEQ / ms * 1e3),
           "last_loss": round(float(tr.loggers[0].data["loss/train/total"][-1][1]), 4),
           "peak_torch_gib": round(torch.cuda.max_memory_allocated(dev) / 2**30, 2), "arena_gib": round(comm.arena.nbytes / 2**30, 2)}
    if precision == "amp_fp8":
        n = 5
        comm.before_param_write()
        a.record()
        for _ in range(n):
            comm.requantize()
        b.record()
        comm.params_changed()
        torch.cuda.synchronize(dev)
        row["requant_ms"] = round(a.elapsed_time(b) / n, 3)
    tr.close()
    comm.close()
    del tr, comm
    gc.collect()
    torch.cuda.empty_cache()
    return row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="mpt-1b,mpt-3b")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="bf16 / fp8 pairs per model, alternating")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("zero3_fp8_bench.py measures on a CUDA device")
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.parallel.zero3 import UnitPlan
    from photon_b200.utils.flat import layout_for_model_cfg

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)
    doc = {"card": card(), "world_size": world, "seq_len": SEQ, "steps": args.steps, "warmup": args.warmup, "rows": []}
    for model in args.models.split(","):
        shape, mb = MODELS[model]
        cfg = MPTConfig(max_seq_len=SEQ, vocab_size=50368, **shape)
        mc = {"name": "mpt_causal_lm", "expansion_ratio": 4, "max_seq_len": SEQ, "vocab_size": 50368, **shape}
        row = {"model": model, "microbatch": mb, "gather_bytes": gather_bytes(UnitPlan(layout_for_model_cfg(mc), shape["n_layers"], world)),
               "amp_bf16": [], "amp_fp8": []}
        for _ in range(args.rounds):
            for prec in ("amp_bf16", "amp_fp8"):
                row[prec].append(time_arm(cfg, mb, prec, args.steps, args.warmup, rank, world, dev))
        best = {p: min(r["step_ms"] for r in row[p]) for p in ("amp_bf16", "amp_fp8")}
        row["fp8_speedup"] = round(best["amp_bf16"] / best["amp_fp8"], 3)
        doc["rows"].append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
    if rank == 0:
        text = json.dumps(doc, indent=1)
        print(text)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text(text)
    if world > 1:
        import torch.distributed as dist

        dist.destroy_process_group()


if __name__ == "__main__":
    main()
