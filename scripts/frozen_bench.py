"""Training-step time of partly frozen models (``fl.frozen_layers``): the sm_90a engine with the freeze list, the same engine
with nothing frozen, and the stock-PyTorch backend with the same freeze list (the path these runs took before the engine
covered freeze lists). One optimizer step = one microbatch of ``mb`` × 2048 tokens through ``Trainer.fit``, timed with CUDA
events after warm-up. Prints one JSON document (card name and power limit read in the same run).

    python scripts/frozen_bench.py [--steps 6] [--warmup 3] [--models mpt-125m,mpt-1b] [--out FILE]
"""
from __future__ import annotations

import argparse
import gc
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

SEQ = 2048
MODELS = {"mpt-125m": (dict(d_model=768, n_heads=12, n_layers=12), 32), "mpt-1b": (dict(d_model=2048, n_heads=16, n_layers=24), 8)}
TORCH = {k: "torch" for k in ("gemm", "attention", "norm", "loss", "optimizer")}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().splitlines() or ["?, ?, ?"])[0].split(", ")
    return {"name": name, "power_limit": power, "max_sm_clock": clk, "torch_device": torch.cuda.get_device_name(0)}


def freeze_lists(n_layers: int) -> dict[str, list[str] | None]:
    lower = ["transformer.wte.weight", "transformer.wpe.weight"] + [f"transformer.blocks.{i}." for i in range(n_layers // 2)]
    return {"none": None, "wte": ["transformer.wte.weight"], "emb+lower_half": lower,
            "all_but_last_block": ["transformer.wte.weight", "transformer.wpe.weight", "transformer.norm_f."]
            + [f"transformer.blocks.{i}." for i in range(n_layers - 1)]}


def expand(cfg, prefixes: list[str] | None) -> list[str] | None:
    """Exact names for the prefixes above (freeze lists take exact names)."""
    if prefixes is None:
        return None
    from photon_b200.models.mpt import MPTForCausalLM

    names = [n for n, _ in MPTForCausalLM(cfg, device="meta", init=False).named_parameters()]
    return [n for n in names if any(n == p or (p.endswith(".") and n.startswith(p)) for p in prefixes)]


def time_step(cfg, mb: int, kernels: dict, frozen: list[str] | None, steps: int, warmup: int) -> dict:
    from photon_b200.train.trainer import Trainer

    ids = torch.randint(0, cfg.vocab_size, (mb, SEQ)).pin_memory()

    class Loader:
        def __iter__(self):
            while True:
                yield {"input_ids": ids, "labels": ids}

    tr = Trainer(cfg, optimizer_cfg=dict(name="adopt", lr=6e-4, betas=[0.9, 0.9999], eps=1e-6, weight_decay=0.0),
                 scheduler_cfg=dict(name="constant_with_warmup", t_warmup="1ba"), train_loader=Loader(), global_train_batch_size=mb,
                 device_train_microbatch_size=mb, precision="amp_bf16", max_duration=f"{warmup + steps + 1}ba", grad_clip_norm=1.0,
                 device=torch.device("cuda", 0), kernels=kernels, seed=17, frozen_layers=frozen)
    kind = tr.state.backend.kind
    tr.fit(f"{warmup}ba")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    tr.fit(f"{warmup + steps}ba")
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    launches = int(getattr(tr.state.backend, "launches_per_microbatch", 0))
    loss = tr.loggers[0].data["loss/train/total"][-1][1]
    tr.close()
    del tr
    gc.collect()
    torch.cuda.empty_cache()
    return {"backend": kind, "step_ms": round(ms, 2), "tokens_per_s": round(mb * SEQ / ms * 1e3), "launches_per_microbatch": launches,
            "last_loss": round(float(loss), 4)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", default="mpt-125m,mpt-1b")
    ap.add_argument("--lists", default="none,wte,emb+lower_half,all_but_last_block", help="freeze lists to time (comma-separated)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frozen_bench.py measures on a CUDA device")
    from photon_b200.models.mpt import MPTConfig

    doc = {"card": card(), "seq_len": SEQ, "precision": "amp_bf16", "steps": args.steps, "warmup": args.warmup, "rows": []}
    for model in args.models.split(","):
        shape, mb = MODELS[model]
        cfg = MPTConfig(max_seq_len=SEQ, vocab_size=50368, **shape)
        unfrozen = time_step(cfg, mb, {}, None, args.steps, args.warmup)
        for name, prefixes in freeze_lists(cfg.n_layers).items():
            if name not in args.lists.split(","):
                continue
            frozen = expand(cfg, prefixes)
            row = {"model": model, "microbatch": mb, "frozen": name, "n_frozen": len(frozen or []), "engine_unfrozen": unfrozen}
            row["engine"] = unfrozen if frozen is None else time_step(cfg, mb, {}, frozen, args.steps, args.warmup)
            row["torch"] = time_step(cfg, mb, TORCH, frozen, args.steps, args.warmup)
            row["engine_vs_unfrozen"] = round(unfrozen["step_ms"] / row["engine"]["step_ms"], 3)
            row["engine_vs_torch"] = round(row["torch"]["step_ms"] / row["engine"]["step_ms"], 3)
            doc["rows"].append(row)
            print(json.dumps(row), flush=True)
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)


if __name__ == "__main__":
    main()
