"""Feed-forward variants (``model.ffn_config``) at MPT-125M (d_model 768, microbatch 16 x 2048) and MPT-1B (d_model 2048,
microbatch 4 x 2048) shapes, three variants each:

* ``mptmlp_gelu``: the default block, ``down(gelu(up(x)))`` at F = 4 * d_model, on the sm_90a engine;
* ``mptglu_silu``: ``down(silu(gate(x)) * up(x))`` at the parameter-matched F (2048 for d_model 768, 5376 for d_model 2048:
  three F x d matrices instead of two 4d x d ones), on the sm_90a engine;
* ``mptglu_silu_torch``: the same gated block through the stock PyTorch backend (bf16 autocast, library GEMMs).

Two timings per variant: one training microbatch (``fwd_bwd``, every block, head and loss) and one FFN half of one block at
the microbatch's token count (the FFN GEMMs forward and backward with their epilogues and bias-gradient sums: the engine's
kernel sequence, or autograd through the PyTorch module). Variants are alternated inside every repeat, the spread of the
repeats is printed, and the card's name and power limit are read in the same run. Prints one JSON document.

    python scripts/ffn_bench.py [--repeats 3] [--models 125m,1b] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

S, V = 2048, 50368
MODELS = {"125m": dict(d_model=768, n_heads=12, n_layers=12, mb=16, glu_hidden=2048),
          "1b": dict(d_model=2048, n_heads=16, n_layers=24, mb=4, glu_hidden=5376)}
VARIANTS = ("mptmlp_gelu", "mptglu_silu", "mptglu_silu_torch")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().splitlines() or ["?, ?, ?"])[0].split(", ")
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def time_fn(fn, iters: int, warmup: int = 2) -> float:
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


def config(model: str, variant: str):
    from photon_b200.models.mpt import MPTConfig

    m = MODELS[model]
    kw = dict(d_model=m["d_model"], n_heads=m["n_heads"], n_layers=m["n_layers"], max_seq_len=S, vocab_size=V)
    if variant != "mptmlp_gelu":
        kw.update(ffn_type="mptglu", ffn_act="silu", ffn_hidden_size=m["glu_hidden"])
    return MPTConfig(**kw)


def backend(cfg, variant: str, dev):
    if variant.endswith("_torch"):
        from photon_b200.train.backend import TorchBackend

        return TorchBackend(cfg, dev, "amp_bf16", seed=0)
    from photon_b200.models.engine import B200Engine

    return B200Engine(cfg, dev, "amp_bf16", {}, seed=0)


def ffn_half(cfg, variant: str, T: int, dev):
    """One block's FFN forward + backward over T tokens (all weights trainable, input gradient computed)."""
    from photon_b200 import ops
    from photon_b200.models.mpt import MPTGLU, MPTMLP

    d, Fh = cfg.d_model, cfg.ffn_hidden
    g = torch.Generator(device=dev).manual_seed(0)
    bf = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.02).bfloat16()  # noqa: E731
    f32 = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
    ln, hmid, dh = bf(T, d), bf(T, d), bf(T, d)
    if variant.endswith("_torch"):
        ffn = (MPTGLU(cfg) if cfg.ffn_gated else MPTMLP(cfg)).to(dev)
        x = ln.float().requires_grad_(True)

        def run_torch():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = hmid + ffn(x)
            y.backward(dh)
        return run_torch
    wup, wdown, bup, bdown = bf(Fh, d), bf(d, Fh), f32(Fh), f32(d)
    dwup, dwdown, dbup, dbdown = f32(Fh, d), f32(d, Fh), f32(Fh), f32(d)
    u, z, dz, h, dln = bf(T, Fh), bf(T, Fh), bf(T, Fh), bf(T, d), bf(T, d)
    if not cfg.ffn_gated:
        def run_mlp():
            ops.linear_act_grad_fwd(cfg.ffn_act, ln, wup, bup, z, u)
            ops.linear_fwd(u, wdown, bdown, h, residual=hmid)
            ops.col_sum(dh, dbdown), ops.linear_wgrad(dh, u, dwdown), ops.linear_dgrad(dh, wdown, dz, mul=z)
            ops.col_sum(dz, dbup), ops.linear_wgrad(dz, ln, dwup), ops.linear_dgrad(dz, wup, dln)
        return run_mlp
    wg, bg, dwg, dbg = bf(Fh, d), f32(Fh), f32(Fh, d), f32(Fh)
    a, dg, tmp = bf(T, Fh), bf(T, Fh), bf(T, d)

    def run_glu():
        ops.linear_act_grad_fwd(cfg.ffn_act, ln, wg, bg, dz, a)
        ops.linear_glu_up_fwd(ln, wup, bup, a, dz, u, z)
        ops.linear_fwd(u, wdown, bdown, h, residual=hmid)
        ops.col_sum(dh, dbdown), ops.linear_wgrad(dh, u, dwdown), ops.linear_glu_dgrad(dh, wdown, a, z, dz, dg)
        ops.col_sum(dz, dbup), ops.linear_wgrad(dz, ln, dwup), ops.col_sum(dg, dbg), ops.linear_wgrad(dg, ln, dwg)
        ops.linear_dgrad(dg, wg, tmp), ops.linear_dgrad(dz, wup, dln, residual=tmp)
    return run_glu


def spread(v: list[float]) -> dict:
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--models", default="125m,1b")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ffn_bench.py measures on the GPU; there is none here")
    dev = torch.device("cuda", 0)
    res: dict = {"card": card(), "seq": S, "variants": list(VARIANTS)}
    for model in a.models.split(","):
        m = MODELS[model]
        T = m["mb"] * S
        cfgs = {v: config(model, v) for v in VARIANTS}
        out: dict = {"microbatch": [m["mb"], S], "ffn_hidden": {v: c.ffn_hidden for v, c in cfgs.items()},
                     "num_params": {v: c.num_params() for v, c in cfgs.items()}}
        halves = {v: ffn_half(cfgs[v], v, T, dev) for v in VARIANTS}
        t_half: dict = {v: [] for v in VARIANTS}
        for _ in range(a.repeats):
            for v in VARIANTS:   # alternated inside every repeat
                t_half[v].append(time_fn(halves[v], 10) * 1e3)
        del halves
        torch.cuda.empty_cache()
        backends = {v: backend(cfgs[v], v, dev) for v in VARIANTS}
        ids = torch.randint(0, V, (m["mb"], S), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        denom = float(ids.numel())
        t_train: dict = {v: [] for v in VARIANTS}
        for _ in range(a.repeats):
            for v, be in backends.items():
                t_train[v].append(time_fn(lambda b=be: b.fwd_bwd(ids, denom), 3, warmup=2) * 1e3)
                be.close()          # one workspace at a time (the parameters stay resident)
                torch.cuda.empty_cache()
        del backends
        torch.cuda.empty_cache()
        out["ffn_half_fwd_bwd_ms"] = {v: spread(t) for v, t in t_half.items()}
        out["train_microbatch_ms"] = {v: spread(t) for v, t in t_train.items()}
        res[model] = out
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
