"""RMSNorm against LayerNorm on the sm_90a kernels (``model.norm_type``).

Kernels, at T = 16384 rows and d = 768, 2048, 2560 and 4096, RMSNorm and LayerNorm alternated inside every repeat:

* ``fwd``: bf16 x -> bf16 y, row statistics saved (``rmsnorm_fwd`` / ``layernorm_fwd``, LayerNorm with beta);
* ``fwd_q8``: the same, written as E4M3 (``rmsnorm_fwd_q8`` / ``layernorm_fwd_q8``), the amp_fp8 block norms;
* ``bwd``: dx with the residual gradient added, and dgamma (and a LayerNorm's dbeta): one pass up to d = 1024, a dx kernel
  and a column reduction above.

Each kernel's rate is the bytes it must move (the one-pass minimum: the bf16 rows read and written, the fp32 row statistics;
the split backward reads dy and x a second time on top) over its time, also as a share of the H100 SXM's 3.35 TB/s.

Training, one ``fwd_bwd`` microbatch on the engine at MPT-125M (16 x 2048) and MPT-1B (4 x 2048) shapes, norm_type layernorm
against rmsnorm, alternated. The spread of the repeats is printed and the card's name and power limit are read in the same
run. Prints one JSON document.

    python scripts/norm_bench.py [--repeats 5] [--models 125m,1b] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from ffn_bench import card, spread, time_fn  # noqa: E402

T_ROWS = 16384
DS = (768, 2048, 2560, 4096)
HBM = 3.35e12
S, V = 2048, 50368
MODELS = {"125m": dict(d_model=768, n_heads=12, n_layers=12, mb=16), "1b": dict(d_model=2048, n_heads=16, n_layers=24, mb=4)}
NORMS = ("layernorm", "rmsnorm")


def kernel_cases(d: int, dev: torch.device) -> dict:
    """{(op, norm): (callable, bytes)} for one row length."""
    from photon_b200 import ops

    T = T_ROWS
    g = torch.Generator(device=dev).manual_seed(d)
    x, dy, dres = ((torch.randn(T, d, device=dev, generator=g)).bfloat16() for _ in range(3))
    gamma, beta = torch.rand(d, device=dev, generator=g) + 0.5, torch.randn(d, device=dev, generator=g) * 0.1
    y, dx = torch.empty_like(x), torch.empty_like(x)
    y8 = torch.empty(T, d, dtype=torch.uint8, device=dev)
    mean, rstd = torch.empty(T, device=dev), torch.empty(T, device=dev)
    dg, db = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
    meta = torch.ones(3, 2, device=dev)
    ops.layernorm_fwd(x, gamma, beta, y, mean, rstd)   # valid statistics for the backward
    row = 2 * T * d
    return {
        ("fwd", "layernorm"): (lambda: ops.layernorm_fwd(x, gamma, beta, y, mean, rstd), 2 * row + 8 * T),
        ("fwd", "rmsnorm"): (lambda: ops.rmsnorm_fwd(x, gamma, y, rstd), 2 * row + 4 * T),
        ("fwd_q8", "layernorm"): (lambda: ops.layernorm_fwd_q8(x, gamma, beta, y8, mean, rstd, 1e-5, meta, 0), row + T * d + 8 * T),
        ("fwd_q8", "rmsnorm"): (lambda: ops.rmsnorm_fwd_q8(x, gamma, y8, rstd, 1e-5, meta, 0), row + T * d + 4 * T),
        ("bwd", "layernorm"): (lambda: ops.layernorm_bwd(dy, x, gamma, mean, rstd, dres, dx, dg, db), 4 * row + 8 * T),
        ("bwd", "rmsnorm"): (lambda: ops.rmsnorm_bwd(dy, x, gamma, rstd, dres, dx, dg), 4 * row + 4 * T),
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--models", default="125m,1b")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("norm_bench.py measures on the GPU; there is none here")
    dev = torch.device("cuda", 0)
    res: dict = {"card": card(), "rows": T_ROWS, "hbm_bytes_per_s": HBM, "kernels": {}}
    for d in DS:
        cases = kernel_cases(d, dev)
        times: dict = {k: [] for k in cases}
        for _ in range(a.repeats):
            for k, (fn, _) in cases.items():   # RMSNorm and LayerNorm alternated inside every repeat
                times[k].append(time_fn(fn, 50, warmup=5) * 1e6)
        out: dict = {}
        for (op, norm), t in times.items():
            sp = spread(t)
            nbytes = cases[(op, norm)][1]
            gbs = nbytes / (sp["median"] * 1e-6) / 1e9
            out.setdefault(op, {})[norm] = {"us": sp, "bytes": nbytes, "GB_per_s": round(gbs, 1), "share_of_hbm": round(gbs * 1e9 / HBM, 3)}
        res["kernels"][str(d)] = out
        del cases
        torch.cuda.empty_cache()
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    for model in a.models.split(","):
        m = MODELS[model]
        engines = {n: B200Engine(MPTConfig(d_model=m["d_model"], n_heads=m["n_heads"], n_layers=m["n_layers"], max_seq_len=S,
                                           vocab_size=V, norm_type=n), dev, "amp_bf16", {}, seed=0) for n in NORMS}
        ids = torch.randint(0, V, (m["mb"], S), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        denom = float(ids.numel())
        t: dict = {n: [] for n in NORMS}
        for _ in range(a.repeats):
            for n, e in engines.items():
                t[n].append(time_fn(lambda e=e: e.fwd_bwd(ids, denom), 3, warmup=2) * 1e3)
                e.close()           # one workspace at a time (the parameters stay resident)
                torch.cuda.empty_cache()
        res[model] = {"microbatch": [m["mb"], S], "train_microbatch_ms": {n: spread(v) for n, v in t.items()},
                      "launches_per_microbatch": {n: e.launches_per_microbatch for n, e in engines.items()}}
        del engines
        torch.cuda.empty_cache()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
