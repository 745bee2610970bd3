"""The LM head's logit transform and an untied head on the sm_90a engine (``logit_scale``, ``final_logit_softcapping``,
``tie_word_embeddings``).

Kernel: the fused cross-entropy at the engine's head chunk, 16 896 rows x V = 50 368 (the shared-memory kernel), training (the
gradient written back), without the transform, with a scale, and with a scale and a cap of 30, alternated inside every repeat.
The bytes it must move are one read and one write of the bf16 row; their time at the H100 SXM's 3.35 TB/s over the kernel time is
its bytes-bound share.

Training, one ``fwd_bwd`` microbatch on the engine at MPT-125M (16 x 2048) and MPT-1B (4 x 2048) shapes: tied head against an
untied head with ``logit_scale: inv_sqrt_d_model`` and ``final_logit_softcapping: 30``, alternated. The card's name and power
limit are read in the same run. Prints one JSON document.

    python scripts/head_bench.py [--repeats 5] [--models 125m,1b] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

from ffn_bench import card, spread, time_fn  # noqa: E402

ROWS, V, S = 16896, 50368, 2048
HBM = 3.35e12
MODELS = {"125m": dict(d_model=768, n_heads=12, n_layers=12, mb=16), "1b": dict(d_model=2048, n_heads=16, n_layers=24, mb=4)}
TRANSFORMS = {"none": (None, None), "scale": (1 / math.sqrt(768), None), "scale_cap30": (1 / math.sqrt(768), 30.0)}
HEADS = {"tied": {}, "untied_scale_cap30": dict(tie_word_embeddings=False, logit_scale="inv_sqrt_d_model", final_logit_softcapping=30.0)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--models", default="125m,1b")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_bench.py measures on the GPU; there is none here")
    from photon_b200 import ops

    dev = torch.device("cuda", 0)
    res: dict = {"card": card(), "ce_rows": ROWS, "vocab": V, "hbm_bytes_per_s": HBM}
    g = torch.Generator(device=dev).manual_seed(0)
    src = (torch.randn(ROWS, V, device=dev, generator=g) * 4).bfloat16()
    work = torch.empty_like(src)
    tgt = torch.randint(0, V, (ROWS,), device=dev, generator=g)
    stats = torch.zeros(4, dtype=torch.float64, device=dev)
    nbytes = 2 * src.numel() * 2   # one read and one write of the bf16 logits
    copy_t = []
    t: dict = {k: [] for k in TRANSFORMS}
    for _ in range(a.repeats):
        copy_t.append(time_fn(lambda: work.copy_(src), 10, warmup=2) * 1e3)
        for k, (s, c) in TRANSFORMS.items():
            # the kernel overwrites its input with the gradient: refresh it before each call (the copy is timed on its own)
            t[k].append(time_fn(lambda s=s, c=c: (work.copy_(src), ops.cross_entropy(work, tgt, 1e-4, True, stats, None, None, s, c)),
                                10, warmup=2) * 1e3 - copy_t[-1])
    bound_ms = nbytes / HBM * 1e3
    res["cross_entropy_ms"] = {k: {**spread(v), "bytes": nbytes, "bytes_bound_share": round(bound_ms / spread(v)["median"], 3)}
                               for k, v in t.items()}
    res["refresh_copy_ms"] = spread(copy_t)
    del src, work
    torch.cuda.empty_cache()

    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    for model in a.models.split(","):
        m = MODELS[model]
        engines = {h: B200Engine(MPTConfig(d_model=m["d_model"], n_heads=m["n_heads"], n_layers=m["n_layers"], max_seq_len=S,
                                           vocab_size=V, **kw), dev, "amp_bf16", {}, seed=0) for h, kw in HEADS.items()}
        ids = torch.randint(0, V, (m["mb"], S), device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        denom = float(ids.numel())
        tm: dict = {h: [] for h in HEADS}
        for _ in range(a.repeats):
            for h, e in engines.items():
                tm[h].append(time_fn(lambda e=e: e.fwd_bwd(ids, denom), 3, warmup=2) * 1e3)
                e.close()
                torch.cuda.empty_cache()
        res[model] = {"microbatch": [m["mb"], S], "train_microbatch_ms": {h: spread(v) for h, v in tm.items()},
                      "launches_per_microbatch": {h: e.launches_per_microbatch for h, e in engines.items()}}
        del engines
        torch.cuda.empty_cache()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
