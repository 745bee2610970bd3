"""Scoring measurements on the GPU: questions/s of ``KVDecoder.score`` (at task batch sizes 4 and 16) against the evaluator's
pair-at-a-time path (``engine.logits``, one (context, continuation) pair per call), on seeded random weights and tokens with
mpt-125m and mpt-1b shapes; and ``cache_attention`` against ``attention_fwd`` at equal query rows and keys, with achieved
TFLOP/s. Both scoring arms run on the same questions in the same run, and their per-pair log-likelihoods must agree within
the bf16 tolerance. Prints one JSON document (card name and power limit read in the same run).

    python scripts/score_bench.py [--quick] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from decode_bench import MODELS, card, time_kernel  # noqa: E402

# workload: (context tokens, choices, scored tokens per choice)
WORKLOADS = {"0-shot": (64, 4, 8), "few-shot": (1024, 4, 1), "hellaswag-like": (512, 4, 24), "LM": (512, 1, 4)}
LOGP_TOL = 0.15   # per scored token: both arms compute in bf16


def _sync_time(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def score_rows(dev, quick: bool) -> list[dict]:
    from photon_b200.eval.icl import ICLEvaluator
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    out = []
    n_q = 16 if quick else 32
    for model, m in MODELS.items():
        cfg = MPTConfig(max_seq_len=2048, vocab_size=50368, **m)
        eng = B200Engine(cfg, dev, "amp_bf16", seed=1)
        ev = ICLEvaluator(eng.logits, None, cfg.max_seq_len)
        g = torch.Generator().manual_seed(0)
        rnd = lambda n: torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist()  # noqa: E731
        for name, (ctx_len, n_ch, n_tok) in WORKLOADS.items():
            questions = []
            for _ in range(n_q):
                ctx = rnd(ctx_len)
                questions.append([(ctx, rnd(n_tok)) for _ in range(n_ch)])
            ev._continuation_stats(*questions[0][0])   # warm-up
            old: list[list[tuple[float, bool]]] = []
            t_old = _sync_time(lambda: old.extend([ev._continuation_stats(c, s) for c, s in q] for q in questions))
            row = {"model": model, "workload": name, "context": ctx_len, "choices": n_ch, "scored_tokens": n_tok, "questions": n_q,
                   "pairwise_questions_per_s": n_q / t_old}
            for bs in (4, 16):
                dec = eng.decoder(bs * n_ch)
                batches = [[p for q in questions[lo: lo + bs] for p in q] for lo in range(0, n_q, bs)]
                dec.score(batches[0])   # warm-up: cache, kernel attributes
                new: list[tuple[float, bool]] = []
                t_new = _sync_time(lambda dec=dec, batches=batches, new=new: [new.extend(dec.score(b)) for b in batches])
                worst = max(abs(a[0] - b[0]) / n_tok for a, b in zip(new, [s for q in old for s in q]))
                assert worst <= LOGP_TOL, (model, name, bs, worst)
                row[f"score_bs{bs}_questions_per_s"] = n_q / t_new
                row[f"score_bs{bs}_speedup"] = t_old / t_new
                row[f"score_bs{bs}_max_logp_diff_per_token"] = worst
                dec.close()
                del dec
                torch.cuda.empty_cache()
            out.append(row)
        eng.close()
        del eng, ev
        torch.cuda.empty_cache()
    return out


def attention_rows(dev) -> list[dict]:
    """cache_attention over S query rows of one slot from position 0 (the causal S x S problem of attention_fwd), and at
    scoring shapes (rows of several slots after a prefix), with useful FLOP/s (masked keys not counted)."""
    from photon_b200 import ops

    out = []
    for model, m in MODELS.items():
        H, dh = m["n_heads"], m["d_model"] // m["n_heads"]
        d = H * dh
        scale = 1.0 / math.sqrt(dh)
        for S in (512, 1024, 2048):
            qkv = torch.randn(1, S, 3 * d, device=dev).bfloat16()
            o = torch.empty(1, S, d, dtype=torch.bfloat16, device=dev)
            lse = torch.empty(1, H, S, device=dev)
            kc = qkv.view(S, 3, H, dh)[:, 1].transpose(0, 1).contiguous().unsqueeze(0)
            vc = qkv.view(S, 3, H, dh)[:, 2].transpose(0, 1).contiguous().unsqueeze(0)
            tiles = ops.cache_tiles([(0, 0, S, 0)], dev)
            o2 = torch.empty(S, d, dtype=torch.bfloat16, device=dev)
            flops = 4.0 * H * dh * S * (S + 1) / 2
            t_ref = time_kernel(lambda: ops.attention_fwd(qkv, o, lse, H, scale, True))
            t = time_kernel(lambda: ops.cache_attention(qkv[0], kc, vc, tiles, o2, H, scale))
            torch.testing.assert_close(o2.float(), o[0].float(), rtol=2e-2, atol=2e-2)
            out.append({"model": model, "shape": f"causal {S}x{S}", "query_rows": S, "d_head": dh,
                        "attention_fwd_us": t_ref * 1e6, "attention_fwd_tflops": flops / t_ref / 1e12,
                        "cache_attention_us": t * 1e6, "cache_attention_tflops": flops / t / 1e12})
        for slots, rows, prefix in ((16, 24, 512), (64, 8, 64), (16, 1, 1024)):
            kc = torch.randn(slots, H, 2048, dh, device=dev).bfloat16()
            vc = torch.randn_like(kc)
            qkv = torch.randn(slots * rows, 3 * d, device=dev).bfloat16()
            o2 = torch.empty(slots * rows, d, dtype=torch.bfloat16, device=dev)
            tiles = ops.cache_tiles([(s, s * rows, rows, prefix) for s in range(slots)], dev)
            flops = 4.0 * H * dh * slots * sum(prefix + i + 1 for i in range(rows))
            t = time_kernel(lambda: ops.cache_attention(qkv, kc, vc, tiles, o2, H, scale))
            out.append({"model": model, "shape": f"{slots} slots x {rows} rows after {prefix}", "query_rows": slots * rows, "d_head": dh,
                        "cache_attention_us": t * 1e6, "cache_attention_tflops": flops / t / 1e12})
            del kc, vc
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="fewer questions")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "attention": attention_rows(dev), "score": score_rows(dev, a.quick)}
    text = json.dumps(res)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))
    print(text)


if __name__ == "__main__":
    main()
