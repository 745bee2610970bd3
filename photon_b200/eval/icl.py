"""In-context-learning evaluation + Eval Gauntlet aggregation.

The reference gets these from llm-foundry (``build_evaluators`` / ``EvalGauntlet``; wired at
photon/centralised_train.py:120-136 and photon/clients/trainer_utils.py) and ships only the task
tables (``conf/icl_tasks_config/*.yaml``, ``conf/eval_gauntlet_config/*.yaml``).  This module is a
self-contained implementation of the two task types that dominate those tables:

* ``language_modeling``   — exact-match of the greedy continuation (teacher-forced argmax);
* ``multiple_choice``     — pick the choice with the highest length-normalised log-likelihood;
  ``schema`` tasks are scored the same way with the context varying instead of the continuation.

* ``generation_task_with_answers`` — greedy decoding until ``max_new_tokens`` or an ``early_stopping_criteria`` string; exact
  match against any of the ``answer`` / ``aliases`` after llm-foundry's normalisation (lower-case, punctuation and articles
  stripped) unless ``do_normalization: false``; with a ``cot_delimiter`` only the text after it counts. With a ``decoder``
  (a KV-cached batched decoder such as :meth:`B200Engine.decoder`) the rows are decoded in batches of the task's
  ``batch_size``; rows whose prompt plus ``max_new_tokens`` exceeds the decoder's cache, and every row when there is no
  decoder, recompute the last ``max_seq_len`` tokens with ``logits_fn`` for every new token (a sliding window, batch of one).

The scoring tasks (the first two kinds and ``schema``) decide each row on the log-likelihood of (context, continuation) pairs,
left-truncated to ``max_seq_len``. When the ``decoder`` also has ``score(pairs)`` (:meth:`KVDecoder.score`), the pairs go to it
in batches of whole rows (at most the task's ``batch_size`` rows and ``decoder.max_batch`` pairs): each distinct context is
prefilled once and shared by its choices. Rows with more pairs than ``max_batch``, pairs with nothing to score, and every
pair when there is no such decoder, run ``logits_fn`` on one pair at a time.

Datasets are jsonl files resolved against ``icl_tasks_config.root_dir`` (there is no network, so missing files yield
``skipped``).
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Any, Callable

import torch

TASK_DEFAULTS = {"num_fewshot": [0], "continuation_delimiter": " ", "example_delimiter": "\n", "prompt_string": "",
                 "question_prelimiter": "", "batch_size": 4, "max_new_tokens": 64, "early_stopping_criteria": [],
                 "cot_delimiter": "", "do_normalization": True}


def expand_task(task: dict[str, Any]) -> dict[str, Any]:
    """Fill the defaults omitted by the compact task tables."""
    t = {**TASK_DEFAULTS, **task}
    if isinstance(t["num_fewshot"], int):
        t["num_fewshot"] = [t["num_fewshot"]]
    if "label" not in t or "dataset_uri" not in t or "icl_task_type" not in t:
        raise ValueError(f"ICL task needs label/dataset_uri/icl_task_type: {task}")
    return t


def _normalize_answer(text: str) -> str:
    """llm-foundry's exact-match normalisation: lower-case, drop punctuation and articles, squeeze whitespace."""
    import re
    import string

    text = "".join(ch for ch in text.lower() if ch not in set(string.punctuation))
    return " ".join(re.sub(r"\b(a|an|the)\b", " ", text).split())


def _rows(path: Path) -> list[dict[str, Any]]:
    return [json.loads(l) for l in path.read_text().splitlines() if l.strip()]


class _RecomputeDecoder:
    """Greedy decoding without a cache: every new token runs ``logits_fn`` on the last ``max_seq_len`` tokens (batch of one).
    Same protocol as the cached decoders: ``start(prompts, max_new_tokens)`` returns the first new token of each prompt,
    ``step()`` the next one."""

    max_batch = 1

    def __init__(self, logits_fn: Callable[[torch.Tensor], torch.Tensor], max_seq_len: int) -> None:
        self.logits_fn, self.max_seq_len = logits_fn, max_seq_len
        self.ids: list[int] = []

    def _next(self) -> list[int]:
        window = self.ids[-self.max_seq_len:]
        nxt = int(self.logits_fn(torch.tensor([window], dtype=torch.long))[0, -1].float().argmax())
        self.ids.append(nxt)
        return [nxt]

    def start(self, prompts: list[list[int]], max_new_tokens: int) -> list[int]:
        (self.ids,) = [list(p) for p in prompts]
        return self._next()

    def step(self) -> list[int]:
        return self._next()


class ICLEvaluator:
    """``logits_fn(ids [B,S] LongTensor) -> [B,S,V]`` abstracts the model (torch backend or engine); ``decoder`` (optional) is
    a batched KV-cached greedy decoder with ``max_batch``, ``max_seq_len``, ``start(prompts, max_new_tokens)`` and ``step()``
    that generation tasks use for every row that fits its cache."""

    def __init__(self, logits_fn: Callable[[torch.Tensor], torch.Tensor], tokenizer: Any, max_seq_len: int, root_dir: str | None = None,
                 decoder: Any = None) -> None:
        self.logits_fn, self.tok, self.max_seq_len, self.root = logits_fn, tokenizer, int(max_seq_len), Path(root_dir or ".")
        self.decoder = decoder

    def _enc(self, text: str) -> list[int]:
        if hasattr(self.tok, "encode") and not hasattr(self.tok, "__call__"):
            return self.tok.encode(text)
        return self.tok(text, add_special_tokens=False)["input_ids"] if callable(self.tok) else self.tok.encode(text)

    def _fewshot_prefix(self, rows: list[dict[str, Any]], idx: int, k: int, t: dict[str, Any]) -> str:
        shots = [r for i, r in enumerate(rows) if i != idx][:k]
        parts = []
        for r in shots:
            cont = r.get("continuation", r["choices"][r["gold"]] if "choices" in r else "")
            parts.append(f"{t['question_prelimiter']}{r.get('context', r.get('query', ''))}{t['continuation_delimiter']}{cont}")
        return t["prompt_string"] + t["example_delimiter"].join(parts) + (t["example_delimiter"] if parts else "")

    def _truncate(self, ctx: list[int], cont: list[int]) -> tuple[list[int], list[int]]:
        """The (context, scored tokens) of a pair after left truncation: ``ctx + cont`` keeps its last ``max_seq_len`` tokens,
        of which the last ``min(len(cont), kept - 1)`` are scored (at least one context token stays)."""
        ids = (ctx + cont)[-self.max_seq_len:]
        n = min(len(cont), len(ids) - 1)
        return ids[: len(ids) - n], ids[len(ids) - n:]

    @torch.no_grad()
    def _continuation_stats(self, ctx: list[int], cont: list[int]) -> tuple[float, bool]:
        """(sum log p(cont | ctx), greedy-exact-match) with left truncation to ``max_seq_len`` (see ``_truncate``)."""
        head, tail = self._truncate(ctx, cont)
        ids, n = head + tail, len(tail)
        x = torch.tensor([ids], dtype=torch.long)
        logp = torch.log_softmax(self.logits_fn(x)[0].float(), dim=-1)
        pos = torch.arange(len(ids) - n - 1, len(ids) - 1)
        tgt = torch.tensor(tail, dtype=torch.long)
        lp = logp[pos].cpu()
        return float(lp[torch.arange(n), tgt].sum()), bool((lp.argmax(-1) == tgt).all())

    def _question_pairs(self, kind: str, prefix: str, r: dict[str, Any], t: dict[str, Any]) -> list[tuple[list[int], list[int]]]:
        """The (context, continuation) token pairs one row of a scoring task is decided on, in choice order."""
        if kind == "language_modeling":
            ctx = self._enc(prefix + t["question_prelimiter"] + r["context"] + t["continuation_delimiter"].rstrip())
            return [(ctx, self._enc(" " + r["continuation"].lstrip()))]
        if kind == "multiple_choice":
            ctx = self._enc(prefix + t["question_prelimiter"] + r["query"] + t["continuation_delimiter"].rstrip())
            return [(ctx, self._enc(" " + ch.lstrip())) for ch in r["choices"]]
        cont = self._enc(" " + r["continuation"].lstrip())   # schema: the context options vary, the continuation is shared
        return [(self._enc(prefix + opt), cont) for opt in r["context_options"]]

    @torch.no_grad()
    def _score_questions(self, questions: list[list[tuple[list[int], list[int]]]], batch_size: int) -> list[list[tuple[float, bool]]]:
        """``_continuation_stats`` of every pair of every question. With a decoder that has ``score``, the truncated pairs go to
        it in batches of whole questions: at most ``batch_size`` questions and ``decoder.max_batch`` pairs per call. A question
        with more pairs than that, and a pair with nothing to score or that does not fit the decoder's cache, take
        ``logits_fn`` one pair at a time."""
        out: list[list[tuple[float, bool] | None]] = [[None] * len(q) for q in questions]
        dec = self.decoder
        if dec is not None and callable(getattr(dec, "score", None)):
            cap, per = int(dec.max_batch), max(1, int(batch_size))
            batch: list[tuple[int, int, list[int], list[int]]] = []   # (question, pair, context, scored)
            n_q = 0

            def flush() -> None:
                for (qi, pi, _, _), st in zip(batch, dec.score([(c, s) for _, _, c, s in batch])):
                    out[qi][pi] = st

            for qi, q in enumerate(questions):
                if len(q) > cap:
                    continue
                items = [(qi, pi, *self._truncate(ctx, cont)) for pi, (ctx, cont) in enumerate(q)]
                items = [it for it in items if it[2] and it[3] and len(it[2]) + len(it[3]) <= dec.max_seq_len]
                if not items:
                    continue
                if batch and (n_q == per or len(batch) + len(items) > cap):
                    flush()
                    batch, n_q = [], 0
                batch += items
                n_q += 1
            if batch:
                flush()
        return [[st if st is not None else self._continuation_stats(ctx, cont) for st, (ctx, cont) in zip(row, q)]
                for row, q in zip(out, questions)]

    @torch.no_grad()
    def _generate(self, ctx: list[int], max_new_tokens: int, stops: list[str]) -> str:
        """Greedy continuation of ``ctx`` as text, cut at the first stop string (sliding window, no cache)."""
        return self._generate_batch(_RecomputeDecoder(self.logits_fn, self.max_seq_len), [ctx], max_new_tokens, stops)[0]

    def _generate_batch(self, dec: Any, ctxs: list[list[int]], max_new_tokens: int, stops: list[str]) -> list[str]:
        """Greedy continuations of a batch of prompts with ``dec``. Per row: EOS ends the row and is not emitted; after each
        token the decoded text is checked against the stop strings and cut at the first one."""
        eos = getattr(self.tok, "eos_token_id", None)
        new: list[list[int]] = [[] for _ in ctxs]
        texts: list[str | None] = [None] * len(ctxs)
        if max_new_tokens <= 0:
            return [self.tok.decode([]) for _ in ctxs]
        toks = dec.start(ctxs, max_new_tokens)
        for t in range(max_new_tokens):
            for i, nxt in enumerate(toks):
                if texts[i] is not None:
                    continue
                if eos is not None and nxt == eos:
                    texts[i] = self.tok.decode(new[i])
                    continue
                new[i].append(nxt)
                text = self.tok.decode(new[i])
                hit = [text.index(s) for s in stops if s and s in text]
                if hit:
                    texts[i] = text[: min(hit)]
            if t == max_new_tokens - 1 or all(x is not None for x in texts):
                break
            toks = dec.step()
        return [x if x is not None else self.tok.decode(n) for x, n in zip(texts, new)]

    @torch.no_grad()
    def _generate_rows(self, ctxs: list[list[int]], max_new_tokens: int, stops: list[str], batch_size: int) -> list[str]:
        """Every row that fits the decoder's cache in batches of ``batch_size``; the others one by one on the sliding window."""
        out: list[str | None] = [None] * len(ctxs)
        dec = self.decoder
        if dec is not None:
            fits = [i for i, c in enumerate(ctxs) if 1 <= len(c) and len(c) + max_new_tokens <= dec.max_seq_len]
            n = max(1, min(int(batch_size), dec.max_batch))
            for lo in range(0, len(fits), n):
                idx = fits[lo: lo + n]
                for i, text in zip(idx, self._generate_batch(dec, [ctxs[i] for i in idx], max_new_tokens, stops)):
                    out[i] = text
        return [x if x is not None else self._generate(c, max_new_tokens, stops) for x, c in zip(out, ctxs)]

    def evaluate_task(self, task: dict[str, Any]) -> dict[str, float | str]:
        t = expand_task(task)
        path = self.root / t["dataset_uri"]
        if not path.exists():
            return {"status": "skipped (dataset missing offline)"}
        kind = t["icl_task_type"]
        if kind not in ("language_modeling", "multiple_choice", "schema", "generation_task_with_answers"):
            return {"status": f"unsupported task type {kind}"}
        if kind == "generation_task_with_answers" and not hasattr(self.tok, "decode"):
            return {"status": "generation tasks need a tokenizer with decode()"}
        rows = _rows(path)
        out: dict[str, float | str] = {}
        for k in t["num_fewshot"]:
            correct = 0
            texts: list[str] = []
            stats: list[list[tuple[float, bool]]] = []
            if kind == "generation_task_with_answers":
                ctxs = [self._enc(self._fewshot_prefix(rows, i, k, t) + t["question_prelimiter"] + r["context"]
                                  + t["continuation_delimiter"].rstrip()) for i, r in enumerate(rows)]
                texts = self._generate_rows(ctxs, int(t["max_new_tokens"]), list(t["early_stopping_criteria"] or []), int(t["batch_size"]))
            else:
                questions = [self._question_pairs(kind, self._fewshot_prefix(rows, i, k, t), r, t) for i, r in enumerate(rows)]
                stats = self._score_questions(questions, int(t["batch_size"]))
            for i, r in enumerate(rows):
                if kind == "generation_task_with_answers":
                    text = texts[i]
                    if t["cot_delimiter"] and t["cot_delimiter"] in text:
                        text = text.split(t["cot_delimiter"])[-1]
                    golds = [str(r["answer"])] + [str(a) for a in r.get("aliases", [])]
                    norm = _normalize_answer if t["do_normalization"] else (lambda x: x.strip())
                    correct += int(any(norm(text).startswith(norm(g)) for g in golds if norm(g)))
                elif kind == "language_modeling":
                    correct += int(stats[i][0][1])
                else:   # multiple_choice / schema: the highest length-normalised log-likelihood
                    scores = [lp / max(1, len(cont)) for (lp, _), (_, cont) in zip(stats[i], questions[i])]
                    correct += int(int(torch.tensor(scores).argmax()) == int(r["gold"]))
            out[f"{t['label']}/{k}-shot/accuracy"] = correct / max(1, len(rows))
            out[f"{t['label']}/{k}-shot/n_samples"] = float(len(rows))
        return out


class EvalGauntlet:
    """Category averages over benchmark accuracies with random-baseline subtraction and rescaling
    (the semantics of llm-foundry's EvalGauntlet for ``weighting: EQUAL``)."""

    def __init__(self, cfg: dict[str, Any]) -> None:
        self.cfg = cfg
        if cfg.get("weighting", "EQUAL") not in ("EQUAL", "SAMPLE_SZ", "LOG_SAMPLE_SZ"):
            raise ValueError(f"unknown eval_gauntlet weighting {cfg.get('weighting')!r} (EQUAL | SAMPLE_SZ | LOG_SAMPLE_SZ)")

    def _weight(self, n_samples: float) -> float:
        """llm-foundry's benchmark weights inside a category: equal, by sample count, or by log2 of it (at least 1)."""
        import math

        mode = self.cfg.get("weighting", "EQUAL")
        if mode == "EQUAL" or n_samples <= 0:
            return 1.0
        return float(n_samples) if mode == "SAMPLE_SZ" else max(math.log2(n_samples), 1.0)

    def aggregate(self, metrics: dict[str, float]) -> dict[str, float]:
        out: dict[str, float] = {}
        for cat in self.cfg.get("categories", []):
            vals, wts = [], []
            for b in cat["benchmarks"]:
                key = f"{b['name']}/{b['num_fewshot']}-shot/accuracy"
                if key not in metrics:
                    continue
                wts.append(self._weight(float(metrics.get(f"{b['name']}/{b['num_fewshot']}-shot/n_samples", 0.0))))
                acc, base = float(metrics[key]), float(b.get("random_baseline", 0.0))
                if self.cfg.get("subtract_random_baseline", True):
                    acc -= base
                if self.cfg.get("rescale_accuracy", True) and base < 1.0:
                    acc /= (1.0 - base)
                vals.append(acc)
            if vals:
                out[f"icl/metrics/eval_gauntlet/{cat['name']}"] = sum(v * w for v, w in zip(vals, wts)) / sum(wts)
        for name, cats in (self.cfg.get("averages") or {}).items():
            vs = [out[f"icl/metrics/eval_gauntlet/{c}"] for c in cats if f"icl/metrics/eval_gauntlet/{c}" in out]
            if vs:
                out[f"icl/metrics/eval_gauntlet/{name}"] = sum(vs) / len(vs)
        return out


def run_icl_suite(logits_fn: Callable[[torch.Tensor], torch.Tensor], tokenizer: Any, cfg: Any, max_seq_len: int,
                  decoder: Any = None) -> dict[str, Any]:
    """Evaluate every task of ``cfg.icl_tasks_config`` and fold through ``cfg.eval_gauntlet_config``; generation tasks decode with
    ``decoder`` when one is given (see :class:`ICLEvaluator`)."""
    icl = cfg.get("icl_tasks_config") or {}
    tasks = icl.get("icl_tasks") or []
    ev = ICLEvaluator(logits_fn, tokenizer, max_seq_len, icl.get("root_dir"), decoder=decoder)
    metrics: dict[str, Any] = {}
    for t in tasks:
        metrics.update({k: v for k, v in ev.evaluate_task(dict(t)).items() if not (k == "status")})
    g = (cfg.get("eval_gauntlet_config") or {}).get("eval_gauntlet")
    if g:
        metrics.update(EvalGauntlet(dict(g)).aggregate({k: v for k, v in metrics.items() if isinstance(v, float)}))
    return metrics
