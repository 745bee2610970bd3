"""The ICL evaluator's batched scoring path (a decoder with ``score``) against its pair-at-a-time ``logits_fn`` path."""
import json

import pytest
import torch

from photon_b200.dataset.utils import ByteTokenizer
from photon_b200.eval import ICLEvaluator
from test_eval_icl_decoder import FakeDecoder, _fake_logits


class FakeScorer:
    """A decoder with ``score`` over the +1 model of ``_fake_logits``: exact stats of each (context, scored tokens) pair."""

    def __init__(self, max_batch=8, max_seq_len=64):
        self.max_batch, self.max_seq_len = max_batch, max_seq_len
        self.calls = []

    def score(self, pairs):
        assert 1 <= len(pairs) <= self.max_batch
        self.calls.append([(list(c), list(s)) for c, s in pairs])
        out = []
        for ctx, sc in pairs:
            assert ctx and sc and len(ctx) + len(sc) <= self.max_seq_len
            ids = ctx + sc
            lp = torch.log_softmax(_fake_logits(torch.tensor([ids]))[0].float(), -1)[len(ctx) - 1: len(ids) - 1]
            tgt = torch.tensor(sc)
            out.append((float(lp[torch.arange(len(sc)), tgt].sum()), bool((lp.argmax(-1) == tgt).all())))
        return out


MC = [{"query": "ab", "choices": ["!\"#", "xyz", "!\"", "q"], "gold": 0},
      {"query": "Q: 12", "choices": ["!", "nope", "!\"#$%", "zz"], "gold": 2},
      {"query": "xyz", "choices": ["a", "!\"", "b", "c"], "gold": 3},
      {"query": "hello there", "choices": ["!!", "!\"", "!", "! "], "gold": 1},
      {"query": "m", "choices": ["1", "2", "3", "!\"#$"], "gold": 3}]
SCHEMA = [{"context_options": ["The cat", "A dog", "It"], "continuation": "ran away", "gold": 0},
          {"context_options": ["x", "xyz \x1f"], "continuation": "!\"#", "gold": 1},
          {"context_options": ["hello", "abc", "abcd", "q"], "continuation": "ok", "gold": 2}]
LM = [{"context": "abc\x1f", "continuation": "!\"#"}, {"context": "The answer is", "continuation": "!"},
      {"context": "xy", "continuation": "zz"}, {"context": "0123\x1f", "continuation": "!\"#$%&"}]
TASKS = {"mc": {"label": "mc", "dataset_uri": "mc.jsonl", "icl_task_type": "multiple_choice", "num_fewshot": [0, 1], "batch_size": 2},
         "schema": {"label": "schema", "dataset_uri": "schema.jsonl", "icl_task_type": "schema", "num_fewshot": [0, 1], "batch_size": 2},
         "lm": {"label": "lm", "dataset_uri": "lm.jsonl", "icl_task_type": "language_modeling", "num_fewshot": [0, 1], "batch_size": 3}}


def _write(tmp_path):
    for name, rows in (("mc", MC), ("schema", SCHEMA), ("lm", LM)):
        (tmp_path / f"{name}.jsonl").write_text("\n".join(json.dumps(r) for r in rows))


def _counting_logits(calls):
    def fn(ids):
        calls.append(ids.shape[1])
        return _fake_logits(ids)

    return fn


@pytest.mark.parametrize("max_seq_len", [64, 6])
@pytest.mark.parametrize("task", list(TASKS))
def test_scorer_matches_pair_at_a_time(tmp_path, task, max_seq_len):
    _write(tmp_path)
    tok = ByteTokenizer()
    plain_calls, scored_calls = [], []
    plain = ICLEvaluator(_counting_logits(plain_calls), tok, max_seq_len, str(tmp_path))
    dec = FakeScorer(max_batch=8, max_seq_len=max_seq_len)
    batched = ICLEvaluator(_counting_logits(scored_calls), tok, max_seq_len, str(tmp_path), decoder=dec)
    want = plain.evaluate_task(TASKS[task])
    assert want == batched.evaluate_task(TASKS[task])
    assert 0.0 < sum(v for key, v in want.items() if key.endswith("accuracy"))   # the tasks are not trivially all wrong
    assert dec.calls and not scored_calls   # every pair went through score
    if max_seq_len == 6 and task == "mc":
        # choices of different lengths keep different context tails: one question, several distinct contexts in one call
        assert any(len({tuple(c) for c, _ in call}) > len(call) // 4 for call in dec.calls)


def test_truncation_helper_returns_the_scored_tokens():
    seen = []

    def logits(ids):
        seen.append(ids[0].tolist())
        return _fake_logits(ids)

    for msl in (4, 5, 8, 64):
        ev = ICLEvaluator(logits, ByteTokenizer(), msl)
        for ctx, cont in (([1, 2, 3], [4, 5]), ([1], [2, 3, 4, 5, 6, 7]), ([9] * 10, [1]), ([1, 2], [])):
            head, tail = ev._truncate(ctx, cont)
            ids = (ctx + cont)[-msl:]
            n = min(len(cont), len(ids) - 1)
            assert head + tail == ids and len(tail) == n and head   # at least one context token stays
            seen.clear()
            lp, em = ev._continuation_stats(ctx, cont)
            assert seen == [head + tail]
            want = FakeScorer(max_seq_len=msl).score([(head, tail)])[0] if tail else (0.0, True)
            assert (lp, em) == pytest.approx(want)


@pytest.mark.parametrize("bs,cap", [(1, 8), (2, 8), (3, 8), (16, 10), (4, 4)])
def test_score_batches_hold_whole_questions(tmp_path, bs, cap):
    _write(tmp_path)
    dec = FakeScorer(max_batch=cap)
    ICLEvaluator(_fake_logits, ByteTokenizer(), 64, str(tmp_path), decoder=dec).evaluate_task({**TASKS["mc"], "batch_size": bs, "num_fewshot": [0]})
    sizes = [len(c) for c in dec.calls]
    assert sum(sizes) == 4 * len(MC)
    per_call = min(bs, cap // 4)
    assert sizes == [4 * per_call] * (len(MC) // per_call) + ([4 * (len(MC) % per_call)] if len(MC) % per_call else [])
    for call in dec.calls:   # whole questions: every context appears exactly four times, once per choice
        ctxs = [tuple(c) for c, _ in call]
        assert all(ctxs.count(c) == 4 for c in ctxs) and len(set(ctxs)) <= bs


def test_question_larger_than_max_batch_uses_logits_fn(tmp_path):
    rows = [{"query": "ab", "choices": ["!", "x"], "gold": 0}, {"query": "cd", "choices": ["!", "x", "y", "z"], "gold": 0},
            {"query": "ef", "choices": ["x", "!"], "gold": 1}]
    (tmp_path / "mc.jsonl").write_text("\n".join(json.dumps(r) for r in rows))
    calls = []
    dec = FakeScorer(max_batch=3)
    ev = ICLEvaluator(_counting_logits(calls), ByteTokenizer(), 64, str(tmp_path), decoder=dec)
    task = {**TASKS["mc"], "num_fewshot": [0], "batch_size": 4}
    got = ev.evaluate_task(task)
    assert len(calls) == 4   # the 4-choice question, one pair at a time
    assert [len(c) for c in dec.calls] == [2, 2]   # the 2-choice questions (3 pairs would split the second one)
    assert got == ICLEvaluator(_fake_logits, ByteTokenizer(), 64, str(tmp_path)).evaluate_task(task)
    assert got["mc/0-shot/accuracy"] == 1.0


def test_decoder_without_score_keeps_the_old_path(tmp_path):
    _write(tmp_path)
    tok = ByteTokenizer()
    for task in TASKS.values():
        a, b = [], []
        plain = ICLEvaluator(_counting_logits(a), tok, 64, str(tmp_path)).evaluate_task(task)
        dec = FakeDecoder()
        assert plain == ICLEvaluator(_counting_logits(b), tok, 64, str(tmp_path), decoder=dec).evaluate_task(task)
        assert a == b and dec.batches == []
