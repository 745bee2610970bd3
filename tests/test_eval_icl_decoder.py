"""The ICL evaluator's batched decoding path against its unbatched sliding-window path, with a fake cached decoder."""
import json

import torch

from photon_b200.dataset.utils import ByteTokenizer
from photon_b200.eval import ICLEvaluator


def _fake_logits(ids):
    """A 'model' that always predicts next byte = current byte + 1 (mod 257)."""
    B, S = ids.shape
    out = torch.full((B, S, 257), -10.0)
    out[torch.arange(B)[:, None], torch.arange(S)[None], (ids + 1) % 257] = 10.0
    return out


class FakeDecoder:
    """A batched 'cached' decoder over the +1 model: it keeps only the last token of every row."""

    def __init__(self, max_batch=8, max_seq_len=64):
        self.max_batch, self.max_seq_len = max_batch, max_seq_len
        self.batches = []

    def start(self, prompts, max_new_tokens):
        assert len(prompts) <= self.max_batch
        assert all(len(p) + max_new_tokens <= self.max_seq_len for p in prompts)
        self.batches.append(len(prompts))
        self.last = [(p[-1] + 1) % 257 for p in prompts]
        return list(self.last)

    def step(self):
        self.last = [(t + 1) % 257 for t in self.last]
        return list(self.last)


# contexts end in bytes whose +1 chains hit a stop string, the EOS byte (0 after 256), or nothing within max_new_tokens
ROWS = [{"context": "a", "answer": "b"}, {"context": "wxy", "answer": "z"}, {"context": "\x07", "answer": "\x08\t"},
        {"context": "\xfd", "answer": "x"}, {"context": "AB", "answer": "C"}, {"context": "0", "answer": "12"},
        {"context": "r" * 70, "answer": "s"}]
TASK = {"label": "gen", "dataset_uri": "gen.jsonl", "icl_task_type": "generation_task_with_answers", "max_new_tokens": 5,
        "batch_size": 3, "early_stopping_criteria": ["\n", "E"], "do_normalization": False}


def _write(tmp_path):
    (tmp_path / "gen.jsonl").write_text("\n".join(json.dumps(r) for r in ROWS))


def test_batched_decoding_matches_unbatched(tmp_path):
    _write(tmp_path)
    tok = ByteTokenizer()
    plain = ICLEvaluator(_fake_logits, tok, 64, str(tmp_path))
    dec = FakeDecoder()
    batched = ICLEvaluator(_fake_logits, tok, 64, str(tmp_path), decoder=dec)
    for task in (TASK, {**TASK, "cot_delimiter": "c"}, {**TASK, "num_fewshot": [0, 1]}):
        assert plain.evaluate_task(task) == batched.evaluate_task(task)
    ctxs = [tok.encode(r["context"]) for r in ROWS]
    for stops in ([], ["\n", "E"], ["z"]):
        want = [plain._generate(c, 5, stops) for c in ctxs]
        assert batched._generate_rows(ctxs, 5, stops, 3) == want
    assert plain._generate(tok.encode("AB"), 5, ["E"]) == "CD"          # cut at the stop string
    assert plain._generate([253], 5, []) == tok.decode([254, 255, 256])   # EOS (0 after 256) ends the row, not emitted
    assert batched._generate_rows([[253], [65]], 5, [], 2) == [tok.decode([254, 255, 256]), "ABCDE"]


def test_rows_past_the_cache_take_the_sliding_window(tmp_path):
    tok = ByteTokenizer()
    calls = []

    def logits(ids):
        calls.append(ids.shape[1])
        return _fake_logits(ids)

    dec = FakeDecoder(max_seq_len=64)
    ev = ICLEvaluator(logits, tok, 64, str(tmp_path), decoder=dec)
    out = ev._generate_rows([tok.encode("r" * 70), tok.encode("ab")], 5, [], 4)
    assert out == ["stuvw", "cdefg"]
    assert dec.batches == [1] and calls and max(calls) == 64   # only the long row recomputed, on the last 64 tokens


def test_decoder_batches_honour_batch_size(tmp_path):
    _write(tmp_path)
    for bs, cap, want in ((3, 8, [3, 3]), (2, 8, [2, 2, 2]), (8, 4, [4, 2]), (1, 8, [1] * 6)):
        dec = FakeDecoder(max_batch=cap)
        ICLEvaluator(_fake_logits, ByteTokenizer(), 64, str(tmp_path), decoder=dec).evaluate_task({**TASK, "batch_size": bs})
        assert dec.batches == want, (bs, cap, dec.batches)


def test_suite_builders_forward_the_decoder(tmp_path, monkeypatch):
    import photon_b200.eval.icl as icl_mod
    from photon_b200.clients.trainer_utils import build_icl_suite

    _write(tmp_path)
    cfg = {"icl_tasks_config": {"root_dir": str(tmp_path), "icl_tasks": [TASK]}}
    dec = FakeDecoder()
    out = icl_mod.run_icl_suite(_fake_logits, ByteTokenizer(), cfg, 64, decoder=dec)
    assert dec.batches == [3, 3] and "gen/0-shot/accuracy" in out
    seen = {}
    monkeypatch.setattr(icl_mod, "run_icl_suite", lambda *a, **k: seen.update(k) or {})
    monkeypatch.setattr("photon_b200.dataset.utils.build_tokenizer", lambda name: ByteTokenizer())
    suite = build_icl_suite({**cfg, "llm_config": {"tokenizer": {"name": "bytes"}}}, 64)
    suite(_fake_logits, decoder=dec)
    assert seen["decoder"] is dec
