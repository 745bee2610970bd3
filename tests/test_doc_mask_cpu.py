"""CPU checks of document-masked attention (llm-foundry's ``attn_uses_sequence_id`` with ``dataset.{eos,bos}_token_id``):
the collator's ids, config parsing, the trainer's plumbing and the PyTorch model's mask."""
import pytest
import torch

from photon_b200.data.streaming import build_text_loader, sequence_ids
from photon_b200.models.mpt import MPTConfig, MPTForCausalLM
from photon_b200.train.trainer import Trainer, check_sequence_id_runs

TORCH_KERNELS = dict(gemm="torch", attention="torch", norm="torch", loss="torch", optimizer="torch")


# ------------------------------------------------------------------------------------------------ collator
def test_eos_mode_ids_end_documents_with_their_eos():
    ids = torch.tensor([[5, 0, 7, 8, 0, 0, 9], [0, 1, 2, 3, 4, 5, 0]])
    assert sequence_ids(ids, eos_token_id=0).tolist() == [[0, 0, 1, 1, 1, 2, 3], [0, 1, 1, 1, 1, 1, 1]]


def test_bos_mode_ids_open_documents_with_their_bos():
    ids = torch.tensor([[1, 5, 6, 1, 7, 1, 1], [4, 4, 1, 4, 4, 4, 4]])
    assert sequence_ids(ids, bos_token_id=1).tolist() == [[1, 1, 1, 2, 2, 3, 4], [0, 0, 1, 1, 1, 1, 1]]


def test_both_separator_keys_are_an_error():
    with pytest.raises(ValueError):
        sequence_ids(torch.zeros(1, 4, dtype=torch.long), eos_token_id=0, bos_token_id=1)
    cfg = {"dataset": {"streams": {"a": {"local": "synthetic://c4"}}, "max_seq_len": 32, "eos_token_id": 0, "bos_token_id": 1}}
    with pytest.raises(ValueError):
        build_text_loader(cfg, batch_size=2, vocab_size=128)


def _first_batch(extra):
    cfg = {"dataset": {"streams": {"a": {"local": "synthetic://c4"}}, "max_seq_len": 64, "synthetic_samples": 8, **extra}}
    loader = build_text_loader(cfg, batch_size=4, vocab_size=128)
    return next(iter(loader))


def test_loader_adds_sequence_id_only_with_a_separator_key():
    plain = _first_batch({})
    assert "sequence_id" not in plain
    eos = _first_batch({"eos_token_id": 0})
    assert eos["sequence_id"].dtype == eos["input_ids"].dtype == torch.int64
    assert torch.equal(eos["sequence_id"], sequence_ids(eos["input_ids"], eos_token_id=0))
    assert torch.equal(eos["input_ids"], plain["input_ids"])
    bos = _first_batch({"bos_token_id": 0})
    assert torch.equal(bos["sequence_id"], sequence_ids(bos["input_ids"], bos_token_id=0))


def test_client_stream_surgery_keeps_the_separator_keys():
    from photon_b200.clients.llm_config_functions import set_stream
    from photon_b200.config.composer import ConfigNode

    ds = ConfigNode({"streams": [{"c4": {"local": "synthetic://c4"}}, {"c4b": {"local": "synthetic://c4"}}],
                     "eos_token_id": 0, "bos_token_id": None, "max_seq_len": 64})
    set_stream(ds, 1)
    assert ds["eos_token_id"] == 0 and "bos_token_id" in ds and isinstance(ds["streams"], dict)


# ------------------------------------------------------------------------------------------------ config
def test_config_parses_attn_uses_sequence_id():
    m = {"d_model": 32, "n_heads": 2, "n_layers": 1, "attn_config": {"attn_impl": "torch", "attn_uses_sequence_id": True}}
    assert MPTConfig.from_model_cfg(m).attn_uses_sequence_id is True
    cfg = MPTConfig.from_model_cfg({**m, "attn_config": {"attn_impl": "torch"}})
    assert cfg.attn_uses_sequence_id is False and "attn_config" not in cfg.extra


# ------------------------------------------------------------------------------------------------ trainer
class _Loader:
    def __init__(self, ids, sid=None):
        self.ids, self.sid = ids, sid

    def __iter__(self):
        while True:
            yield {"input_ids": self.ids} if self.sid is None else {"input_ids": self.ids, "sequence_id": self.sid}


def _trainer(loader, uses=True, mb=2):
    cfg = MPTConfig(d_model=32, n_heads=2, n_layers=1, max_seq_len=16, vocab_size=64, attn_impl="torch", attn_uses_sequence_id=uses)
    return Trainer(cfg, optimizer_cfg=dict(name="decoupled_adamw", lr=1e-3), scheduler_cfg=dict(name="constant_with_warmup", t_warmup="0ba"),
                   train_loader=loader, global_train_batch_size=6, device_train_microbatch_size=mb, precision="fp32", device="cpu",
                   kernels=TORCH_KERNELS)


def test_trainer_slices_sequence_id_with_the_microbatches():
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, 64, (6, 16), generator=g)
    ids[:, 5] = 0
    sid = sequence_ids(ids, eos_token_id=0) + torch.arange(6)[:, None]   # a different offset per row: slices are traceable
    tr = _trainer(_Loader(ids, sid))
    seen = []
    real = tr.state.backend.fwd_bwd

    def spy(x, denom, scale=1.0, sequence_id=None):
        seen.append((x.clone(), None if sequence_id is None else sequence_id.clone()))
        return real(x, denom, scale, sequence_id=sequence_id)

    tr.state.backend.fwd_bwd = spy
    tr.fit("1ba")
    assert len(seen) == 3
    for i, (x, s) in enumerate(seen):
        assert torch.equal(x, ids[2 * i:2 * i + 2]) and torch.equal(s, sid[2 * i:2 * i + 2])
    # a batch without ids passes none, and the backend then refuses to train with the flag on
    tr2 = _trainer(_Loader(ids))
    with pytest.raises(ValueError, match="sequence_id"):
        tr2.fit("1ba")
    # the flag off: ids in the batch are ignored by the model, the step matches one without them
    a, b = _trainer(_Loader(ids, sid), uses=False), _trainer(_Loader(ids), uses=False)
    a.fit("1ba"), b.fit("1ba")
    assert torch.equal(a.state.flat.params, b.state.flat.params)
    for t in (tr, tr2, a, b):
        t.close()


def test_trainer_eval_passes_sequence_id():
    ids = torch.randint(1, 64, (4, 16), generator=torch.Generator().manual_seed(2))
    sid = torch.zeros_like(ids)
    sid[:, 8:] = 1
    tr = _trainer(_Loader(ids, sid))
    got = []
    real = tr.state.backend.eval_stats
    tr.state.backend.eval_stats = lambda x, sequence_id=None: got.append(sequence_id) or real(x, sequence_id=sequence_id)
    tr._eval_batch_stats(ids, sid)
    tr._eval_batch_stats(ids)
    assert torch.equal(got[0], sid) and got[1] is None
    tr.close()


def test_non_monotone_sequence_ids_are_rejected():
    check_sequence_id_runs(torch.tensor([[0, 0, 1, 1, 2]]))
    with pytest.raises(ValueError, match="non-decreasing"):
        check_sequence_id_runs(torch.tensor([[0, 0, 1, 0, 2]]))
    ids = torch.randint(1, 64, (6, 16), generator=torch.Generator().manual_seed(3))
    sid = torch.zeros_like(ids)
    sid[:, 4] = 1                      # 0 0 0 0 1 0 ...: the same id in two runs
    tr = _trainer(_Loader(ids, sid))
    with pytest.raises(ValueError, match="non-decreasing"):
        tr.fit("1ba")
    tr.close()


# ------------------------------------------------------------------------------------------------ model
@pytest.mark.parametrize("pos", ["learned", "alibi", "rope"])
@pytest.mark.parametrize("impl", ["torch", "flash"])
def test_model_attends_within_documents(pos, impl):
    extra = {"learned": {}, "alibi": dict(alibi=True, learned_pos_emb=False), "rope": dict(rope=True, learned_pos_emb=False)}[pos]
    cfg = MPTConfig(d_model=32, n_heads=2, n_layers=2, max_seq_len=24, vocab_size=64, attn_impl=impl, attn_uses_sequence_id=True, **extra)
    model = MPTForCausalLM(cfg, seed=0).eval()
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(1, 64, (2, 24), generator=g)
    sid = torch.tensor([[0] * 7 + [1] * 9 + [2] * 8, [0] * 24])
    with torch.no_grad():
        full = model(ids, sequence_id=sid)
        # document 1 alone: its prefix run by itself (positions are absolute, so the first document is the prefix)
        alone = model(ids[:1, :7])
        torch.testing.assert_close(full[0, :7], alone[0], rtol=1e-5, atol=1e-5)
        # new tokens in document 2 leave document 3 unchanged (and document 1)
        other = ids.clone()
        other[0, 7:16] = torch.randint(1, 64, (9,), generator=g)
        again = model(other, sequence_id=sid)
        torch.testing.assert_close(again[0, 16:], full[0, 16:], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(again[0, :7], full[0, :7], rtol=1e-5, atol=1e-5)
        assert not torch.allclose(again[0, 7:16], full[0, 7:16])
        # one document per row is the plain causal model; the flag off ignores the ids
        torch.testing.assert_close(full[1], model(ids[1:])[0], rtol=1e-5, atol=1e-5)
        cfg_off = MPTConfig(**{**cfg.__dict__, "attn_uses_sequence_id": False})
        off = MPTForCausalLM(cfg_off, seed=0).eval()
        torch.testing.assert_close(off(ids, sequence_id=sid), off(ids), rtol=0, atol=0)


def test_model_sequence_id_through_activation_checkpointing():
    cfg = MPTConfig(d_model=32, n_heads=2, n_layers=2, max_seq_len=16, vocab_size=64, attn_impl="torch", attn_uses_sequence_id=True)
    ids = torch.randint(1, 64, (2, 16), generator=torch.Generator().manual_seed(5))
    sid = torch.tensor([[0] * 5 + [1] * 11, [0] * 9 + [1] * 7])
    grads = []
    for ckpt in (False, True):
        m = MPTForCausalLM(cfg, seed=0).train()
        m.activation_checkpointing = ckpt
        loss, n = m.loss(ids, sequence_id=sid)
        loss.backward()
        grads.append(torch.cat([p.grad.flatten() for p in m.parameters()]))
        assert int(n) == 2 * 15   # the cross-document targets stay in the loss
    torch.testing.assert_close(grads[0], grads[1], rtol=1e-5, atol=1e-6)

