"""Grouped-query and multi-query attention (attn_config.attn_type / kv_n_heads) in the config and the PyTorch model, without a GPU."""
import math

import numpy as np
import pytest
import torch

from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, alibi_slopes, apply_rope, rope_tables
from photon_b200.utils.flat import FlatParams


def _m(**attn):
    return {"d_model": 64, "n_heads": 8, "n_layers": 2, "max_seq_len": 32, "vocab_size": 96, "attn_config": attn}


# ------------------------------------------------------------------------------------------------ config
def test_config_parses_attn_type():
    assert MPTConfig.from_model_cfg(_m()).kv_n_heads == 8
    assert MPTConfig(d_model=64, n_heads=8).kv_n_heads == 8
    gqa = MPTConfig.from_model_cfg(_m(attn_type="grouped_query_attention", kv_n_heads=2))
    assert gqa.kv_n_heads == 2 and gqa.kv_dim == 16 and gqa.qkv_dim == 96
    assert "attn_config" not in gqa.extra   # both keys are consumed, nothing lands in the ignored extras
    assert MPTConfig.from_model_cfg(_m(attn_type="multiquery_attention")).kv_n_heads == 1
    assert MPTConfig.from_model_cfg(_m(attn_type="multiquery_attention", kv_n_heads=4)).kv_n_heads == 1
    # llm-foundry ignores kv_n_heads under multi-head attention
    assert MPTConfig.from_model_cfg(_m(attn_type="multihead_attention", kv_n_heads=2)).kv_n_heads == 8
    # qk_gn / fused_qkv keep their existing (multi-head) handling
    assert MPTConfig.from_model_cfg(_m(qk_gn=True)).extra["attn_config"] == {"qk_gn": True}


@pytest.mark.parametrize("attn,match", [
    ({"attn_type": "sliding_window_attention"}, "unknown attn_config.attn_type"),
    ({"attn_type": "grouped_query_attention"}, "needs attn_config.kv_n_heads"),
    ({"attn_type": "grouped_query_attention", "kv_n_heads": 3}, "must divide"),
    ({"attn_type": "grouped_query_attention", "kv_n_heads": 0}, "must divide"),
    ({"attn_type": "grouped_query_attention", "kv_n_heads": 2, "qk_gn": True}, "qk_gn"),
    ({"attn_type": "multiquery_attention", "qk_gn": True}, "qk_gn"),
    ({"attn_type": "grouped_query_attention", "kv_n_heads": 2, "fused_qkv": False}, "fused_qkv"),
    ({"attn_type": "multiquery_attention", "fused_qkv": False}, "fused_qkv"),
])
def test_config_rejects(attn, match):
    with pytest.raises(ValueError, match=match):
        MPTConfig.from_model_cfg(_m(**attn))


def test_direct_config_rejects_a_kv_count_that_does_not_divide():
    with pytest.raises(ValueError, match="must divide"):
        MPTConfig(d_model=64, n_heads=8, kv_n_heads=3)


# ------------------------------------------------------------------------------------------------ parameters
@pytest.mark.parametrize("kv,no_bias,qk_ln", [(8, False, False), (2, False, False), (1, True, False), (2, False, True), (1, False, True)])
def test_parameter_shapes_and_count(kv, no_bias, qk_ln):
    cfg = MPTConfig(d_model=64, n_heads=8, n_layers=2, max_seq_len=32, vocab_size=96, kv_n_heads=kv, no_bias=no_bias, qk_ln=qk_ln)
    model = MPTForCausalLM(cfg, seed=0)
    named = dict(model.named_parameters())
    w = 64 + 2 * kv * 8
    assert named["transformer.blocks.0.attn.Wqkv.weight"].shape == (w, 64)
    if not no_bias:
        assert named["transformer.blocks.0.attn.Wqkv.bias"].shape == (w,)
    if qk_ln:
        assert named["transformer.blocks.1.attn.q_ln.weight"].shape == (64,)
        assert named["transformer.blocks.1.attn.k_ln.weight"].shape == (kv * 8,)
        assert named["transformer.blocks.1.attn.k_ln.bias"].shape == (kv * 8,)
    ln_params = sum(p.numel() for n, p in named.items() if "q_ln" in n or "k_ln" in n)   # not counted by num_params (as before)
    assert cfg.num_params() == sum(p.numel() for p in named.values()) - ln_params


def test_qkv_slices_are_initialised_independently():
    """q, k and v rows each get the kaiming std of the input width, whatever their heights."""
    cfg = MPTConfig(d_model=256, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96, kv_n_heads=2)
    w = MPTForCausalLM(cfg, seed=3).transformer.blocks[0].attn.Wqkv.weight.detach()
    for lo, hi in ((0, 256), (256, 320), (320, 384)):
        assert abs(w[lo:hi].std().item() / math.sqrt(2.0 / 256) - 1.0) < 0.05


def test_kv_equal_to_heads_is_multi_head_bitwise():
    mha = MPTConfig.from_model_cfg(_m(attn_impl="torch", qk_ln=True, rope=True, clip_qkv=2.0))
    gqa = MPTConfig.from_model_cfg(_m(attn_impl="torch", qk_ln=True, rope=True, clip_qkv=2.0, attn_type="grouped_query_attention",
                                      kv_n_heads=8))
    a, b = MPTForCausalLM(mha, seed=5), MPTForCausalLM(gqa, seed=5)
    for (na, pa), (nb, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert na == nb and torch.equal(pa, pb)
    ids = torch.randint(0, 96, (2, 32), generator=torch.Generator().manual_seed(0))
    la, _ = a.loss(ids)
    lb, _ = b.loss(ids)
    la.backward()
    lb.backward()
    assert torch.equal(la, lb)
    assert all(torch.equal(pa.grad, pb.grad) for pa, pb in zip(a.parameters(), b.parameters()))


# ------------------------------------------------------------------------------------------------ forward
def _reference_attention(attn, x, cfg, rope, alibi, keep):
    """The module's attention written out in float64 with K / V heads explicitly repeated per query head."""
    W = attn.Wqkv.weight.double()
    qkv = x.double() @ W.t() + (attn.Wqkv.bias.double() if attn.Wqkv.bias is not None else 0.0)
    if cfg.clip_qkv:
        qkv = qkv.clamp(-cfg.clip_qkv, cfg.clip_qkv)
    d, kvd, H, Hkv, dh = cfg.d_model, cfg.kv_dim, cfg.n_heads, cfg.kv_n_heads, cfg.d_head
    q, k, v = qkv[..., :d], qkv[..., d:d + kvd], qkv[..., d + kvd:]
    if cfg.qk_ln:
        ln = lambda t, m: torch.nn.functional.layer_norm(t, (t.shape[-1],), m.weight.double(), m.bias.double(), cfg.norm_eps)  # noqa: E731
        q, k = ln(q, attn.q_ln), ln(k, attn.k_ln)
    B, S, _ = x.shape
    q = q.view(B, S, H, dh).transpose(1, 2)
    k, v = (t.view(B, S, Hkv, dh).transpose(1, 2) for t in (k, v))
    if rope is not None:
        q, k = apply_rope(q, rope[0][:S].double(), rope[1][:S].double()), apply_rope(k, rope[0][:S].double(), rope[1][:S].double())
    g = H // Hkv
    k = torch.stack([k[:, h // g] for h in range(H)], 1)   # query head h reads kv head h // g
    v = torch.stack([v[:, h // g] for h in range(H)], 1)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
    if alibi is not None:
        s = s + alibi[:, :, :S, :S].double()
    mask = torch.ones(S, S, dtype=torch.bool).tril()
    if keep is not None:
        mask = mask & keep
    o = torch.softmax(s.masked_fill(~mask, float("-inf")), -1) @ v
    return attn.out_proj(o.transpose(1, 2).reshape(B, S, d).float()).double()


FORWARD = [pytest.param(kv, impl, feats, id=f"kv{kv}-{impl}-{'+'.join(feats) or 'plain'}")
           for kv in (2, 1) for impl in ("flash", "torch")
           for feats in ((), ("qk_ln",), ("clip_qkv",), ("rope",), ("alibi",), ("doc",), ("qk_ln", "clip_qkv", "rope", "doc"),
                         ("alibi", "doc"))]


@pytest.mark.parametrize("kv,impl,feats", FORWARD)
def test_module_matches_repeated_kv_reference(kv, impl, feats):
    cfg = MPTConfig(d_model=64, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96, kv_n_heads=kv, attn_impl=impl,
                    qk_ln="qk_ln" in feats, clip_qkv=0.8 if "clip_qkv" in feats else None, rope="rope" in feats,
                    alibi="alibi" in feats, attn_uses_sequence_id="doc" in feats)
    model = MPTForCausalLM(cfg, seed=11)
    attn = model.transformer.blocks[0].attn
    x = torch.randn(2, 32, 64, generator=torch.Generator().manual_seed(1))
    rope, alibi = model._aux(32, x.device)   # noqa: SLF001
    sid = torch.tensor([[0] * 10 + [1] * 12 + [2] * 10, [0] * 32])
    keep = model.doc_keep(sid) if "doc" in feats else None
    got = attn(x, rope, alibi, keep).double()
    want = _reference_attention(attn, x, cfg, rope, alibi, keep)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_gqa_gradients_reach_every_kv_head_and_match_the_reference():
    cfg = MPTConfig(d_model=64, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96, kv_n_heads=2, attn_impl="flash", rope=True)
    model = MPTForCausalLM(cfg, seed=2)
    attn = model.transformer.blocks[0].attn
    x = torch.randn(2, 32, 64, generator=torch.Generator().manual_seed(4))
    rope, _ = model._aux(32, x.device)   # noqa: SLF001
    attn(x, rope, None).square().sum().backward()
    g = attn.Wqkv.weight.grad.clone()
    attn.zero_grad()
    _reference_attention(attn, x, cfg, rope, None, None).square().sum().backward()
    torch.testing.assert_close(g, attn.Wqkv.weight.grad, rtol=1e-3, atol=1e-4)
    for h in range(2):   # every kv head's k and v rows get a gradient
        assert g[64 + 8 * h: 64 + 8 * (h + 1)].abs().sum() > 0 and g[80 + 8 * h: 80 + 8 * (h + 1)].abs().sum() > 0


def test_alibi_slopes_are_per_query_head():
    cfg = MPTConfig(d_model=64, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96, kv_n_heads=1, alibi=True)
    _, alibi = MPTForCausalLM(cfg, seed=0)._aux(32, torch.device("cpu"))   # noqa: SLF001
    assert alibi.shape[1] == 8 and torch.allclose(alibi[0, :, 5, 0], -5 * alibi_slopes(8))


def test_rope_tables_rotate_kv_heads_like_query_heads():
    cos, sin = rope_tables(16, 8, 10000.0)
    k = torch.randn(1, 2, 16, 8)
    torch.testing.assert_close(apply_rope(k, cos, sin)[:, 1], apply_rope(k[:, 1:], cos, sin)[:, 0])


# ------------------------------------------------------------------------------------------------ payloads
def test_multi_head_payload_does_not_load_into_a_gqa_model():
    mha = MPTConfig(d_model=64, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96)
    gqa = MPTConfig(d_model=64, n_heads=8, n_layers=1, max_seq_len=32, vocab_size=96, kv_n_heads=2)
    src = FlatParams(MPTForCausalLM(mha, seed=0))
    dst = FlatParams(MPTForCausalLM(gqa, seed=0))
    arrays = src.layout.to_ndarrays(src.params)
    with pytest.raises(ValueError, match="attn.Wqkv"):
        dst.layout.from_ndarrays(dst.params, arrays)
    with pytest.raises(ValueError, match="attn.Wqkv"):
        src.layout.from_ndarrays(src.params, dst.layout.to_ndarrays(dst.params))


def test_federated_round_with_a_gqa_config(tmp_path):
    from photon_b200.config import compose
    from photon_b200.server_app import run_server

    tiny = ["llm_config.model.d_model=32", "llm_config.model.n_heads=4", "llm_config.model.n_layers=1", "llm_config.max_seq_len=16",
            "llm_config.global_train_batch_size=4", "llm_config.device_train_microbatch_size=2", "llm_config.device_eval_batch_size=4",
            "llm_config.local_steps=2ba", "llm_config.precision=fp32", "llm_config.model.attn_config.attn_impl=torch",
            "+llm_config.model.attn_config.attn_type=grouped_query_attention", "+llm_config.model.attn_config.kv_n_heads=2",
            "llm_config.eval_subset_num_batches=1", "llm_config.log_to_console=false", "~llm_config.loggers.wandb",
            "~llm_config.loggers.tensorboard", "~llm_config.callbacks", "llm_config.optimizer.lr=1.0e-2",
            "llm_config.scheduler.schedulers.lr.t_warmup=1ba", "fl.n_total_clients=4", "fl.n_clients_per_round=2", "photon.resume_round=null",
            f"photon.saving_path={tmp_path}", f"llm_config.save_folder={tmp_path}/clients", "run_uuid=gqa", "photon.checkpoint=true",
            "fl.n_rounds=1", "fl.strategy_name=fedavg"]
    h = run_server(compose(tiny))
    assert h.latest("server/l2_norm_pseudo_gradient") > 0
    from photon_b200.checkpoint import CheckpointStore

    with np.load(CheckpointStore(tmp_path, "checkpoints").round_dir("gqa", 1) / "current_server_parameters.npz") as z:
        assert z["arr_0"].shape == (32 + 2 * 2 * 8,)   # transformer.blocks.0.attn.Wqkv.bias: q, then 2 k heads, then 2 v heads
