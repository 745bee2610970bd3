"""``attn_config.sliding_window_size`` / ``attn_config.softmax_scale`` on the CPU: parsing and rejection, an unchanged
parameter set, the PyTorch module's mask against a float64 formula (alone, with the document mask and with ALiBi), a window
as wide as the sequence being bitwise causal attention, the explicit and SDPA branches agreeing, the scale reaching the
scores, and one federated round with both keys."""
import math

import numpy as np
import pytest
import torch

from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, apply_rope, window_keep
from photon_b200.utils.flat import FlatParams

BASE = dict(name="mpt_causal_lm", d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256)


def _cfg(**attn):
    return MPTConfig.from_model_cfg(dict(BASE, attn_config=attn))


# ------------------------------------------------------------------------------------------------------------ parsing
def test_defaults_are_off():
    c = _cfg()
    assert c.sliding_window_size == -1 and c.softmax_scale is None
    assert c.attn_scale == 1.0 / math.sqrt(c.d_head)


def test_both_keys_parse_and_leave_extra():
    c = _cfg(sliding_window_size=7, softmax_scale=0.25, rope_theta=500.0)
    assert (c.sliding_window_size, c.softmax_scale, c.attn_scale) == (7, 0.25, 0.25)
    assert "attn_config" not in c.extra
    c = _cfg(sliding_window_size=0, softmax_scale=2)
    assert c.sliding_window_size == 0 and c.softmax_scale == 2.0 and isinstance(c.softmax_scale, float)
    assert _cfg(sliding_window_size=-1, softmax_scale=None).sliding_window_size == -1
    assert _cfg(sliding_window_size=np.int64(5)).sliding_window_size == 5


@pytest.mark.parametrize("bad", [-2, -100, 3.0, 2.5, "8", True, None])
def test_bad_window_is_refused(bad):
    with pytest.raises(ValueError, match="sliding_window_size"):
        _cfg(sliding_window_size=bad)
    with pytest.raises(ValueError, match="sliding_window_size"):
        MPTConfig(sliding_window_size=bad)


@pytest.mark.parametrize("bad", [0, 0.0, -0.5, float("inf"), float("nan"), "0.1", True])
def test_bad_softmax_scale_is_refused(bad):
    with pytest.raises(ValueError, match="softmax_scale"):
        _cfg(softmax_scale=bad)
    with pytest.raises(ValueError, match="softmax_scale"):
        MPTConfig(softmax_scale=bad)


@pytest.mark.parametrize("extra", [dict(), dict(attn_type="grouped_query_attention", kv_n_heads=2, rope=True)])
def test_keys_add_no_parameter(extra):
    plain, win = _cfg(**extra), _cfg(sliding_window_size=5, softmax_scale=0.3, **extra)
    a, b = MPTForCausalLM(plain, seed=3), MPTForCausalLM(win, seed=3)
    assert plain.num_params() == win.num_params() == sum(p.numel() for p in b.parameters())
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert FlatParams(a).layout.total == FlatParams(b).layout.total
    assert plain.flops_per_token() == win.flops_per_token()


# ------------------------------------------------------------------------------------------------------------ masks
def test_window_keep_formula():
    assert window_keep(16, -1) is None and window_keep(16, 15) is None and window_keep(16, 40) is None
    for W in (0, 1, 3, 14):
        i, j = torch.arange(16)[:, None], torch.arange(16)[None, :]
        keep = window_keep(16, W)
        assert torch.equal(keep & (j <= i), (j <= i) & (j >= i - W))
        assert int((keep & (j <= i))[15].sum()) == W + 1   # the last row sees W + 1 keys, its own included


def _reference(attn, x, cfg, rope, alibi, keep, window, scale):
    """The attention of one block in float64, with the mask written out element by element."""
    qkv = x.double() @ attn.Wqkv.weight.double().t() + attn.Wqkv.bias.double()
    d, kvd, H, Hkv, dh = cfg.d_model, cfg.kv_dim, cfg.n_heads, cfg.kv_n_heads, cfg.d_head
    B, S, _ = x.shape
    q = qkv[..., :d].view(B, S, H, dh).transpose(1, 2)
    k, v = (t.view(B, S, Hkv, dh).transpose(1, 2) for t in (qkv[..., d:d + kvd], qkv[..., d + kvd:]))
    if rope is not None:
        q, k = (apply_rope(t, rope[0][:S].double(), rope[1][:S].double()) for t in (q, k))
    g = H // Hkv
    k, v = k.repeat_interleave(g, 1), v.repeat_interleave(g, 1)
    s = (q @ k.transpose(-1, -2)) * scale
    if alibi is not None:
        s = s + alibi[:, :, :S, :S].double()
    mask = torch.zeros(B, 1, S, S, dtype=torch.bool)
    for b in range(B):
        for i in range(S):
            for j in range(S):
                mask[b, 0, i, j] = j <= i and (window < 0 or i - window <= j) and (keep is None or bool(keep[b, 0, i, j]))
    o = torch.softmax(s.masked_fill(~mask, float("-inf")), -1) @ v
    return attn.out_proj(o.transpose(1, 2).reshape(B, S, d).float()).double()


CASES = [pytest.param(W, impl, feats, id=f"W{W}-{impl}-{'+'.join(feats) or 'plain'}")
         for W in (0, 1, 5, 30) for impl in ("flash", "torch")
         for feats in ((), ("doc",), ("alibi",), ("alibi", "doc"), ("gqa", "rope", "scale"))]


@pytest.mark.parametrize("W,impl,feats", CASES)
def test_module_against_fp64_formula(W, impl, feats):
    scale = 0.4 if "scale" in feats else None
    cfg = MPTConfig(d_model=64, n_heads=4, n_layers=1, max_seq_len=32, vocab_size=96, attn_impl=impl, alibi="alibi" in feats,
                    rope="rope" in feats, kv_n_heads=2 if "gqa" in feats else None, attn_uses_sequence_id="doc" in feats,
                    sliding_window_size=W, softmax_scale=scale)
    model = MPTForCausalLM(cfg, seed=5)
    attn = model.transformer.blocks[0].attn
    x = torch.randn(2, 32, 64, generator=torch.Generator().manual_seed(2))
    rope, alibi = model._aux(32, x.device)   # noqa: SLF001
    keep = model.doc_keep(torch.tensor([[0] * 9 + [1] * 13 + [2] * 10, [0] * 32])) if "doc" in feats else None
    got = attn(x, rope, alibi, keep).double()
    want = _reference(attn, x, cfg, rope, alibi, keep, W, cfg.attn_scale)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("impl", ["flash", "torch"])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("W", [31, 32, 1000])
def test_window_as_wide_as_the_sequence_is_bitwise_causal(impl, alibi, W):
    kw = dict(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=96, attn_impl=impl, alibi=alibi)
    ids = torch.randint(0, 96, (2, 32), generator=torch.Generator().manual_seed(0))
    a = MPTForCausalLM(MPTConfig(**kw), seed=1)(ids)
    b = MPTForCausalLM(MPTConfig(**kw, sliding_window_size=W), seed=1)(ids)
    assert torch.equal(a, b)


@pytest.mark.parametrize("feats", [(), ("doc",), ("alibi",)])
def test_explicit_and_sdpa_branches_agree(feats):
    ids = torch.randint(0, 96, (2, 32), generator=torch.Generator().manual_seed(3))
    sid = torch.tensor([[0] * 12 + [1] * 20, [0] * 32]) if "doc" in feats else None
    out = {}
    for impl in ("flash", "torch"):
        cfg = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=96, attn_impl=impl, alibi="alibi" in feats,
                        attn_uses_sequence_id="doc" in feats, sliding_window_size=6, softmax_scale=0.3)
        out[impl] = MPTForCausalLM(cfg, seed=4)(ids, sid)
    torch.testing.assert_close(out["flash"], out["torch"], rtol=1e-4, atol=1e-5)


def test_window_changes_the_output():
    ids = torch.randint(0, 96, (1, 32), generator=torch.Generator().manual_seed(6))
    kw = dict(d_model=64, n_heads=4, n_layers=1, max_seq_len=32, vocab_size=96)
    a = MPTForCausalLM(MPTConfig(**kw), seed=1)(ids)
    b = MPTForCausalLM(MPTConfig(**kw, sliding_window_size=4), seed=1)(ids)
    assert torch.equal(a[:, :5], b[:, :5])           # rows 0 .. 4 see all their keys either way
    assert not torch.allclose(a[:, 5:], b[:, 5:])


@pytest.mark.parametrize("impl", ["flash", "torch"])
def test_softmax_scale_reaches_the_scores(impl):
    kw = dict(d_model=64, n_heads=4, n_layers=1, max_seq_len=32, vocab_size=96, attn_impl=impl)
    ids = torch.randint(0, 96, (1, 32), generator=torch.Generator().manual_seed(7))
    default = MPTForCausalLM(MPTConfig(**kw), seed=1)(ids)
    explicit = MPTForCausalLM(MPTConfig(**kw, softmax_scale=1.0 / math.sqrt(16)), seed=1)(ids)
    assert torch.equal(default, explicit)
    # a scale of 0 is refused, but a tiny one makes attention uniform over the visible keys: row i is the mean of v_0..v_i
    m = MPTForCausalLM(MPTConfig(**kw, softmax_scale=1e-30), seed=1)
    attn = m.transformer.blocks[0].attn
    x = torch.randn(1, 32, 64, generator=torch.Generator().manual_seed(8))
    v = (x @ attn.Wqkv.weight.t() + attn.Wqkv.bias)[..., 128:]
    mean = torch.cumsum(v, 1) / torch.arange(1, 33)[None, :, None]
    torch.testing.assert_close(attn(x, None, None), attn.out_proj(mean), rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------- federated round
def test_one_federated_round_with_window_and_scale(tmp_path):
    from photon_b200.config import compose
    from photon_b200.server_app import run_server

    tiny = ["llm_config.model.d_model=32", "llm_config.model.n_heads=4", "llm_config.model.n_layers=1", "llm_config.max_seq_len=16",
            "llm_config.global_train_batch_size=4", "llm_config.device_train_microbatch_size=2", "llm_config.device_eval_batch_size=4",
            "llm_config.local_steps=2ba", "llm_config.precision=fp32", "llm_config.model.attn_config.attn_impl=torch",
            "+llm_config.model.attn_config.sliding_window_size=4", "+llm_config.model.attn_config.softmax_scale=0.3",
            "llm_config.eval_subset_num_batches=1", "llm_config.log_to_console=false", "~llm_config.loggers.wandb",
            "~llm_config.loggers.tensorboard", "~llm_config.callbacks", "llm_config.optimizer.lr=1.0e-2",
            "llm_config.scheduler.schedulers.lr.t_warmup=1ba", "fl.n_total_clients=4", "fl.n_clients_per_round=2", "photon.resume_round=null",
            f"photon.saving_path={tmp_path}", f"llm_config.save_folder={tmp_path}/clients", "run_uuid=win", "photon.checkpoint=true",
            "fl.n_rounds=1", "fl.strategy_name=fedavg"]
    h = run_server(compose(tiny))
    assert h.latest("server/l2_norm_pseudo_gradient") > 0
