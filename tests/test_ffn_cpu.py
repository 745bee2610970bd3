"""Feed-forward variants of ``model.ffn_config`` on the CPU: parsing, parameter names / layout / init of the gated block, its
math against an fp64 formula, the engine's backward plan with frozen gate tensors, the backend's fallback decision and one
federated round that carries the gate tensors."""
import math

import numpy as np
import pytest
import torch

from photon_b200.models.engine import BackwardPlan
from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, build_model, trainable_named_parameters
from photon_b200.utils.flat import FlatParams

BASE = dict(name="mpt_causal_lm", d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256)


def _cfg(ffn=None, **kw):
    m = dict(BASE, **kw)
    if ffn is not None:
        m["ffn_config"] = ffn
    return MPTConfig.from_model_cfg(m)


# ------------------------------------------------------------------------------------------------------------ parsing
def test_defaults_are_mptmlp_exact_gelu_at_expansion_ratio_width():
    c = _cfg()
    assert (c.ffn_type, c.ffn_act, c.ffn_hidden_size, c.ffn_hidden) == ("mptmlp", "gelu", None, 4 * 64)
    assert "ffn_config" not in c.extra


@pytest.mark.parametrize("ffn_type", ["mptmlp", "mptglu"])
@pytest.mark.parametrize("act,want", [({"name": "gelu"}, "gelu"), ({"name": "gelu", "approximate": "none"}, "gelu"),
                                      ({"name": "silu"}, "silu"), (None, "gelu")])
def test_supported_combinations(ffn_type, act, want):
    ffn = {"ffn_type": ffn_type}
    if act is not None:
        ffn["ffn_act_fn"] = act
    c = _cfg(ffn)
    assert (c.ffn_type, c.ffn_act, c.ffn_gated) == (ffn_type, want, ffn_type == "mptglu")


@pytest.mark.parametrize("ffn,match", [
    ({"ffn_type": "te_ln_mlp"}, "ffn_type 'te_ln_mlp'.*mptmlp, mptglu"),
    ({"ffn_type": "mb_moe"}, "ffn_type 'mb_moe'"),
    ({"ffn_type": "mb_dmoe"}, "ffn_type 'mb_dmoe'"),
    ({"ffn_act_fn": {"name": "gelu", "approximate": "tanh"}}, "ffn_act_fn.*tanh"),
    ({"ffn_act_fn": {"name": "relu"}}, "ffn_act_fn.*relu"),
    ({"ffn_act_fn": {"name": "swish_unknown"}}, "ffn_act_fn.*swish_unknown"),
    ({"ffn_type": "mptglu", "ffn_act_fn": {"name": "silu", "inplace": True}}, "ffn_act_fn"),
])
def test_rejected_values_name_what_is_supported(ffn, match):
    with pytest.raises(ValueError, match=match):
        _cfg(ffn)


def test_direct_construction_rejects_unknown_type_and_activation():
    with pytest.raises(ValueError, match="mptmlp, mptglu"):
        MPTConfig(ffn_type="mb_moe")
    with pytest.raises(ValueError, match="gelu, silu"):
        MPTConfig(ffn_act="relu")


def test_float_expansion_ratio_and_hidden_size_precedence():
    assert _cfg(expansion_ratio=2.75).ffn_hidden == int(64 * 2.75) == 176
    assert _cfg({"ffn_hidden_size": 96}, expansion_ratio=2.75).ffn_hidden == 96
    assert _cfg({"ffn_hidden_size": 96}).ffn_hidden == 96


def test_unknown_ffn_keys_stay_in_extra():
    c = _cfg({"ffn_type": "mptglu", "fc_type": {"name": "torch"}, "bias": True})
    assert c.extra["ffn_config"] == {"fc_type": {"name": "torch"}, "bias": True}


# ------------------------------------------------------------------------------------------------ names, layout, init
def test_no_ffn_config_is_bitwise_the_plain_config():
    plain = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256)
    parsed = _cfg()
    a, b = build_model(plain, seed=11), build_model(parsed, seed=11)
    na, nb = trainable_named_parameters(a), trainable_named_parameters(b)
    assert [n for n, _ in na] == [n for n, _ in nb]
    assert all(torch.equal(p, q) for (_, p), (_, q) in zip(na, nb))
    fa, fb = FlatParams(a), FlatParams(b)
    assert fa.layout.names == fb.layout.names and fa.layout.offsets == fb.layout.offsets and fa.layout.total == fb.layout.total
    assert torch.equal(fa.params, fb.params)
    assert plain.num_params() == parsed.num_params() == fa.layout.n_params


def test_gate_names_shapes_and_sorted_placement():
    c = _cfg({"ffn_type": "mptglu", "ffn_hidden_size": 192})
    names = [n for n, _ in trainable_named_parameters(build_model(c, seed=0))]
    m = dict(build_model(c, seed=0).named_parameters())
    for i in range(2):
        p = f"transformer.blocks.{i}.ffn."
        assert tuple(m[p + "gate_proj.weight"].shape) == (192, 64) and tuple(m[p + "gate_proj.bias"].shape) == (192,)
        assert tuple(m[p + "up_proj.weight"].shape) == (192, 64) and tuple(m[p + "down_proj.weight"].shape) == (64, 192)
        j = names.index(p + "gate_proj.bias")
        assert names[j - 2: j + 4] == [p + "down_proj.bias", p + "down_proj.weight", p + "gate_proj.bias", p + "gate_proj.weight",
                                       p + "up_proj.bias", p + "up_proj.weight"]
    assert all("gate_proj" not in n for n in (k for k, _ in build_model(_cfg(), seed=0).named_parameters()))


@pytest.mark.parametrize("ffn_type", ["mptmlp", "mptglu"])
@pytest.mark.parametrize("no_bias", [False, True])
@pytest.mark.parametrize("hidden", [None, 1408 // 8, 200])
def test_num_params_is_the_layout_size(ffn_type, no_bias, hidden):
    ffn = {"ffn_type": ffn_type}
    if hidden is not None:
        ffn["ffn_hidden_size"] = hidden
    c = _cfg(ffn, no_bias=no_bias, expansion_ratio=3.5)
    flat = FlatParams(build_model(c, seed=0))
    assert c.num_params() == flat.layout.n_params
    assert c.flops_per_token(32) == 6.0 * c.num_params() + 12.0 * c.n_layers * c.d_model * 32


def test_init_statistics_of_gate_and_down():
    """kaiming_normal_: std sqrt(2 / fan_in); gate_proj is an ordinary linear, down_proj keeps the 1/sqrt(2 n_layers) divisor."""
    c = MPTConfig(d_model=256, n_heads=4, n_layers=4, max_seq_len=32, vocab_size=256, ffn_type="mptglu", ffn_act="silu",
                  ffn_hidden_size=704)
    m = {k: v.detach() for k, v in build_model(c, seed=3).named_parameters()}
    g, dn, up = (m[f"transformer.blocks.1.ffn.{k}.weight"] for k in ("gate_proj", "down_proj", "up_proj"))
    assert abs(g.std().item() / math.sqrt(2 / 256) - 1) < 0.02
    assert abs(up.std().item() / math.sqrt(2 / 256) - 1) < 0.02
    assert abs(dn.std().item() / (math.sqrt(2 / 704) / math.sqrt(8)) - 1) < 0.02
    assert abs(g.mean().item()) < 3e-3 and float(m["transformer.blocks.1.ffn.gate_proj.bias"].abs().sum()) == 0.0
    assert not torch.equal(g, up)


@pytest.mark.parametrize("act", ["gelu", "silu"])
@pytest.mark.parametrize("ffn_type", ["mptmlp", "mptglu"])
def test_ffn_forward_against_fp64_formula(act, ffn_type):
    c = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, ffn_type=ffn_type, ffn_act=act,
                  ffn_hidden_size=96)
    ffn = build_model(c, seed=5).transformer.blocks[0].ffn
    with torch.no_grad():
        for mod in ffn.modules():
            if isinstance(mod, torch.nn.Linear):
                mod.bias.normal_(0, 0.1, generator=torch.Generator().manual_seed(1))
    x = torch.randn(3, 7, 64, generator=torch.Generator().manual_seed(2))
    got = ffn(x).double()
    xd = x.double()

    def lin(mod, t):
        return t @ mod.weight.double().t() + mod.bias.double()

    def f(z):
        if act == "silu":
            return z / (1 + torch.exp(-z))
        return 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))

    h = f(lin(ffn.gate_proj, xd)) * lin(ffn.up_proj, xd) if ffn_type == "mptglu" else f(lin(ffn.up_proj, xd))
    want = lin(ffn.down_proj, h)
    assert (got - want).abs().max().item() < 1e-5


# ---------------------------------------------------------------------------------------------------- backward plan
def _names(**kw):
    c = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, ffn_type="mptglu", **kw)
    return [n for n, _ in MPTForCausalLM(c, device="meta", init=False).named_parameters()]


def test_plan_without_gate_names_is_unchanged():
    names = [n for n, _ in MPTForCausalLM(MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256),
                                          device="meta", init=False).named_parameters()]
    up_frozen = [n for n in names if ".ffn.up_proj." not in n]
    p = BackwardPlan(2, up_frozen)
    assert p.block_stages(0) == p.block_stages(1) == ["down", "up", "ln2", "out", "attn", "qkv", "ln1"]
    only_down = BackwardPlan(2, [n for n in names if ".blocks.1.ffn.down_proj." in n])
    assert only_down.block_stages(1) == ["down"] and not only_down.dx((1, "down")) and only_down.lowest_block == 1


def test_plan_with_frozen_gate_still_runs_up():
    names = _names()
    frozen_gate = [n for n in names if ".ffn.gate_proj." not in n]
    p = BackwardPlan(2, frozen_gate)
    assert p.block_stages(0) == ["down", "up", "ln2", "out", "attn", "qkv", "ln1"]
    assert not p.grad("transformer.blocks.0.ffn.gate_proj.weight") and p.grad("transformer.blocks.0.ffn.up_proj.weight")


def test_plan_with_only_gate_trainable():
    names = _names()
    only_gate = [n for n in names if ".blocks.1.ffn.gate_proj." in n]
    p = BackwardPlan(2, only_gate)
    assert p.lowest_block == 1 and p.block_stages(1) == ["down", "up"]
    assert p.dx((1, "down")) and not p.dx((1, "up"))
    assert p.grad("transformer.blocks.1.ffn.gate_proj.bias") and not p.grad("transformer.blocks.1.ffn.up_proj.weight")


# ---------------------------------------------------------------------------------------------------- backend fallback
@pytest.mark.parametrize("cfg_kw,precision,zero3,fallback", [
    (dict(ffn_type="mptglu"), "amp_fp8", None, True),
    (dict(ffn_act="silu"), "amp_fp8", None, True),
    (dict(ffn_type="mptglu", ffn_act="silu"), "amp_bf16", object(), True),
    (dict(ffn_hidden_size=192), "amp_fp8", None, False),
    (dict(ffn_type="mptglu", ffn_act="silu"), "amp_bf16", None, False),
])
def test_build_backend_falls_back_for_gated_ffn_under_fp8_or_zero3(monkeypatch, capsys, cfg_kw, precision, zero3, fallback):
    import photon_b200.models.engine as engine_mod
    from photon_b200.train import backend

    made = {}

    class FakeEngine:
        def __init__(self, cfg, **kw):
            made["engine"] = kw

    class FakeTorch:
        def __init__(self, cfg, **kw):
            made["torch"] = kw

    monkeypatch.setattr(engine_mod, "B200Engine", FakeEngine)
    monkeypatch.setattr(backend, "TorchBackend", FakeTorch)
    cfg = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, **cfg_kw)
    kw = {"zero3": zero3} if zero3 is not None else {}
    backend.build_backend(cfg, torch.device("cuda", 0), precision, **kw)
    assert ("torch" in made) == fallback and ("engine" in made) != fallback
    out = capsys.readouterr().out
    if fallback:
        assert "ffn_config" in out and "stock PyTorch backend" in out and "zero3" not in made["torch"]


# ------------------------------------------------------------------------------------------------- federated round
def test_one_federated_round_carries_the_gate(tmp_path):
    from photon_b200.config import compose
    from photon_b200.federation import FederationRuntime
    from photon_b200.server_app import run_server
    from test_federation_cpu import TINY

    cfg = compose(TINY + [f"photon.saving_path={tmp_path}", f"llm_config.save_folder={tmp_path}/clients", "run_uuid=glu",
                          "fl.n_rounds=1", "++llm_config.model.ffn_config.ffn_type=mptglu",
                          "++llm_config.model.ffn_config.ffn_act_fn.name=silu"])
    rt = FederationRuntime(cfg, device=torch.device("cpu"), rank=0, world_size=1)
    h = run_server(cfg, runtime=rt)
    names = rt.model_layout.names
    assert "transformer.blocks.0.ffn.gate_proj.weight" in names and "transformer.blocks.0.ffn.gate_proj.bias" in names
    fit = h.metrics_distributed_fit
    assert [v for _, v in fit["server/n_failures"]] == [0]
    assert all(np.isfinite(v) for _, v in fit["server/l2_norm_pseudo_gradient"])
    g = rt.round_backend.global_params()
    gate = rt.model_layout.view(g, "transformer.blocks.0.ffn.gate_proj.weight")
    assert gate.shape == (4 * 32, 32) and float(gate.abs().sum()) > 0
    rt.close()
