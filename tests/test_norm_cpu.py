"""``model.norm_type`` / ``model.norm_eps`` on the CPU: parsing, parameter names / layout / init of RMSNorm models, the
PyTorch forward against an fp64 ``rms_norm`` formula, the engine's backward plan with frozen norm weights, what happens when
a LayerNorm payload meets an RMSNorm model, and one federated round that carries an RMSNorm model."""
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from photon_b200.models.engine import BackwardPlan
from photon_b200.models.mpt import NORM_TYPES, MPTConfig, MPTForCausalLM, RMSNorm, build_model, trainable_named_parameters
from photon_b200.utils.flat import FlatParams

BASE = dict(name="mpt_causal_lm", d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256)
GOLDEN = Path(__file__).parent / "golden" / "norm_default_params.json"


def _cfg(**kw):
    return MPTConfig.from_model_cfg(dict(BASE, **kw))


def _norms(model):
    return {n: m for n, m in model.named_modules() if isinstance(m, (torch.nn.LayerNorm, RMSNorm))}


# ------------------------------------------------------------------------------------------------------------ parsing
@pytest.mark.parametrize("name,kind", [("layernorm", "layernorm"), ("low_precision_layernorm", "layernorm"),
                                       ("rmsnorm", "rmsnorm"), ("low_precision_rmsnorm", "rmsnorm"),
                                       ("triton_rmsnorm", "rmsnorm"), ("RMSNorm", "rmsnorm")])
def test_the_five_registry_names_parse(name, kind):
    c = _cfg(norm_type=name)
    assert c.norm_type == kind and c.rmsnorm == (kind == "rmsnorm")
    assert "norm_type" not in c.extra
    want = RMSNorm if kind == "rmsnorm" else torch.nn.LayerNorm
    assert all(isinstance(m, want) for m in _norms(build_model(c, seed=0)).values())


def test_default_is_layernorm_at_1e_5():
    c = _cfg()
    assert (c.norm_type, c.norm_eps, c.rmsnorm) == ("layernorm", 1e-5, False)
    assert set(NORM_TYPES) == {"layernorm", "low_precision_layernorm", "rmsnorm", "low_precision_rmsnorm", "triton_rmsnorm"}


@pytest.mark.parametrize("bad", ["groupnorm", "te_layernorm", "rms_norm"])
def test_unknown_norm_type_names_what_is_supported(bad):
    with pytest.raises(ValueError, match=f"norm_type '{bad}'.*layernorm, low_precision_layernorm, rmsnorm"):
        _cfg(norm_type=bad)
    with pytest.raises(ValueError, match="triton_rmsnorm"):
        MPTConfig(norm_type=bad)


@pytest.mark.parametrize("norm_type", ["layernorm", "rmsnorm"])
def test_norm_eps_reaches_every_norm(norm_type):
    c = _cfg(norm_type=norm_type, norm_eps=1e-6, attn_config={"qk_ln": True})
    assert c.norm_eps == 1e-6 and "norm_eps" not in c.extra
    norms = _norms(build_model(c, seed=0))
    assert len(norms) == 2 * 2 + 1 + 2 * 2
    assert all(m.eps == 1e-6 for m in norms.values())


# ------------------------------------------------------------------------------------------------ names, layout, init
@pytest.mark.parametrize("case", ["default", "no_bias", "qk_ln_gqa_rope"])
def test_configs_without_norm_type_are_bitwise_the_parent_commit(case):
    """Names, shapes, num_params and the initial values of configs that do not set ``norm_type``, against what the commit
    before it was read recorded."""
    want = json.loads(GOLDEN.read_text())[case]
    cfg = MPTConfig.from_model_cfg(want["model"])
    named = trainable_named_parameters(build_model(cfg, seed=11))
    h = hashlib.sha256()
    for _, p in named:
        h.update(p.detach().contiguous().numpy().tobytes())
    assert [n for n, _ in named] == want["names"]
    assert [list(p.shape) for _, p in named] == want["shapes"]
    assert h.hexdigest() == want["sha256"]
    assert cfg.num_params() == want["num_params"] and cfg.norm_eps == want["norm_eps"]


def test_rmsnorm_names_shapes_and_sorted_placement():
    c = _cfg(norm_type="rmsnorm", attn_config={"qk_ln": True, "attn_type": "grouped_query_attention", "kv_n_heads": 2})
    model = build_model(c, seed=0)
    m = dict(model.named_parameters())
    names = [n for n, _ in trainable_named_parameters(model)]
    assert not any(n.endswith("ln.bias") or (".norm_" in n and n.endswith(".bias")) for n in names)
    for i in range(2):
        p = f"transformer.blocks.{i}."
        for k in ("norm_1", "norm_2", "attn.q_ln"):
            assert tuple(m[p + k + ".weight"].shape) == (64,)
        assert tuple(m[p + "attn.k_ln.weight"].shape) == (2 * 16,)
        j = names.index(p + "attn.Wqkv.bias")
        assert names[j: j + 6] == [p + "attn.Wqkv.bias", p + "attn.Wqkv.weight", p + "attn.k_ln.weight", p + "attn.out_proj.bias",
                                   p + "attn.out_proj.weight", p + "attn.q_ln.weight"]
        assert names[names.index(p + "ffn.up_proj.weight") + 1: names.index(p + "ffn.up_proj.weight") + 3] == [p + "norm_1.weight",
                                                                                                         p + "norm_2.weight"]
    assert names[-3:] == ["transformer.norm_f.weight", "transformer.wpe.weight", "transformer.wte.weight"]


@pytest.mark.parametrize("ffn_type", ["mptmlp", "mptglu"])
@pytest.mark.parametrize("no_bias", [False, True])
@pytest.mark.parametrize("norm_type", ["layernorm", "rmsnorm"])
def test_num_params_is_the_layout_size(ffn_type, no_bias, norm_type):
    c = _cfg(norm_type=norm_type, no_bias=no_bias, ffn_config={"ffn_type": ffn_type})
    flat = FlatParams(build_model(c, seed=0))
    assert c.num_params() == flat.layout.n_params
    assert c.flops_per_token(32) == 6.0 * c.num_params() + 12.0 * c.n_layers * c.d_model * 32


def test_rmsnorm_init_is_ones_and_the_rest_is_the_layernorm_model():
    """RMSNorm weights start at one; every other tensor gets the same initial values as the LayerNorm model of that seed (norms
    draw no random numbers)."""
    ln, rms = (dict(build_model(_cfg(norm_type=t), seed=4).named_parameters()) for t in ("layernorm", "rmsnorm"))
    for n, p in rms.items():
        if ".norm_" in n or "norm_f" in n:
            assert torch.equal(p, torch.ones_like(p))
        else:
            assert torch.equal(p, ln[n]), n
    assert set(ln) - set(rms) == {f"transformer.blocks.{i}.norm_{k}.bias" for i in range(2) for k in (1, 2)} | {"transformer.norm_f.bias"}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rmsnorm_forward_against_fp64_formula(dtype):
    c = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, norm_type="rmsnorm", norm_eps=1e-3)
    norm = build_model(c, seed=5).transformer.blocks[0].norm_1
    with torch.no_grad():
        norm.weight.normal_(1.0, 0.3, generator=torch.Generator().manual_seed(1))
    x = (torch.randn(3, 7, 64, generator=torch.Generator().manual_seed(2)) * 3 + 0.5).to(dtype)
    got = norm(x)
    assert got.dtype == dtype
    xd = x.double()
    want = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-3) * norm.weight.double()
    tol = 1e-5 if dtype == torch.float32 else 2 ** -8 * 4
    assert (got.double() - want).abs().max().item() <= tol * max(1.0, want.abs().max().item())
    assert not hasattr(norm, "bias")


def test_model_forward_runs_rmsnorm_everywhere():
    """The whole model against itself with every norm replaced by the fp64 formula: the norms are the only difference."""
    c = _cfg(norm_type="rmsnorm", attn_config={"qk_ln": True, "attn_impl": "torch"}, no_bias=True)
    model = build_model(c, seed=3).double()
    ids = torch.randint(0, 256, (2, 16), generator=torch.Generator().manual_seed(0))
    got = model(ids)

    def formula(self, x):
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps) * self.weight

    orig = RMSNorm.forward
    RMSNorm.forward = formula
    try:
        want = model(ids)
    finally:
        RMSNorm.forward = orig
    # the module computes in fp32: the difference is fp32 rounding, not a different function
    assert (got - want).abs().max().item() < 1e-4


# ---------------------------------------------------------------------------------------------------- backward plan
def _names(**kw):
    c = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, norm_type="rmsnorm", **kw)
    return [n for n, _ in MPTForCausalLM(c, device="meta", init=False).named_parameters()]


def test_plan_with_frozen_norm_weights():
    names = _names(qk_ln=True)
    frozen_norms = [n for n in names if not n.endswith("norm_1.weight") and not n.endswith("norm_2.weight") and "_ln." not in n
                    and "norm_f" not in n]
    p = BackwardPlan(2, frozen_norms)
    assert p.block_stages(0) == p.block_stages(1) == ["down", "up", "ln2", "out", "attn", "qkv", "ln1"]
    assert p.runs("norm_f") and not p.grad("transformer.norm_f.weight") and not p.grad("transformer.blocks.0.attn.q_ln.weight")


def test_plan_with_only_norm_weights_trainable():
    names = _names()
    only = [n for n in names if n.endswith(".blocks.1.norm_2.weight") or n.endswith("norm_f.weight")]
    p = BackwardPlan(2, only)
    assert p.lowest_block == 1 and p.block_stages(1) == ["down", "up", "ln2"]
    assert p.dx((1, "up")) and not p.dx((1, "ln2")) and p.runs("norm_f") and p.dx("norm_f")
    only_qk = BackwardPlan(2, [n for n in _names(qk_ln=True) if n.endswith(".blocks.0.attn.k_ln.weight")])
    assert only_qk.block_stages(0) == ["down", "up", "ln2", "out", "attn"] and not only_qk.dx((0, "attn"))


# ---------------------------------------------------------------------------------------- LayerNorm payload -> RMSNorm
def test_a_layernorm_payload_does_not_load_into_an_rmsnorm_model():
    from photon_b200.utils.core import set_parameters

    ln_model, rms_model = (build_model(_cfg(norm_type=t), seed=0) for t in ("layernorm", "rmsnorm"))
    payload = FlatParams(ln_model).layout.to_ndarrays(FlatParams(ln_model).params)
    rms_flat = FlatParams(rms_model)
    with pytest.raises(ValueError, match=r"expected 23 arrays, got 28"):
        rms_flat.layout.from_ndarrays(rms_flat.params, payload)
    with pytest.raises(ValueError, match=r"28 arrays for 23 trainable tensors"):
        set_parameters(rms_model, payload)
    # q_ln / k_ln keep their bias under no_bias, so a no_bias LayerNorm payload with qk_ln still differs in count ...
    qk = dict(no_bias=True, attn_config={"qk_ln": True})
    ln_qk, rms_qk = (FlatParams(build_model(_cfg(norm_type=t, **qk), seed=0)) for t in ("layernorm", "rmsnorm"))
    with pytest.raises(ValueError, match="expected 19 arrays, got 23"):
        rms_qk.layout.from_ndarrays(rms_qk.params, ln_qk.layout.to_ndarrays(ln_qk.params))
    # ... while without qk_ln a no_bias LayerNorm model has exactly the tensors of an RMSNorm model: nothing can tell them apart
    a, b = (FlatParams(build_model(_cfg(norm_type=t, no_bias=True), seed=0)) for t in ("layernorm", "rmsnorm"))
    assert a.layout.names == b.layout.names and a.layout.shapes == b.layout.shapes


# ------------------------------------------------------------------------------------------------- federated round
def test_one_federated_round_carries_an_rmsnorm_model(tmp_path):
    from photon_b200.config import compose
    from photon_b200.federation import FederationRuntime
    from photon_b200.server_app import run_server
    from test_federation_cpu import TINY

    cfg = compose(TINY + [f"photon.saving_path={tmp_path}", f"llm_config.save_folder={tmp_path}/clients", "run_uuid=rms",
                          "fl.n_rounds=1", "++llm_config.model.norm_type=rmsnorm", "++llm_config.model.norm_eps=1e-6"])
    rt = FederationRuntime(cfg, device=torch.device("cpu"), rank=0, world_size=1)
    h = run_server(cfg, runtime=rt)
    names = rt.model_layout.names
    assert "transformer.blocks.0.norm_1.weight" in names and "transformer.norm_f.weight" in names
    assert not any(".norm_" in n and n.endswith(".bias") for n in names) and "transformer.norm_f.bias" not in names
    fit = h.metrics_distributed_fit
    assert [v for _, v in fit["server/n_failures"]] == [0]
    assert all(np.isfinite(v) for _, v in fit["server/l2_norm_pseudo_gradient"])
    g = rt.round_backend.global_params()
    w = rt.model_layout.view(g, "transformer.blocks.0.norm_1.weight")
    assert w.shape == (32,) and float((w - 1).abs().sum()) > 0   # trained away from its initial ones
    rt.close()


# ---------------------------------------------------------------------------------------------------- backend choice
@pytest.mark.parametrize("precision,zero3", [("amp_bf16", None), ("amp_fp8", None), ("amp_bf16", object()), ("amp_fp8", object())])
def test_build_backend_keeps_rmsnorm_on_the_engine(monkeypatch, capsys, precision, zero3):
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
    cfg = MPTConfig(d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256, norm_type="rmsnorm", qk_ln=True)
    kw = {"zero3": zero3} if zero3 is not None else {}
    backend.build_backend(cfg, torch.device("cuda", 0), precision, **kw)
    assert "engine" in made and "torch" not in made
    assert "stock PyTorch backend" not in capsys.readouterr().out
