"""The LM head keys ``tie_word_embeddings``, ``logit_scale`` and ``final_logit_softcapping`` on the CPU: parsing and rejection,
unchanged defaults, the untied head's name, place, size and init, the module's logits / loss / gradients against a float64
formula, the ZeRO-3 unit plan with a head unit, the backward plan's stages, and one federated round with an untied head."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from photon_b200.models.engine import BackwardPlan
from photon_b200.models.mpt import MPTConfig, MPTForCausalLM, build_model, head_transform, shift_labels
from photon_b200.train.backend import apply_freeze
from photon_b200.utils.flat import FlatParams, layout_for_model_cfg

BASE = dict(name="mpt_causal_lm", d_model=64, n_heads=4, n_layers=2, max_seq_len=32, vocab_size=256)
KEYS = ("tie_word_embeddings", "logit_scale", "final_logit_softcapping")


def _cfg(**kw):
    return MPTConfig.from_model_cfg(dict(BASE, **kw))


# ------------------------------------------------------------------------------------------------------------ parsing
def test_defaults_are_a_tied_untransformed_head():
    c = _cfg()
    assert c.tie_word_embeddings is True and c.logit_scale is None and c.final_logit_softcapping is None
    assert c.head_scale is None and not c.head_transformed


def test_keys_parse_and_leave_extra():
    c = _cfg(tie_word_embeddings=False, logit_scale="inv_sqrt_d_model", final_logit_softcapping=30)
    assert not any(k in c.extra for k in KEYS)
    assert c.tie_word_embeddings is False and c.head_scale == 1.0 / math.sqrt(64) and c.final_logit_softcapping == 30.0
    assert c.head_transformed
    c = _cfg(logit_scale=0.5, tie_word_embeddings=np.bool_(True))
    assert c.head_scale == 0.5 and isinstance(c.logit_scale, float) and c.tie_word_embeddings is True
    assert _cfg(final_logit_softcapping=5).head_transformed and _cfg(logit_scale=None).head_scale is None


@pytest.mark.parametrize("bad", ["false", 0, 1, None, "no"])
def test_non_bool_tie_word_embeddings_is_refused(bad):
    with pytest.raises(ValueError, match="tie_word_embeddings"):
        _cfg(tie_word_embeddings=bad)


@pytest.mark.parametrize("bad", ["inv_sqrt_d_head", "sqrt", "", 0, -0.5, float("inf"), float("nan"), True])
def test_bad_logit_scale_is_refused(bad):
    with pytest.raises(ValueError, match="logit_scale"):
        _cfg(logit_scale=bad)
    with pytest.raises(ValueError, match="logit_scale"):
        MPTConfig(logit_scale=bad)


@pytest.mark.parametrize("bad", [0, -30.0, float("inf"), float("nan"), "30", True])
def test_bad_softcap_is_refused(bad):
    with pytest.raises(ValueError, match="final_logit_softcapping"):
        _cfg(final_logit_softcapping=bad)


# ------------------------------------------------------------------------------------------------------------ parameters
@pytest.mark.parametrize("extra", [dict(), dict(no_bias=True, norm_type="rmsnorm")])
def test_defaults_change_no_parameter(extra):
    plain = _cfg(**extra)
    explicit = _cfg(tie_word_embeddings=True, logit_scale=None, final_logit_softcapping=None, **extra)
    a, b = MPTForCausalLM(plain, seed=3), MPTForCausalLM(explicit, seed=3)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert plain.num_params() == explicit.num_params() == sum(p.numel() for p in a.parameters())
    assert FlatParams(a).layout.names == FlatParams(b).layout.names
    ids = torch.randint(0, 256, (2, 32), generator=torch.Generator().manual_seed(0))
    assert torch.equal(a(ids), b(ids))


def test_untied_head_name_place_size_and_init():
    tied, untied = _cfg(), _cfg(tie_word_embeddings=False)
    a, b = MPTForCausalLM(tied, seed=3), MPTForCausalLM(untied, seed=3)
    assert b.lm_head.weight.shape == (256, 64) and b.lm_head.bias is None
    lay = FlatParams(b).layout
    assert lay.names[0] == "lm_head.weight" and lay.offsets[0] == 0
    assert untied.num_params() == tied.num_params() + 256 * 64 == sum(p.numel() for p in b.parameters())
    assert untied.flops_per_token() == tied.flops_per_token() + 6.0 * 256 * 64
    # the transformer's seeded values are those of the tied model: lm_head is initialised after them
    sa = a.state_dict()
    assert all(torch.equal(sa[k], v) for k, v in b.state_dict().items() if k != "lm_head.weight")
    big = MPTForCausalLM(MPTConfig(d_model=256, n_heads=4, n_layers=1, max_seq_len=16, vocab_size=4096, tie_word_embeddings=False),
                         seed=1)
    std = float(big.lm_head.weight.detach().std())
    assert abs(std - math.sqrt(2.0 / 256)) < 0.01 * math.sqrt(2.0 / 256)   # kaiming normal, fan_in d_model
    assert abs(float(big.lm_head.weight.mean())) < 1e-3


def test_tied_payload_does_not_load_into_an_untied_config():
    from photon_b200.utils.core import set_parameters

    tied, untied = (build_model(_cfg(tie_word_embeddings=t), seed=0) for t in (True, False))
    payload = FlatParams(tied).layout.to_ndarrays(FlatParams(tied).params)
    flat = FlatParams(untied)
    n = len(payload)
    with pytest.raises(ValueError, match=f"expected {n + 1} arrays, got {n}"):
        flat.layout.from_ndarrays(flat.params, payload)
    with pytest.raises(ValueError, match=f"{n} arrays for {n + 1} trainable tensors"):
        set_parameters(untied, payload)


# ------------------------------------------------------------------------------------------------------ fp64 formula
def _fp64_head(h, w, scale, cap):
    x = h.double() @ w.double().t()
    y = x * (scale if scale is not None else 1.0)
    if cap is not None:
        y = cap * torch.tanh(y / cap)
    return y


@pytest.mark.parametrize("tied", [True, False])
@pytest.mark.parametrize("cap", [None, 30.0, 5.0])
@pytest.mark.parametrize("scale", [1.0, 0.3, "inv_sqrt_d_model"])
def test_module_logits_loss_and_gradients_against_fp64(scale, cap, tied):
    cfg = MPTConfig(d_model=64, n_heads=4, n_layers=1, max_seq_len=16, vocab_size=96, tie_word_embeddings=tied, logit_scale=scale,
                    final_logit_softcapping=cap)
    m = MPTForCausalLM(cfg, seed=2)
    w = m.transformer.wte.weight if tied else m.lm_head.weight
    with torch.no_grad():   # large logits: the cap saturates
        w.mul_(40.0)
    ids = torch.randint(0, 96, (2, 16), generator=torch.Generator().manual_seed(1))
    h = m.hidden_states(ids).detach()
    want = _fp64_head(h, w.detach(), cfg.head_scale, cap)
    got = m(ids)
    assert got.dtype == (torch.float32 if cfg.head_transformed else h.dtype)
    torch.testing.assert_close(got.double(), want, rtol=2e-5, atol=2e-4)
    if cap is not None:
        assert float(got.abs().max()) <= cap
    if cap == 5.0:
        assert float(want.abs().max()) > 0.999 * cap   # saturated logits are covered
    # loss and gradients w.r.t. the head weight and the final hidden state, against autograd in float64
    loss, n = m.loss(ids)
    loss.backward()
    h64 = h.double().requires_grad_(True)
    w64 = w.detach().double().requires_grad_(True)
    t = shift_labels(ids).view(-1)
    ref = F.cross_entropy(_fp64_head(h64, w64, cfg.head_scale, cap).view(-1, 96), t, ignore_index=-100, reduction="sum") / int(n)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)) + 1e-6
    gw = w.grad if not tied else None
    if gw is not None:
        torch.testing.assert_close(gw.double(), w64.grad, rtol=1e-4, atol=1e-7)
    # the scale and cap reach the transform as the shared helper computes it
    torch.testing.assert_close(head_transform(torch.tensor([0.0, 3.0, -1e4]), 0.5, 5.0),
                               torch.tensor([0.0, 5.0 * math.tanh(1.5 / 5.0), -5.0]))


def test_untied_head_gives_wte_no_head_gradient():
    cfg = MPTConfig(d_model=64, n_heads=4, n_layers=1, max_seq_len=16, vocab_size=96, tie_word_embeddings=False)
    m = MPTForCausalLM(cfg, seed=2)
    ids = torch.randint(0, 96, (1, 16), generator=torch.Generator().manual_seed(1))
    m.loss(ids)[0].backward()
    used = torch.zeros(96, dtype=torch.bool)
    used[ids.view(-1)] = True
    g = m.transformer.wte.weight.grad
    assert float(g[~used].abs().max()) == 0.0 and float(g[used].abs().max()) > 0   # only the embedded rows
    assert float(m.lm_head.weight.grad.abs().min(dim=1).values.max()) > 0


# ------------------------------------------------------------------------------------------------------- ZeRO-3 plan
MC = {"name": "mpt_causal_lm", "d_model": 128, "n_heads": 4, "n_layers": 12, "expansion_ratio": 4, "max_seq_len": 64, "vocab_size": 512}


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_unit_plan_with_a_head_unit_partitions_the_flat_space(n):
    from photon_b200.parallel.zero3 import UnitPlan

    lay = layout_for_model_cfg(dict(MC, tie_word_embeddings=False))
    pl = UnitPlan(lay, 12, n)
    spans = sorted((u.lo, u.hi) for u in pl.units)
    assert spans[0][0] == 0 and spans[-1][1] == lay.total and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert [u.name for u in pl.units] == [f"block.{i}" for i in range(12)] + ["rest", "head"]
    assert pl.head == 13 and pl.rest == 12 and pl.resident_unit(13) and pl.resident_unit(12) and not pl.resident_unit(0)
    assert pl.units[pl.head].lo == 0 and pl.units[pl.head].hi == lay.offsets[lay.index("transformer.blocks.0.attn.Wqkv.bias")]
    for i, name in enumerate(lay.names):
        u = pl.units[pl.unit_of[i]]
        assert u.lo <= lay.offsets[i] and lay.offsets[i] + lay.numels[i] <= u.hi, name
    assert pl.unit_of[lay.index("lm_head.weight")] == pl.head
    assert all(u.per % 256 == 0 and u.per * n >= u.hi - u.lo for u in pl.units)
    assert pl.shard_len == sum(u.per for u in pl.units)
    full = torch.arange(lay.total, dtype=torch.float32)
    rec = torch.full((lay.total,), -1.0)
    shards = [pl.full_to_shard(full, r, torch.empty(pl.shard_len)) for r in range(n)]
    for r in range(n):
        pl.shard_to_full(shards[r], r, rec)
    assert torch.equal(rec, full)
    small = torch.zeros(pl.small_len)
    for r, so, do, k in pl.small_copies():
        small[do: do + k] = shards[r][so: so + k]
    for name, i in pl.small_index.items():
        o = pl.small_offsets[name]
        assert torch.equal(small[o: o + lay.numels[i]], full[lay.offsets[i]: lay.offsets[i] + lay.numels[i]]), name
    mem, tied = pl.bytes_per_rank(), UnitPlan(layout_for_model_cfg(MC), 12, n)
    assert pl.head_span == pl.units[pl.head].per * n >= 512 * 128
    assert mem["unit_weight_buffers_bf16"] == 4 * pl.max_block_span + 2 * pl.rest_span + 2 * pl.head_span
    assert mem["grad_staging_fp32"] == 8 * pl.max_block_span + 4 * pl.rest_span + 4 * pl.head_span
    assert pl.bytes_per_rank(fp8=True)["unit_weight_buffers_bf16"] == 2 * pl.rest_span + 2 * pl.head_span
    # the block units are those of the tied layout, shifted by the head
    assert [(u.hi - u.lo) for u in pl.units[:13]] == [(u.hi - u.lo) for u in tied.units]


@pytest.mark.parametrize("n", [1, 3])
def test_tied_unit_plan_is_unchanged(n):
    from photon_b200.parallel.zero3 import UnitPlan

    pl = UnitPlan(layout_for_model_cfg(MC), 12, n)
    assert pl.head is None and pl.head_span == 0 and [u.name for u in pl.units] == [f"block.{i}" for i in range(12)] + ["rest"]
    assert pl.units[0].lo == 0 and pl.bytes_per_rank()["unit_weight_buffers_bf16"] == 4 * pl.max_block_span + 2 * pl.rest_span


# ---------------------------------------------------------------------------------------------------- backward plan
def _trainable(frozen=None, unfrozen=None):
    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=4, max_seq_len=256, vocab_size=2048, tie_word_embeddings=False)
    m = MPTForCausalLM(cfg, device="meta", init=False)
    apply_freeze(m, frozen, unfrozen)
    return [n for n, p in m.named_parameters() if p.requires_grad]


def test_plan_only_lm_head_trainable_stops_after_the_head_wgrad():
    p = BackwardPlan(4, _trainable(unfrozen=["lm_head.weight"]), tied=False)
    assert p.runs("head") and p.head_wgrad and not p.dx("head") and not p.runs("norm_f")
    assert p.lowest_block == 4 and not p.runs("embed")


def test_plan_only_wte_trainable_runs_the_chain_without_the_head_wgrad():
    p = BackwardPlan(4, _trainable(unfrozen=["transformer.wte.weight"]), tied=False)
    assert not p.head_wgrad and p.dx("head") and p.runs("embed") and p.lowest_block == 0
    assert p.grad("transformer.wte.weight")


def test_plan_frozen_lm_head():
    p = BackwardPlan(4, _trainable(frozen=["lm_head.weight"]), tied=False)
    assert not p.head_wgrad and p.dx("head") and p.runs("embed") and p.lowest_block == 0
    # tied, the same trainable set would give the head a wgrad into wte
    assert BackwardPlan(4, _trainable(frozen=["lm_head.weight"])).head_wgrad


# ------------------------------------------------------------------------------------------------- federated round
def test_one_federated_round_carries_an_untied_head(tmp_path):
    from photon_b200.config import compose
    from photon_b200.federation import FederationRuntime
    from photon_b200.server_app import run_server
    from test_federation_cpu import TINY

    cfg = compose(TINY + [f"photon.saving_path={tmp_path}", f"llm_config.save_folder={tmp_path}/clients", "run_uuid=head",
                          "fl.n_rounds=1", "++llm_config.model.tie_word_embeddings=false", "++llm_config.model.logit_scale=0.5",
                          "++llm_config.model.final_logit_softcapping=20.0"])
    rt = FederationRuntime(cfg, device=torch.device("cpu"), rank=0, world_size=1)
    h = run_server(cfg, runtime=rt)
    assert rt.model_layout.names[0] == "lm_head.weight"
    fit = h.metrics_distributed_fit
    assert [v for _, v in fit["server/n_failures"]] == [0]
    assert all(np.isfinite(v) for _, v in fit["server/l2_norm_pseudo_gradient"])
    g = rt.round_backend.global_params()
    w = rt.model_layout.view(g, "lm_head.weight")
    assert w.shape == (cfg.llm_config.model.vocab_size, cfg.llm_config.model.d_model) and float(w.abs().sum()) > 0
    # the payload round-trips lm_head.weight: arrays out, into a fresh flat, and back
    arrays = rt.model_layout.to_ndarrays(g)
    assert arrays[0].shape == tuple(w.shape) and np.array_equal(arrays[0], w.cpu().numpy())
    back = torch.zeros_like(g)
    rt.model_layout.from_ndarrays(back, arrays)
    assert torch.equal(rt.model_layout.view(back, "lm_head.weight"), w)
    rt.close()
