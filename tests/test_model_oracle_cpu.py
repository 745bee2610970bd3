"""The whole-model fp64 oracle and its criterion (``model_oracle``), on the CPU: the oracle computes in float64 only, agrees
with the fp32 module, and the criterion flags small planted errors on top of the bf16 baseline."""
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode
from torch.utils._pytree import tree_flatten

import model_oracle as MO
from photon_b200.models.mpt import MPTConfig, MPTForCausalLM

BASE = dict(d_model=256, n_heads=4, n_layers=2, max_seq_len=160, vocab_size=1000, ffn_hidden_size=520)
PURITY = {
    "default": {},
    "alibi": dict(alibi=True, learned_pos_emb=False),
    "rmsnorm_rope_untied_cap": dict(norm_type="rmsnorm", qk_ln=True, rope=True, learned_pos_emb=False, tie_word_embeddings=False,
                                    logit_scale=1.5, final_logit_softcapping=5.0, kv_n_heads=2),
}
B, S = 2, 128


def _setup(extra, seed=0):
    cfg = MPTConfig(**BASE, **extra)
    weights = MO.bf16_exact_weights(MPTForCausalLM(cfg, seed=seed).named_parameters(), seed)
    g = torch.Generator().manual_seed(seed + 1)
    batches = [MO.Batch(torch.randint(0, cfg.vocab_size, (B, S), generator=g), scale=s, denom=2.0 * B * (S - 1))
               for s in (1.0, 0.6)]
    return cfg, weights, batches


class _Probe(TorchDispatchMode):
    """Records every (op, dtype) of a floating-point tensor other than float64 among the inputs and outputs of every op."""

    def __init__(self):
        super().__init__()
        self.seen = set()

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        for t in tree_flatten((args, kwargs, out))[0]:
            if isinstance(t, torch.Tensor) and t.is_floating_point() and t.dtype != torch.float64:
                self.seen.add((str(func), t.dtype))
        return out


@pytest.mark.parametrize("variant", list(PURITY))
def test_oracle_computes_in_float64_only(variant):
    cfg, weights, batches = _setup(PURITY[variant])
    m = MO.build(cfg, weights, torch.float64)   # built outside the probe: construction starts in fp32
    with _Probe() as probe:
        res = MO.run(m, batches[:1])
    assert not probe.seen, sorted(probe.seen)
    assert all(g.dtype == torch.float64 for g in res.grads.values())


@pytest.mark.parametrize("variant", list(PURITY))
def test_oracle_matches_fp32_module_and_baseline_differs(variant):
    cfg, weights, batches = _setup(PURITY[variant])
    ref = MO.oracle(cfg, weights, batches)
    m = MO.build(cfg, weights, torch.float32)
    total = 0.0
    for mb in batches:
        loss, n = m.loss(mb.ids, reduction="sum")
        (loss * (mb.scale / mb.denom)).backward()
        total += float(loss.detach())
    assert abs(total - ref.loss_sum) <= 1e-5 * abs(ref.loss_sum), (total, ref.loss_sum)
    assert ref.n_tokens == 2 * B * (S - 1)
    for n, p in m.named_parameters():
        o = ref.grads[n]
        rel = float((p.grad.double() - o).norm() / o.norm())
        assert rel < 1e-4, (n, rel)
    base = MO.baseline(cfg, weights, batches)
    for n, o in ref.grads.items():
        rel = float((base.grads[n] - o).norm() / o.norm())
        assert rel > 1e-4, (n, rel)   # bf16 arithmetic: the yardstick is not zero
    lrel = float((base.logits[0] - ref.logits[0]).norm() / ref.logits[0].norm())
    assert 1e-4 < lrel < 0.05, lrel


def test_check_tensor_passes_the_baseline_and_flags_plants():
    """Each plant is applied to the bf16 baseline's gradient and checked with the baseline as the yardstick: the criterion
    must flag every plant, and pass the baseline itself on every tensor."""
    cfg, weights, batches = _setup({})
    ref = MO.oracle(cfg, weights, batches)
    base = MO.baseline(cfg, weights, batches)
    for n, o in ref.grads.items():
        rep = MO.tensor_report(n, base.grads[n], o, base.grads[n])
        assert not MO.failed_parts(rep), rep["msg"]
    # the exact-zero part has something to check: wpe rows S.. of the oracle are exactly zero
    assert bool((ref.grads["transformer.wpe.weight"][S:] == 0).all())
    one = MO.baseline(cfg, weights, batches[:1])   # the first microbatch's contribution only
    for name, got in MO.plants(cfg, S, base.grads, one.grads).items():
        tensor = name.split(" ")[0]
        rep = MO.tensor_report(tensor, got, ref.grads[tensor], base.grads[tensor])
        print(name, MO.failed_parts(rep), rep["msg"])
        assert MO.failed_parts(rep), f"plant not flagged: {name}: {rep['msg']}"


def test_check_tensor_flags_nonzero_where_the_oracle_is_zero():
    o = torch.zeros(300, 8, dtype=torch.float64)
    o[:200] = torch.randn(200, 8, dtype=torch.float64)
    b = o + 1e-3 * torch.randn_like(o) * (o != 0)
    g = b.clone()
    g[250, 3] = 1e-30
    assert MO.failed_parts(MO.tensor_report("x", g, o, b)) == ["zeros"]
