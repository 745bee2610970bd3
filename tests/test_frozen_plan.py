"""The engine's backward plan for partly frozen models (CPU: a pure function of the config and the trainable names)."""
import pytest

from photon_b200.models.engine import BLOCK_STAGES, BackwardPlan
from photon_b200.models.mpt import MPTConfig, MPTForCausalLM
from photon_b200.train.backend import apply_freeze

L = 4
ALL_STAGES = [s for s, _ in BLOCK_STAGES]


def _trainable(frozen=None, unfrozen=None, **kw):
    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=L, max_seq_len=256, vocab_size=2048, **kw)
    m = MPTForCausalLM(cfg, device="meta", init=False)
    apply_freeze(m, frozen, unfrozen)
    names = [n for n, _ in m.named_parameters()]
    return names, [n for n, p in m.named_parameters() if p.requires_grad]


NAMES, _ = _trainable()
EMB = ["transformer.wte.weight", "transformer.wpe.weight"]
LOWER = EMB + [n for n in NAMES if any(f".blocks.{i}." in n for i in range(L // 2))]
FFN1 = [n for n in NAMES if ".blocks.1.ffn." in n]
NORMS_BIASES = [n for n in NAMES if ".norm_" in n or "norm_f" in n or n.endswith(".bias")]


def test_nothing_frozen_is_the_full_schedule():
    p = BackwardPlan(L, NAMES)
    assert p.lowest_block == 0 and p.head_wgrad and p.runs("head") and p.dx("head") and p.runs("norm_f") and p.dx("norm_f")
    for i in range(L):
        assert p.block_stages(i) == ALL_STAGES
        assert all(p.dx((i, s)) for s in ALL_STAGES)
    assert p.runs("embed") and not p.dx("embed")
    assert all(p.grad(n) for n in NAMES)


def test_frozen_wte_skips_the_head_wgrad_only():
    _, tr = _trainable(frozen=["transformer.wte.weight"])
    p = BackwardPlan(L, tr)
    assert not p.head_wgrad and p.dx("head")
    assert p.lowest_block == 0 and all(p.block_stages(i) == ALL_STAGES for i in range(L))
    assert p.runs("embed") and not p.grad("transformer.wte.weight") and p.grad("transformer.wpe.weight")


def test_frozen_wpe_keeps_the_whole_backward():
    _, tr = _trainable(frozen=["transformer.wpe.weight"])
    p = BackwardPlan(L, tr)
    assert p.head_wgrad and p.lowest_block == 0 and p.runs("embed") and p.dx((0, "ln1"))
    assert not p.grad("transformer.wpe.weight")


def test_embeddings_and_lower_half_frozen_stop_at_the_first_trainable_block():
    _, tr = _trainable(frozen=LOWER)
    p = BackwardPlan(L, tr)
    assert not p.head_wgrad and p.dx("head")
    assert p.lowest_block == L // 2
    for i in range(L // 2):
        assert p.block_stages(i) == []
    low = L // 2
    assert p.block_stages(low) == ALL_STAGES
    # the lowest trainable block still needs the QKV dgrad (its norm_1 is trainable), but no gradient below its LN1
    assert p.dx((low, "qkv")) and not p.dx((low, "ln1"))
    assert not p.runs("embed")


def test_only_one_block_ffn_trainable_stops_after_that_half():
    _, tr = _trainable(unfrozen=FFN1)
    p = BackwardPlan(L, tr)
    assert p.lowest_block == 1
    assert p.block_stages(1) == ["down", "up"]
    assert p.dx((1, "down")) and not p.dx((1, "up"))   # up-projection wgrad runs, its dgrad (into LN2) does not
    for i in range(2, L):
        assert p.block_stages(i) == ALL_STAGES          # the gradient still flows down through the blocks above
    assert not p.runs("embed") and not p.head_wgrad
    assert all(p.grad(n) == (n in FFN1) for n in NAMES)


def test_frozen_norms_and_biases_skip_their_gradients_but_not_the_chain():
    _, tr = _trainable(frozen=NORMS_BIASES)
    p = BackwardPlan(L, tr)
    assert p.lowest_block == 0 and all(p.block_stages(i) == ALL_STAGES for i in range(L)) and p.runs("embed")
    assert not any(p.grad(n) for n in NORMS_BIASES)
    assert p.grad("transformer.blocks.0.attn.Wqkv.weight")


def test_only_wte_trainable_runs_the_whole_chain_for_the_tied_embedding():
    _, tr = _trainable(unfrozen=["transformer.wte.weight"])
    p = BackwardPlan(L, tr)
    assert p.head_wgrad and p.runs("embed") and p.lowest_block == 0
    assert all(p.block_stages(i) == ALL_STAGES for i in range(L))
    assert p.trainable == {"transformer.wte.weight"}


def test_only_the_last_block_trainable():
    _, tr = _trainable(unfrozen=[n for n in NAMES if f".blocks.{L - 1}." in n])
    p = BackwardPlan(L, tr)
    assert p.lowest_block == L - 1 and p.block_stages(L - 1) == ALL_STAGES and not p.dx((L - 1, "ln1"))
    assert not p.runs("embed") and not p.head_wgrad


@pytest.mark.parametrize("kw", [dict(no_bias=True), dict(qk_ln=True), dict(alibi=True, learned_pos_emb=False)])
def test_q_k_layernorm_and_missing_tensors(kw):
    names, _ = _trainable(**kw)
    p = BackwardPlan(L, names)
    assert all(p.block_stages(i) == ALL_STAGES for i in range(L)) and p.runs("embed")
    if kw.get("qk_ln"):
        # with every tensor below frozen, trainable q/k LayerNorms are the last stage of their block
        only = [n for n in names if ".blocks.2.attn.q_ln." in n]
        q = BackwardPlan(L, only)
        assert q.lowest_block == 2 and q.block_stages(2) == ["down", "up", "ln2", "out", "attn"] and not q.dx((2, "attn"))
