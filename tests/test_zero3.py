"""Full parameter sharding (ZeRO-3, ``fsdp_config.sharding_strategy: FULL_SHARD``; ref: photon/conf/llm_config/mpt-7b.yaml:85-91).

CPU: the unit / slice arithmetic and the policy. GPU: the sharded engine against the plain engine (same kernels, so gradients and
parameters must agree to the last bit with one rank), a checkpoint round trip, and two ranks against plain DDP."""
import pytest
import torch

MC = {"name": "mpt_causal_lm", "d_model": 128, "n_heads": 4, "n_layers": 12, "expansion_ratio": 4, "max_seq_len": 64, "vocab_size": 512}


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_unit_plan_partitions_the_flat_space(n):
    from photon_b200.parallel.zero3 import UnitPlan
    from photon_b200.utils.flat import layout_for_model_cfg

    lay = layout_for_model_cfg(MC)
    pl = UnitPlan(lay, 12, n)
    # units tile [0, total) in flat order, blocks in EXECUTION order (the flat layout sorts "blocks.10" before "blocks.2")
    spans = sorted((u.lo, u.hi) for u in pl.units)
    assert spans[0][0] == 0 and spans[-1][1] == lay.total and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert [u.name for u in pl.units] == [f"block.{i}" for i in range(12)] + ["rest"]
    assert pl.units[2].lo > pl.units[11].lo          # lexicographic flat order
    for i, name in enumerate(lay.names):
        u = pl.units[pl.unit_of[i]]
        assert u.lo <= lay.offsets[i] and lay.offsets[i] + lay.numels[i] <= u.hi, name
    assert all(u.per % 256 == 0 and u.per * n >= u.hi - u.lo for u in pl.units)
    assert pl.shard_len == sum(u.per for u in pl.units)
    # every flat index has exactly one owner; shards round-trip
    full = torch.arange(lay.total, dtype=torch.float32)
    rec = torch.full((lay.total,), -1.0)
    shards = []
    for r in range(n):
        sh = pl.full_to_shard(full, r, torch.empty(pl.shard_len))
        shards.append(sh)
        pl.shard_to_full(sh, r, rec)
    assert torch.equal(rec, full)
    assert sum(hi - lo for u in range(len(pl.units)) for lo, hi in [pl.slice_range(u, r) for r in range(n)]) == lay.total
    # the packed buffer of 1-D parameters is assembled from pieces of the owners' shards
    small = torch.zeros(pl.small_len)
    for r, so, do, k in pl.small_copies():
        small[do: do + k] = shards[r][so: so + k]
    for name, i in pl.small_index.items():
        o = pl.small_offsets[name]
        assert torch.equal(small[o: o + lay.numels[i]], full[lay.offsets[i]: lay.offsets[i] + lay.numels[i]]), name
    assert set(pl.small_index) == {nm for nm, shp in zip(lay.names, lay.shapes) if len(shp) <= 1}
    mem = pl.bytes_per_rank()
    assert mem["masters_fp32"] == 4 * pl.shard_len and mem["moments_fp32"] == 8 * pl.shard_len


def test_full_sharding_policy():
    from photon_b200.parallel.ddp import wants_full_sharding

    def cfg(strategy="FULL_SHARD", mode="auto", fsdp=True):
        return {"llm_config": {"fsdp_config": {"sharding_strategy": strategy} if fsdp else None}, "kernels": {"param_sharding": mode}}

    assert wants_full_sharding(cfg(), 6_650_000_000)                  # MPT-7B: 120 GB of replicated state
    assert not wants_full_sharding(cfg(), 125_000_000)                # MPT-125M keeps the fused ZeRO-1 step
    assert not wants_full_sharding(cfg(), 1_320_000_000)              # MPT-1B: 22 GB, fits beside its activations on 80 GB
    assert wants_full_sharding(cfg(), 2_650_000_000)                  # MPT-3B: 44 GB, more than 40 % of an 80 GB H100
    assert not wants_full_sharding(cfg("SHARD_GRAD_OP"), 6_650_000_000)
    assert not wants_full_sharding(cfg(fsdp=False), 6_650_000_000)
    assert wants_full_sharding(cfg(mode="zero3", fsdp=False), 125_000_000)
    assert not wants_full_sharding(cfg(mode="zero1"), 6_650_000_000)


# --------------------------------------------------------------------------------------------------------- GPU
def _engines(n_layers=3, act_ckpt=False):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.parallel.zero3 import NvlZero3Comm
    from photon_b200.utils.flat import layout_for_model_cfg

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=n_layers, max_seq_len=256, vocab_size=2048, attn_impl="flash")
    dev = torch.device("cuda", 0)
    plain = B200Engine(cfg, dev, "amp_bf16", {"cuda_graph": False}, seed=5, activation_checkpointing=act_ckpt)
    comm = NvlZero3Comm(plain.flat.layout, n_layers, rank=0, world_size=1, device=dev)
    shard = B200Engine(cfg, dev, "amp_bf16", {}, seed=5, activation_checkpointing=act_ckpt, zero3=comm)
    return cfg, plain, shard, comm


@pytest.mark.gpu
@pytest.mark.parametrize("act_ckpt", [False, True])
def test_sharded_engine_equals_plain_engine(act_ckpt):
    cfg, plain, shard, comm = _engines(act_ckpt=act_ckpt)
    assert torch.equal(shard.flat.full_params(), plain.flat.params)
    assert shard.flat.params.numel() == comm.plan.shard_len and not shard.use_graph
    denom = float(4 * (cfg.max_seq_len - 1))
    plain.flat.zero_grad(), shard.flat.zero_grad()
    for s in range(2):          # two microbatches: the shard accumulates what the staging planes deliver
        ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device="cuda:0", generator=torch.Generator("cuda").manual_seed(s))
        la, na = plain.fwd_bwd(ids, denom)
        lb, nb = shard.fwd_bwd(ids, denom)
        assert float(na) == float(nb) and abs(float(la) - float(lb)) <= 1e-5 * abs(float(la))   # loss sums are atomics: order-dependent rounding
    torch.cuda.synchronize()
    full = torch.zeros_like(plain.flat.grads)
    comm.plan.shard_to_full(shard.flat.grads, 0, full)
    assert plain.flat.grads.abs().max() > 0
    # same kernels, same order; the only extra operation is `shard += 1.0 * staged` (embedding / LayerNorm gradients are atomics)
    rel = ((full - plain.flat.grads).norm() / plain.flat.grads.norm()).item()
    assert rel < 1e-5, rel
    lay = plain.flat.layout
    for i, n in enumerate(lay.names):
        a, b = lay.view(plain.flat.grads, i), lay.view(full, i)
        assert (a - b).norm() <= 1e-4 * a.norm() + 1e-9, n
    a, b = plain.eval_stats(ids), shard.eval_stats(ids)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) <= 1e-5 * abs(float(a["loss_sum"]))
    # the ICL evaluator's logits() path: a temporary whole-model copy assembled from the shards
    torch.testing.assert_close(shard.logits(ids[:1, :64]).float(), plain.logits(ids[:1, :64]).float(), rtol=1e-3, atol=1e-3)
    shard.train_mode(True)
    assert shard._eval_model is None
    comm.close()


@pytest.mark.gpu
def test_sharded_trainer_steps_and_checkpoints_like_the_plain_one(tmp_path):
    from photon_b200.data.synthetic import synthetic_batch
    from photon_b200.models.mpt import MPTConfig
    from photon_b200.parallel.zero3 import NvlZero3Comm
    from photon_b200.train.trainer import Trainer
    from photon_b200.utils.flat import layout_for_model_cfg

    mc = {"name": "mpt_causal_lm", "d_model": 256, "n_heads": 4, "n_layers": 3, "expansion_ratio": 4, "max_seq_len": 256, "vocab_size": 2048}
    cfg = MPTConfig.from_model_cfg(mc)

    class Loader:
        def __init__(self, start=0):
            self.start = start

        def __iter__(self):
            i = self.start
            while True:
                ids = torch.from_numpy(synthetic_batch(8, 256, seed=1, start=8 * i) % 2048)
                yield {"input_ids": ids.pin_memory(), "labels": ids}
                i += 1

    def make(comm, start=0):
        return Trainer(cfg, optimizer_cfg=dict(name="decoupled_adamw", lr=1e-3, betas=[0.9, 0.95], eps=1e-8, weight_decay=1e-4),
                       scheduler_cfg=dict(name="constant_with_warmup", t_warmup="1ba"), train_loader=Loader(start), global_train_batch_size=8,
                       device_train_microbatch_size=4, precision="amp_bf16", max_duration="30ba", grad_clip_norm=1.0, device="cuda:0",
                       kernels={"cuda_graph": False}, grad_comm=comm, save_folder=str(tmp_path / ("z3" if comm else "plain")))

    def lb_last(t):
        return t.loggers[0].data["loss/train/total"][-1][1]

    plain = make(None)
    comm = NvlZero3Comm(layout_for_model_cfg(mc), 3, rank=0, world_size=1, device=torch.device("cuda", 0))
    z3 = make(comm)
    assert z3.state.flat.is_sharded and z3.state.optimizer.exp_avg.numel() == comm.plan.shard_len
    plain.fit("3ba"), z3.fit("3ba")

    def rel(x, y):
        return ((x - y).norm() / y.norm()).item()

    # noise floor: gradients are accumulated with atomics, so two PLAIN runs already differ in the last bits, and Adam amplifies
    # that over the steps; the sharded run must stay within that band of a plain one
    assert rel(z3.state.flat.full_params(), plain.state.flat.params) < 2e-4
    la, lb = plain.loggers[0].data["loss/train/total"], z3.loggers[0].data["loss/train/total"]
    assert len(la) == len(lb) and all(abs(x[1] - y[1]) < 1e-3 for x, y in zip(la, lb)), (la, lb)
    # checkpoint: the file holds the WHOLE model under the usual names; a fresh sharded trainer resumes from it
    path = z3.save_checkpoint()
    ck = torch.load(path, map_location="cpu", weights_only=False)
    lay = plain.state.flat.layout
    full = z3.state.flat.full_params()
    for i, n in enumerate(lay.names):
        assert torch.equal(ck["state"]["model"][n], lay.view(full, i).cpu()), n
    plain.fit("2ba"), z3.fit("2ba")
    want = z3.state.flat.full_params().clone()
    # (Adam turns the rounding noise of atomically accumulated gradients into +-lr steps where g ~ 0: the distance grows with steps)
    assert rel(want, plain.state.flat.params) < 2e-3, rel(want, plain.state.flat.params)
    z3.close()
    comm2 = NvlZero3Comm(layout_for_model_cfg(mc), 3, rank=0, world_size=1, device=torch.device("cuda", 0))
    again = make(comm2, start=3)
    again.load_checkpoint(path)
    assert again.state.timestamp.batch == 3
    again.fit("2ba")
    assert rel(again.state.flat.full_params(), want) < 2e-3, rel(again.state.flat.full_params(), want)
    assert abs(again.loggers[0].data["loss/train/total"][-1][1] - lb_last(z3)) < 1e-3
    again.close(), plain.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4])
def test_ranks_fully_sharded_match_ddp(tmp_path, n):
    """torchrun, n GPUs: ``kernels.param_sharding=zero3`` (per-block copy-engine gathers + fused reduce-scatter kernel: P2P loads at
    n = 2, in-switch ``multimem.ld_reduce`` from n = 4 when NVLS is up) ends on the same parameters as plain DDP with the fused
    all-reduce; every rank holds 1/n of every plane."""
    from test_multiproc_gpu import _torchrun

    _torchrun(tmp_path, n, """
        from photon_b200.config import compose
        from photon_b200.centralised_train import run_centralised
        rank = dist.get_rank(); dev = torch.device('cuda', rank)
        outs = {}
        for name, extra, cls in (('zero3', ['kernels.param_sharding=zero3'], 'NvlZero3Comm'), ('ddp', ['~llm_config.fsdp_config'], 'NvlGradComm')):
            cfg = compose(TINY + ['run_uuid=z3', 'dataset/streams@dataset.train.streams=centralised', 'dataset.train.root_local=synthetic://7',
                                  'llm_config.model.n_layers=3'] + extra)
            W = dist.get_world_size()
            tr = run_centralised(cfg, device=dev, rank=rank, world_size=W, duration='3ba')
            assert type(tr.grad_comm).__name__ == cls, (name, type(tr.grad_comm).__name__)
            x = tr.state.flat.full_params().clone()
            if name == 'zero3':
                pl = tr.grad_comm.plan
                assert tr.state.flat.params.numel() == pl.shard_len and W * pl.shard_len < 1.01 * pl.layout.total + W * 256 * len(pl.units)
                print('nvls' if tr.grad_comm.arena.mc_ptr('gs0') else 'p2p', flush=True)
                assert tr.state.optimizer.exp_avg.numel() == pl.shard_len
            ref = x.clone(); dist.broadcast(ref, src=0)
            assert torch.equal(ref, x), name + ': ranks assembled different models'
            outs[name] = x; outs[name + '_loss'] = tr.loggers[0].data['loss/train/total'][-1][1]
            tr.close()
        rel = ((outs['zero3'] - outs['ddp']).norm() / outs['ddp'].norm()).item()
        assert rel < 2e-3, rel
        assert abs(outs['zero3_loss'] - outs['ddp_loss']) < 5e-3, (outs['zero3_loss'], outs['ddp_loss'])
        if rank == 0: print('RESULT_OK', rel)
    """, 29547)
