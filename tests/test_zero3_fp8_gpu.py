"""Full parameter sharding (ZeRO-3) under ``precision: amp_fp8``: the block weights are quantised once per parameter version by the
owners of their pieces (``zero3_fp8_requant_kernel``) and gathered as E4M3 bytes.

The numerics contract is exact: with the same bf16 values, the sharded E4M3 bytes and weight scales are bitwise what the
unsharded engine's ``fp8_quantize_segments`` makes from its shadow (same global amax, same scale formula, same rounding code). So
sharded and plain fp8 training differ only by the float-atomic noise the bf16 ZeRO-3 tests already allow for."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _cfg(n_layers=3):
    from photon_b200.models.mpt import MPTConfig

    return MPTConfig(d_model=256, n_heads=4, n_layers=n_layers, max_seq_len=256, vocab_size=2048, attn_impl="flash")


def _comm(layout, n_layers, fp8=True):
    from photon_b200.parallel.zero3 import NvlZero3Comm

    return NvlZero3Comm(layout, n_layers, rank=0, world_size=1, device=torch.device("cuda", 0), fp8=fp8)


def _reference_quant(plan, full16):
    """E4M3 bytes and [scale, 1/scale, amax] of every block matrix of a whole bf16 model, by the unsharded engine's kernel."""
    from photon_b200 import ops

    lay = plan.layout
    seg = torch.tensor([(lay.offsets[lay.index(n)], lay.numels[lay.index(n)]) for n in plan.weight_names], dtype=torch.int64,
                       device=DEV)
    meta = torch.ones(3, len(plan.weight_names), device=DEV)
    dst = torch.zeros(lay.total, dtype=torch.uint8, device=DEV)
    ops.fp8_quantize_segments(full16, dst, seg, meta, 0)
    return dst, meta


def _assembled_bf16(comm):
    full = torch.zeros(comm.plan.layout.total, dtype=torch.bfloat16, device=DEV)
    comm.plan.shard_to_full(comm.w16, 0, full)       # world size 1: the shard is the whole model (+ padding)
    return full


def _check_gathered_units(comm, eng, ref_bytes, ref_meta):
    """Every gathered E4M3 block unit and every weight-role column of the engine's fp8 state equal the reference, bitwise."""
    lay = comm.plan.layout
    for j, name in enumerate(comm.plan.weight_names):
        u = comm.plan.rel(name)[0]
        comm.acquire(u)
        torch.cuda.synchronize()
        assert torch.equal(comm.weight8(name), lay.view(ref_bytes, name)), name
        i, key = j // 4, eng._W_ROLES[j % 4]
        assert eng.w8_views[i][key].data_ptr() == comm.weight8(name).data_ptr()
        assert torch.equal(eng.fp8_meta[:, eng._role(key, i)], ref_meta[:, j]), (name, eng.fp8_meta[:, eng._role(key, i)], ref_meta[:, j])


# ------------------------------------------------------------------------------------------------------------ 1. the kernel
def test_requant_kernel_equals_quantize_segments_bitwise():
    from photon_b200.utils.flat import layout_for_model_cfg

    mc = {"name": "mpt_causal_lm", "d_model": 256, "n_heads": 4, "n_layers": 2, "expansion_ratio": 4, "max_seq_len": 256, "vocab_size": 2048}
    lay = layout_for_model_cfg(mc)
    comm = _comm(lay, 2)
    pl = comm.plan
    g = torch.Generator(DEV).manual_seed(0)
    full = torch.zeros(lay.total, dtype=torch.bfloat16, device=DEV)
    for j, name in enumerate(pl.weight_names):     # a wide range of magnitudes; slot 5 stays all zeros
        if j != 5:
            v = lay.view(full, name)
            v.copy_(torch.randn(v.shape, generator=g, device=DEV) * 10.0 ** (j % 7 - 3))
    lay.view(full, pl.weight_names[2]).view(-1)[7] = 3.0e4        # one outlier dominates its tensor's scale
    pl.full_to_shard(full, 0, comm.w16)
    n_dyn = 3                                                      # weight roles after some other columns, in reverse slot order
    meta = torch.full((3, n_dyn + len(pl.weight_names)), 7.0, device=DEV)
    roles = [n_dyn + len(pl.weight_names) - 1 - j for j in range(len(pl.weight_names))]
    comm.attach_fp8(meta, roles)
    comm.requantize()
    ref_bytes, ref_meta = _reference_quant(pl, full)
    torch.cuda.synchronize()
    for j, name in enumerate(pl.weight_names):
        u, rel, n = pl.rel(name)
        off = pl.units[u].off + rel                                 # world size 1: the shard offset of the whole matrix
        assert torch.equal(comm.w8[off: off + n], ref_bytes[lay.offsets[lay.index(name)]: lay.offsets[lay.index(name)] + n]), name
        assert torch.equal(meta[:, roles[j]], ref_meta[:, j]), (name, meta[:, roles[j]], ref_meta[:, j])
    assert torch.equal(meta[:, :n_dyn], torch.full((3, n_dyn), 7.0, device=DEV))   # other roles untouched
    assert meta[0, roles[5]].item() == 1.0 and meta[1, roles[5]].item() == 1.0 and meta[2, roles[5]].item() == 0.0
    assert meta[2, roles[2]].item() == 3.0e4 or abs(meta[2, roles[2]].item() - 3.0e4) < 64   # (bf16 of 3e4)
    assert int(comm.amax_local.abs().max()) == 0                   # the partials are left zeroed for the next version
    first = comm.w8.clone(), meta.clone()
    comm.requantize()
    torch.cuda.synchronize()
    assert torch.equal(comm.w8, first[0]) and torch.equal(meta, first[1])     # two runs: bitwise equal
    assert int(comm.arena.ctl_words()[comm.ext.ctl_status_word_offset()]) == 0
    comm.close()


# ------------------------------------------------------------------------------------------------------------ 2. the engine
def _engines(act_ckpt):
    from photon_b200.models.engine import B200Engine

    cfg = _cfg()
    plain = [B200Engine(cfg, DEV, "amp_fp8", {"cuda_graph": False}, seed=5, activation_checkpointing=act_ckpt) for _ in range(2)]
    comm = _comm(plain[0].flat.layout, cfg.n_layers)
    shard = B200Engine(cfg, DEV, "amp_fp8", {}, seed=5, activation_checkpointing=act_ckpt, zero3=comm)
    return cfg, plain, shard, comm


@pytest.mark.parametrize("act_ckpt", [False, True])
def test_sharded_fp8_engine_equals_plain_fp8_engine(act_ckpt):
    """Gradients after two microbatches, relative L2 distance of the whole vector. Observed on an H100 80GB HBM3: plain fp8 vs
    plain fp8 1.5e-8 to 1.7e-8 (the float-atomic noise band), sharded vs plain 1.8e-8, with and without activation checkpointing.
    The bound is 4x the band of the two plain runs, with a floor of 2e-3 overall and 2e-2 of the norm per tensor."""
    cfg, (plain, plain2), shard, comm = _engines(act_ckpt)
    assert shard.fp8 and shard.w8 is None and shard._n_w8 == 0 and not shard.use_graph
    assert torch.equal(shard.flat.full_params(), plain.flat.params)
    # the weights the plain engine quantises at the start of a microbatch = the sharded engine's gathered units, bitwise
    plain._fp8_prologue(train=False)
    torch.cuda.synchronize()
    lay = plain.flat.layout
    for i in range(cfg.n_layers):
        comm.acquire(i)
        torch.cuda.synchronize()
        for key in plain._W_ROLES:
            assert torch.equal(shard.w8_views[i][key], plain.w8_views[i][key]), (i, key)
            r = plain._role(key, i)
            assert torch.equal(shard.fp8_meta[:, r], plain.fp8_meta[:, r]), (i, key)
    denom = float(4 * (cfg.max_seq_len - 1))
    for e in (plain, plain2, shard):
        e.flat.zero_grad()
    for s in range(2):
        ids = torch.randint(0, cfg.vocab_size, (4, cfg.max_seq_len), device=DEV, generator=torch.Generator("cuda").manual_seed(s))
        la, na = plain.fwd_bwd(ids, denom)
        l2, _ = plain2.fwd_bwd(ids, denom)
        lb, nb = shard.fwd_bwd(ids, denom)
        assert float(na) == float(nb) and abs(float(la) - float(lb)) <= 1e-5 * abs(float(la)), (float(la), float(lb), float(l2))
    torch.cuda.synchronize()
    full = torch.zeros_like(plain.flat.grads)
    comm.plan.shard_to_full(shard.flat.grads, 0, full)
    assert plain.flat.grads.abs().max() > 0

    def rel(x, y):
        return ((x - y).norm() / y.norm()).item()

    band, got = rel(plain2.flat.grads, plain.flat.grads), rel(full, plain.flat.grads)
    print(f"[zero3-fp8] act_ckpt={act_ckpt}: gradient band plain-vs-plain {band:.3e}, sharded-vs-plain {got:.3e}", flush=True)
    assert got <= max(4 * band, 2e-3), (got, band)
    for i, n in enumerate(lay.names):
        a, b, c = lay.view(plain.flat.grads, i), lay.view(full, i), lay.view(plain2.flat.grads, i)
        assert (a - b).norm() <= max(4 * (a - c).norm().item(), 2e-2 * a.norm().item()) + 1e-9, n
    # the scales of the weights stayed paired with the bytes, and evaluation runs on the same weights
    for i in range(cfg.n_layers):
        for key in plain._W_ROLES:
            assert torch.equal(shard.fp8_meta[:, plain._role(key, i)], plain.fp8_meta[:, plain._role(key, i)])
    a, b = plain.eval_stats(ids), shard.eval_stats(ids)
    assert abs(float(a["loss_sum"]) - float(b["loss_sum"])) <= 1e-5 * abs(float(a["loss_sum"]))
    comm.close()


def test_fp8_sharded_engine_memory():
    """No full-size E4M3 copy on the engine and no bf16 block unit buffers: the communicator holds exactly the buffers of
    ``bytes_per_rank(fp8=True)``."""
    from photon_b200.models.engine import B200Engine
    from photon_b200.utils.flat import layout_for_model_cfg

    cfg = _cfg()
    mc = {"name": "mpt_causal_lm", "d_model": 256, "n_heads": 4, "n_layers": 3, "expansion_ratio": 4, "max_seq_len": 256, "vocab_size": 2048}
    comm = _comm(layout_for_model_cfg(mc), 3)
    eng = B200Engine(cfg, DEV, "amp_fp8", {}, seed=5, zero3=comm)
    assert eng.w8 is None and eng.w8_seg is None and comm.wbuf is None
    assert all(v is None for w in eng.layers for v in (w.wqkv, w.wo, w.wup, w.wdown))
    mem = comm.plan.bytes_per_rank(fp8=True)
    nb = lambda *ts: sum(t.numel() * t.element_size() for t in ts)  # noqa: E731
    assert nb(comm.p32) == mem["masters_fp32"] and nb(comm.w16) == mem["bf16_copy"] and nb(comm.gshard) == mem["grad_shard_fp32"]
    assert nb(comm.wrest) == mem["unit_weight_buffers_bf16"] and nb(*comm.wbuf8) == mem["unit_weight_buffers_e4m3"]
    assert nb(comm.w8) == mem["e4m3_shard"] and nb(comm.amax, comm.amax_local) == mem["amax_fp32"]
    assert nb(*comm.gstage, comm.gstage_rest) == mem["grad_staging_fp32"] and nb(comm.small32) == mem["small_fp32"]
    # the precision and the communicator must agree
    with pytest.raises(ValueError):
        B200Engine(cfg, DEV, "amp_bf16", {}, seed=5, zero3=_comm(layout_for_model_cfg(mc), 3))
    with pytest.raises(ValueError):
        B200Engine(cfg, DEV, "amp_fp8", {}, seed=5, zero3=_comm(layout_for_model_cfg(mc), 3, fp8=False))
    comm.close()


# ------------------------------------------------------------------------------------------------------------ 3. the trainer
def test_sharded_fp8_trainer_steps_and_checkpoints_like_the_plain_one(tmp_path):
    from photon_b200.data.synthetic import synthetic_batch
    from photon_b200.models.mpt import MPTConfig
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
                       device_train_microbatch_size=4, precision="amp_fp8", max_duration="30ba", grad_clip_norm=1.0, device="cuda:0",
                       kernels={"cuda_graph": False}, grad_comm=comm, save_folder=str(tmp_path / ("z3" if comm else "plain")))

    def paired(tr):
        comm = tr.grad_comm
        ref_bytes, ref_meta = _reference_quant(comm.plan, _assembled_bf16(comm))
        _check_gathered_units(comm, tr.state.backend, ref_bytes, ref_meta)

    plain = make(None)
    comm = _comm(layout_for_model_cfg(mc), 3)
    z3 = make(comm)
    assert z3.state.flat.is_sharded and z3.state.backend.fp8 and z3.state.backend.w8 is None
    paired(z3)
    for _ in range(3):
        plain.fit("1ba"), z3.fit("1ba")
        paired(z3)                        # after every optimizer step: the E4M3 units are the quantisation of the new weights

    def rel(x, y):
        return ((x - y).norm() / y.norm()).item()

    print(f"[zero3-fp8] trainer, 3 steps: params sharded-vs-plain {rel(z3.state.flat.full_params(), plain.state.flat.params):.3e}",
          flush=True)
    assert rel(z3.state.flat.full_params(), plain.state.flat.params) < 2e-4
    la, lb = plain.loggers[0].data["loss/train/total"], z3.loggers[0].data["loss/train/total"]
    assert len(la) == len(lb) and all(abs(x[1] - y[1]) < 1e-3 for x, y in zip(la, lb)), (la, lb)
    # checkpoint: the fp8 scaling state travels with it; a resumed sharded trainer requantises so bytes and scales stay paired
    path = z3.save_checkpoint()
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert any(isinstance(v, dict) and "meta" in v for v in _walk(ck)), "the checkpoint carries the fp8 scaling state"
    plain.fit("2ba"), z3.fit("2ba")
    want = z3.state.flat.full_params().clone()
    assert rel(want, plain.state.flat.params) < 2e-3, rel(want, plain.state.flat.params)
    z3.close()
    comm2 = _comm(layout_for_model_cfg(mc), 3)
    again = make(comm2, start=3)
    again.load_checkpoint(path)
    assert again.state.timestamp.batch == 3 and again.state.backend._fp8_calibrated
    paired(again)
    again.fit("2ba")
    paired(again)
    assert rel(again.state.flat.full_params(), want) < 2e-3, rel(again.state.flat.full_params(), want)
    assert abs(again.loggers[0].data["loss/train/total"][-1][1] - z3.loggers[0].data["loss/train/total"][-1][1]) < 1e-3
    again.close(), plain.close()


def _walk(d):
    if isinstance(d, dict):
        yield d
        for v in d.values():
            yield from _walk(v)


# ------------------------------------------------------------------------------------------------------------ 4. several GPUs
@pytest.mark.parametrize("n", [2, 4])
def test_ranks_fully_sharded_fp8_match_ddp_fp8(tmp_path, n):
    """torchrun, n GPUs: ``kernels.param_sharding=zero3`` with ``precision=amp_fp8`` ends on the same parameters as DDP amp_fp8;
    after every step all ranks hold bitwise equal weight scales (the amax exchange is global) and rank 0's gathered E4M3 units are
    the quantisation of the whole bf16 model. P2P amax / flag traffic at n = 2; n = 4 runs on the NVLS arena when the box has it."""
    from test_multiproc_gpu import _torchrun

    _torchrun(tmp_path, n, """
        from photon_b200 import ops
        from photon_b200.config import compose
        from photon_b200.centralised_train import run_centralised
        rank = dist.get_rank(); dev = torch.device('cuda', rank)
        outs = {}
        for name, extra, cls in (('zero3', ['kernels.param_sharding=zero3'], 'NvlZero3Comm'), ('ddp', ['~llm_config.fsdp_config'], 'NvlGradComm')):
            cfg = compose(TINY + ['run_uuid=z3f8', 'dataset/streams@dataset.train.streams=centralised', 'dataset.train.root_local=synthetic://7',
                                  'llm_config.model.n_layers=3', 'llm_config.precision=amp_fp8'] + extra)
            W = dist.get_world_size()
            tr = run_centralised(cfg, device=dev, rank=rank, world_size=W, duration='1ba')
            assert type(tr.grad_comm).__name__ == cls, (name, type(tr.grad_comm).__name__)
            be = tr.state.backend
            assert be.fp8
            for step in range(3):
                if step:
                    tr.fit('1ba')
                if name != 'zero3':
                    continue
                z = tr.grad_comm
                cols = be.fp8_meta[:, be._n_dyn:].clone()
                ref = cols.clone(); dist.broadcast(ref, src=0)
                assert torch.equal(ref, cols), 'ranks hold different weight scales'
                full16 = tr.state.flat.full_params().to(torch.bfloat16)
                if rank == 0:
                    lay = z.plan.layout
                    seg = torch.tensor([(lay.offsets[lay.index(m)], lay.numels[lay.index(m)]) for m in z.plan.weight_names], dtype=torch.int64, device=dev)
                    meta = torch.ones(3, len(seg), device=dev); dst = torch.zeros(lay.total, dtype=torch.uint8, device=dev)
                    ops.fp8_quantize_segments(full16, dst, seg, meta, 0)
                    for j, m in enumerate(z.plan.weight_names):
                        z.acquire(z.plan.rel(m)[0]); torch.cuda.synchronize(dev)
                        assert torch.equal(z.weight8(m), lay.view(dst, m)), m
                        assert torch.equal(be.fp8_meta[:, be._role(be._W_ROLES[j % 4], j // 4)], meta[:, j]), m
                dist.barrier()
            if name == 'zero3':
                print('nvls' if tr.grad_comm.arena.mc_ptr('gs0') else 'p2p', flush=True)
            x = tr.state.flat.full_params().clone()
            ref = x.clone(); dist.broadcast(ref, src=0)
            assert torch.equal(ref, x), name + ': ranks assembled different models'
            outs[name] = x; outs[name + '_loss'] = tr.loggers[0].data['loss/train/total'][-1][1]
            tr.close()
        rel = ((outs['zero3'] - outs['ddp']).norm() / outs['ddp'].norm()).item()
        assert rel < 2e-3, rel
        assert abs(outs['zero3_loss'] - outs['ddp_loss']) < 5e-3, (outs['zero3_loss'], outs['ddp_loss'])
        if rank == 0: print('RESULT_OK', rel)
    """, 29548)
