"""Centralised (non-federated) training entry point — the DDP baseline path of the reference
(ref: photon/centralised_train.py:56-166; launched by ``composer --world_size N`` at
scripts/centralised_training.sh:132).  Launch with torchrun; on >1 GPU the gradient all-reduce
is ONE fused NVLink kernel on the flat bucket (``photon_b200.parallel.ddp.NvlGradComm``),
fused with the clipping norm — not 148 NCCL calls.

    PHOTON_SAVE_PATH=... torchrun --nproc-per-node 8 -m photon_b200.centralised_train
"""
from __future__ import annotations

import os
from pathlib import Path
from typing import Any

import numpy as np
import torch

from photon_b200.clients.configs import CentralizedConfig
from photon_b200.clients.trainer_utils import get_trainer_object, initialize_dist, pick_device
from photon_b200.config import load_config
from photon_b200.train.trainer import Trainer
from photon_b200.utils.core import dump_model_parameters_to_file, load_model_parameters_from_file, set_wte_parameters_to_trainer


def _centralized_config(cfg: Any) -> CentralizedConfig:
    c, fl = dict(cfg.get("centralized") or {}), dict(cfg.get("fl") or {})
    return CentralizedConfig(**c, use_unigram_metrics=bool(fl.get("use_unigram_metrics", False)),
                             allow_unigram_metrics_failures=bool(fl.get("allow_unigram_metrics_failures", False)),
                             resize_vocab=fl.get("resize_vocab"), frozen_layers=fl.get("frozen_layers"),
                             unfrozen_layers=fl.get("unfrozen_layers"), pretrained_model_path=cfg.get("pretrained_model_path"),
                             wte_parameters_path=cfg.get("wte_parameters_path"))


def set_wte_parameters(trainer: Trainer, wte: np.ndarray) -> None:
    """Transplant only the token embedding (ref: photon/utils.py:585-599)."""
    set_wte_parameters_to_trainer(trainer, wte)


def resume_centralised(trainer: Trainer, train_cfg: Any) -> Path | None:
    """``llm_config.load_path`` (explicit, may contain ``{rank}``; ``load_ignore_keys`` globs honoured) or — Composer's
    ``autoresume`` — the ``latest-rank{R}.pt`` of the run's own ``save_folder``. Autoresume defaults to ON when a save
    folder is set and ``save_overwrite`` is off, like the reference (ref: clients/trainer_utils.py:437-450). Takes
    precedence over ``pretrained_model_path`` because it restores optimizer, clock and data position too."""
    load_path = train_cfg.get("load_path")
    if load_path:
        path = Path(str(load_path).format(rank=trainer.rank))
        from photon_b200.clients.trainer_utils import load_kwargs_from_config

        trainer.load_checkpoint(path, **load_kwargs_from_config(train_cfg))
        return path
    folder = trainer.save_folder
    auto = bool(train_cfg.get("autoresume")) or (folder is not None and not trainer.save_overwrite)
    if auto and folder is not None:
        latest = Path(str(folder)) / f"latest-rank{trainer.rank}.pt"
        if latest.exists():
            trainer.load_checkpoint(latest)
            print(f"[centralised_train] autoresume from {latest} at batch {trainer.state.timestamp.batch}")
            return latest
    return None


def dump_checkpoint_npz(trainer: Trainer, run_uuid: str, out_dir: str | Path = ".") -> Path:
    """``{run_uuid}-{n_steps}-checkpoint.npz`` with arr_i in sorted-name order (ref: :139-166)."""
    st = trainer.state
    path = Path(out_dir) / f"{run_uuid}-{st.timestamp.batch}-checkpoint.npz"
    return dump_model_parameters_to_file(path, st.flat.to_ndarrays())


def run_centralised(cfg: Any, *, device: torch.device | None = None, rank: int | None = None, world_size: int | None = None,
                    duration: str | None = None, use_nvl_allreduce: bool | None = None, grad_comm: Any = None) -> Trainer:
    """``grad_comm``: an explicit gradient communicator (e.g. ``NcclPerTensorGradComm`` for baseline measurements); default =
    the fused NVLink kernels on a GPU box, one flat NCCL all-reduce otherwise."""
    cc = _centralized_config(cfg)
    device = device or pick_device(int(os.environ.get("LOCAL_RANK", "0")))
    if rank is None or world_size is None:
        rank, world_size = initialize_dist(device)
    if world_size > 1 and grad_comm is None:
        if use_nvl_allreduce is None:
            use_nvl_allreduce = device.type == "cuda" and not all(
                (cfg.get("kernels") or {}).get(k, "auto") == "torch" for k in ("gemm", "optimizer"))
        if use_nvl_allreduce:
            from photon_b200.parallel.ddp import build_nvl_comm, wants_full_sharding, wants_sharded_step
            from photon_b200.utils.flat import layout_for_model_cfg

            lay = layout_for_model_cfg(cfg["llm_config"]["model"], cc.frozen_layers, cc.unfrozen_layers)
            if wants_full_sharding(cfg, lay.n_params, device) and not (cc.frozen_layers or cc.unfrozen_layers):
                from photon_b200.parallel.zero3 import NvlZero3Comm

                # fsdp_config FULL_SHARD on a model whose replicated state would crowd the GPU: parameters, gradients and
                # optimizer state all live as 1/world shards (ZeRO-3); smaller models keep the faster fused ZeRO-1 step
                grad_comm = NvlZero3Comm(lay, int(cfg["llm_config"]["model"]["n_layers"]), rank=rank, world_size=world_size, device=device,
                                         fp8=cfg["llm_config"].get("precision", "amp_bf16") == "amp_fp8")
                print(f"[centralised_train] full parameter sharding over {world_size} GPUs "
                      f"({lay.n_params / 1e9:.2f} B parameters, {16 * grad_comm.plan.shard_len / 2**30:.1f} GiB of state per GPU)", flush=True)
            else:
                grad_comm = build_nvl_comm(lay.total, sharded=wants_sharded_step(cfg["llm_config"]), rank=rank, world_size=world_size, device=device)
        else:
            from photon_b200.parallel.ddp import NcclGradComm

            grad_comm = NcclGradComm()
    trainer, train_cfg = get_trainer_object(cfg, cc.stream_id, log_name="_centralised", device=device, rank=rank, world_size=world_size,
                                    grad_comm=grad_comm, split_eval=cc.split_eval, use_unigram_metrics=cc.use_unigram_metrics,
                                    allow_unigram_metrics_failures=cc.allow_unigram_metrics_failures, frozen_layers=cc.frozen_layers,
                                    unfrozen_layers=cc.unfrozen_layers, resize_vocab=cc.resize_vocab)
    if cc.pretrained_model_path:
        arrays = load_model_parameters_from_file(cc.pretrained_model_path)
        trainer.state.flat.load_ndarrays(arrays[: len(trainer.state.flat.names)])
        trainer.state.backend.params_updated()
    if cc.wte_parameters_path:
        # a FULL model file whose token embedding is transplanted on top of whatever was loaded above
        # (ref: centralised_train.py:98-117); a one-array file holding just the embedding is accepted too
        donor = load_model_parameters_from_file(cc.wte_parameters_path)
        names = list(trainer.state.flat.names)
        if len(donor) >= len(names):
            wte = donor[names.index("transformer.wte.weight")]
        elif len(donor) == 1:
            wte = donor[0]
        else:
            raise ValueError(f"wte_parameters_path holds {len(donor)} arrays; expected a full model ({len(names)}) or the embedding alone")
        set_wte_parameters(trainer, wte)
    resume_centralised(trainer, train_cfg)
    if world_size > 1 and not getattr(trainer.state.flat, "is_sharded", False):  # identical start on every rank
        # (fully sharded runs: every rank initialises from the same seed / loads the same file and keeps only its slices)
        torch.distributed.broadcast(trainer.state.flat.params, src=0)
        trainer.state.backend.params_updated()
    run_uuid = str(cfg["run_uuid"])
    if cfg["llm_config"].get("eval_first") and trainer.eval_loaders:
        trainer.eval()
    if cc.store_init_model and rank == 0:
        dump_checkpoint_npz(trainer, run_uuid)
    if not cc.eval_only:
        trainer.fit(duration=duration, reset_time=cc.reset_timestamp)
    elif trainer.eval_loaders:
        trainer.eval()
    if cc.store_final_model and rank == 0:
        dump_checkpoint_npz(trainer, run_uuid)
    return trainer


def dump_metrics(trainer: Trainer, path: str | os.PathLike) -> Path:
    """Everything the run logged (``{key: [[batch, value], …]}`` from the in-memory logger) + the final clock, as plain JSON."""
    import json

    mem = next((lg for lg in trainer.loggers if hasattr(lg, "data")), None)
    out = {"timestamp": {k: v for k, v in trainer.state.timestamp.state_dict().items() if isinstance(v, (int, float))},
           "metrics": {k: [[int(s), float(v)] for s, v in vals] for k, vals in (mem.data if mem is not None else {}).items()}}
    p = Path(path)
    p.write_text(json.dumps(out, indent=1))
    return p


def main() -> None:
    save_path = os.environ.get("PHOTON_SAVE_PATH")
    if not save_path:
        raise SystemExit("PHOTON_SAVE_PATH must point at the directory holding config.yaml")
    cfg = load_config(Path(save_path) / "config.yaml")
    tr = run_centralised(cfg)
    if tr.rank == 0:
        dump_metrics(tr, Path(save_path) / "centralised_metrics.json")
        print("[centralised_train] done:", tr.state.timestamp, tr.state.train_metric_values)
    tr.close()


if __name__ == "__main__":
    main()
